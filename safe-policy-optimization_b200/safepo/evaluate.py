"""Evaluate saved runs: the reference's safepo/evaluate.py (same functions, same CLI, same ``eval_result.txt`` line).

    python -m safepo.evaluate --benchmark-dir runs/single_agent_exp --eval-episodes 3

walks ``<benchmark-dir>/<env>/<algo>/<seed-run>/``, evaluates every run directory with deterministic actions and appends one
line per (env, algo) with the mean ± std over the seeds to ``<save-dir>/eval_result.txt`` (default: the benchmark directory
with ``runs`` replaced by ``results``).

* A single-agent run (written by safepo.single_agent.*) is rebuilt from its ``config.json``: the environment it trained on
  (``env``: ``synthetic`` or ``mujoco``; a run without the key, such as one of the reference's own, is a MuJoCo run), the
  last ``torch_save/model*.pt`` loaded into the actor and the last ``state*.pkl``'s Normalizer installed as the running
  observation statistics when the run normalised observations.  "Last" is ``sorted(...)[-1]`` as in the reference
  (evaluate.py:36,41): a string sort, so ``model99.pt`` comes after ``model100.pt``.
* A multi-agent run (``algorithm_name`` one of mappolag / mappo / happo / macpo) is restored from ``models_seed{seed}`` and
  evaluated with that algorithm's ``Runner.eval``.

Real MuJoCo environments need the safety_gymnasium package; without it the evaluation raises SpoError, as training does.
The policy runs on the current CUDA device; there is no CPU path."""
from __future__ import annotations

import argparse
import json
import os
from collections import deque

import numpy as np
import torch

from safepo._lib import SpoError

MULTI_AGENT_ALGOS = ("mappolag", "mappo", "happo", "macpo")


def _config(eval_dir):
    path = os.path.join(eval_dir, "config.json")
    if not os.path.isfile(path):
        raise SpoError(f"{eval_dir}: no config.json")
    with open(path) as f:
        return json.load(f)


def _last(directory, suffix):
    """sorted(...)[-1] of the file names ending in ``suffix`` (evaluate.py:34-41): a string sort."""
    names = sorted(n for n in os.listdir(directory) if n.endswith(suffix)) if os.path.isdir(directory) else []
    if not names:
        raise SpoError(f"{directory}: no *{suffix} file")
    return os.path.join(directory, names[-1])


def _load_actor(policy, path):
    """The saved actor state_dict into the packed parameters; SpoError naming a missing, unexpected or misshapen key."""
    sd = torch.load(path, map_location="cpu", weights_only=True)
    if not isinstance(sd, dict):
        raise SpoError(f"{path}: not a state_dict")
    want = policy.actor.state_dict()
    for k, v in want.items():
        if k not in sd:
            raise SpoError(f"{path}: missing key {k!r}")
        if not torch.is_tensor(sd[k]) or tuple(sd[k].shape) != tuple(v.shape):
            got = tuple(sd[k].shape) if torch.is_tensor(sd[k]) else type(sd[k]).__name__
            raise SpoError(f"{path}: key {k!r} has shape {got}, expected {tuple(v.shape)}")
    extra = sorted(set(sd) - set(want))
    if extra:
        raise SpoError(f"{path}: unexpected key {extra[0]!r}")
    policy.actor.load_state_dict(sd)


def _load_normalizer(path, obs_dim, device):
    """The pickled "Normalizer" (gymnasium's RunningMeanStd surface: mean, var, count) as the device's running statistics."""
    import joblib
    from safepo.common.normalizer import SafeNormalizeObservation
    state = joblib.load(path)
    if not isinstance(state, dict) or "Normalizer" not in state:
        raise SpoError(f"{path}: missing key 'Normalizer'")
    rms = state["Normalizer"]
    for k in ("mean", "var"):
        v = getattr(rms, k, None)
        if v is None or np.shape(v) != (obs_dim,):
            raise SpoError(f"{path}: Normalizer.{k} has shape {None if v is None else np.shape(v)}, expected ({obs_dim},)")
    if not isinstance(getattr(rms, "count", None), (int, float, np.floating, np.integer)):
        raise SpoError(f"{path}: Normalizer.count is missing")
    norm = SafeNormalizeObservation(obs_dim, device)
    norm.obs_rms.load_state_dict({"mean": np.asarray(rms.mean), "var": np.asarray(rms.var), "count": rms.count})
    return norm


def _make_env(config, env_id):
    num_envs = int(config["num_envs"])
    if config.get("env", "mujoco") == "synthetic":
        from safepo.common.synthetic_env import make_synthetic_env
        return make_synthetic_env(num_envs, env_id, None, episode_len=int(config.get("episode_len", 1000)))
    from safepo.common.env import make_sa_mujoco_env
    return make_sa_mujoco_env(num_envs=num_envs, env_id=env_id, seed=None)


def eval_single_agent(eval_dir, eval_episodes):
    """evaluate.py:27-87: the run's last actor and Normalizer, ``eval_episodes`` deterministic episodes of the first env
    (``reward[0]`` / ``cost[0]``, the episode ends on ``terminated[0] or truncated[0]``); returns the mean reward and cost
    over the last 50 episodes."""
    from safepo.common.model import ActorVCritic
    if not torch.cuda.is_available():
        raise SpoError("evaluation runs the policy on a CUDA device (no CPU path)")
    device = torch.device("cuda", torch.cuda.current_device())
    config = _config(eval_dir)
    env_id = config["task"] if "task" in config else config["env_name"]
    norm_path = _last(eval_dir, ".pkl")
    model_path = _last(os.path.join(eval_dir, "torch_save"), ".pt")
    env, obs_space, act_space = _make_env(config, env_id)
    D = obs_space.shape[0]
    policy = ActorVCritic(D, act_space.shape[0], config["hidden_sizes"]).to(device)
    _load_actor(policy, model_path)
    wants = getattr(env, "device_wrappers", ())
    norm = None
    if config.get("normalize_obs", False) or "normalize_obs" in wants:
        norm = _load_normalizer(norm_path, D, device)
    rescale = None
    if "rescale_action" in wants:
        from safepo.common.normalizer import SafeRescaleAction
        rescale = SafeRescaleAction(env.action_space.low, env.action_space.high, device)

    def to_device(obs):
        o = torch.as_tensor(np.asarray(obs), dtype=torch.float32).reshape(-1, D).to(device)
        return o if norm is None else norm.normalize(o)

    rew_deque, cost_deque, len_deque = deque(maxlen=50), deque(maxlen=50), deque(maxlen=50)
    for _ in range(eval_episodes):
        eval_done = False
        obs, _ = env.reset()
        obs = to_device(obs)
        eval_rew, eval_cost, eval_len = 0.0, 0.0, 0.0
        while not eval_done:
            act, _, _, _ = policy.step(obs, deterministic=True)
            if rescale is not None:
                act = rescale.action(act)
            obs, reward, cost, terminated, truncated, _ = env.step(act.squeeze().cpu().numpy())
            obs = to_device(obs)
            eval_rew += reward[0]
            eval_cost += cost[0]
            eval_len += 1
            eval_done = bool(terminated[0] or truncated[0])
        rew_deque.append(eval_rew)
        cost_deque.append(eval_cost)
        len_deque.append(eval_len)
    env.close()
    return sum(rew_deque) / len(rew_deque), sum(cost_deque) / len(cost_deque)


def eval_multi_agent(eval_dir, eval_episodes):
    """evaluate.py:90-132: the run's algorithm's Runner, restored from ``models_seed{seed}``, evaluated by Runner.eval on the
    run's evaluation environments."""
    import importlib
    config = _config(eval_dir)
    algo = config.get("algorithm_name")
    if algo not in MULTI_AGENT_ALGOS:
        raise SpoError(f"{eval_dir}: algorithm_name {algo!r} is not one of {', '.join(MULTI_AGENT_ALGOS)}")
    mod = importlib.import_module(f"safepo.multi_agent.{algo}")
    from safepo.multi_agent.mappolag import evaluate_run
    model_dir = os.path.join(eval_dir, f"models_seed{config['seed']}")
    return evaluate_run(config, model_dir, eval_episodes, mod.Runner, mod.DEFAULT_CONFIG, algo, getattr(mod, "MAMUJOCO", None))


def single_runs_eval(eval_dir, eval_episodes):
    """evaluate.py:135-145: one run directory, single- or multi-agent."""
    if _config(eval_dir).get("algorithm_name") in MULTI_AGENT_ALGOS:
        return eval_multi_agent(eval_dir, eval_episodes)
    return eval_single_agent(eval_dir, eval_episodes)


def result_line(eval_episodes, algo, env, rewards, costs):
    """The line evaluate.py:179-184 appends to eval_result.txt (mean ± std over the seeds, two decimals)."""
    r_mean, r_std = round(np.mean(rewards), 2), round(np.std(rewards), 2)
    c_mean, c_std = round(np.mean(costs), 2), round(np.std(costs), 2)
    return (f"After {eval_episodes} episodes evaluation, the {algo} in {env} evaluation reward: {r_mean}±{r_std}, "
            f"cost: {c_mean}±{c_std} \n")


def benchmark_eval(argv=None):
    """evaluate.py:147-184: every <env>/<algo>/<seed-run> directory under --benchmark-dir."""
    parser = argparse.ArgumentParser()
    parser.add_argument("--benchmark-dir", type=str, default="", help="the directory of the evaluation")
    parser.add_argument("--eval-episodes", type=int, default=3, help="the number of episodes to evaluate")
    parser.add_argument("--save-dir", type=str, default=None, help="the directory to save the evaluation result")
    args = parser.parse_args(argv)
    benchmark_dir, eval_episodes = args.benchmark_dir, args.eval_episodes
    if args.save_dir is not None:
        save_dir = args.save_dir
    else:
        save_dir = benchmark_dir.replace("runs", "results")
        os.makedirs(save_dir, exist_ok=True)
    for env in sorted(os.listdir(benchmark_dir)):
        env_path = os.path.join(benchmark_dir, env)
        for algo in sorted(os.listdir(env_path)):
            print(f"Start evaluating {algo} in {env}")
            algo_path = os.path.join(env_path, algo)
            rewards, costs = [], []
            for seed in sorted(os.listdir(algo_path)):
                reward, cost = single_runs_eval(os.path.join(algo_path, seed), eval_episodes)
                rewards.append(reward)
                costs.append(cost)
            line = result_line(eval_episodes, algo, env, rewards, costs)
            print(line.rstrip() + f", the reuslt is saved in {save_dir}/eval_result.txt")
            with open(os.path.join(save_dir, "eval_result.txt"), "a") as f:
                f.write(line)


if __name__ == "__main__":
    benchmark_eval()
