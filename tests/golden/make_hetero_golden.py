"""Generate tests/golden/hetero.pt from the REAL reference's multi-agent runners for agents of different sizes
(safepo/multi_agent/mappolag.py, happo.py).

Runs only where the reference is checked out (make_golden.REF, read-only); it reuses make_golden.py's import of the reference
(environment packages stubbed) and writes hetero.pt and nothing else, so the other fixtures stay byte-identical.  The Runner's
own collect / insert / compute / train are called on a stand-in ``self`` carrying the real policies, trainers and buffers (its
constructor needs environments that are not installable here), for two cases the reference names by task:

* ``humanoid``: env_name "Safety9|8HumanoidVelocity-v0", agents of 9 and 8 actions and equal observations -- collect pads the
  last agent's actions with a zero column for the environment, insert cuts them back (mappolag.py:428-430, 460-461);
* ``franka``: an env_name containing "Frank", observations of 10 and 14 as one tensor per agent, 4 and 3 actions
  (mappolag.py:462-465).

Each case runs MAPPO-Lag with the yaml's mamujoco section (both active-mask flags on; every agent finishes with its
environment, since MAPPO-Lag's NaN standardisation leaves nothing to compare once one finishes alone) and HAPPO with the mask
flags on and an agent finishing alone.  Also stored: two consecutive MAPPO_L_Trainer.ppo_update calls with the policy masks on
and a quarter of the rows inactive.  The initial weights are tests/hetero_oracle.py's ``initial_states`` of a recorded seed,
loaded into the reference's policies; the inputs are stored as tensors and every output of the reference as a bit-exact
``digest`` fingerprint, which keeps the file small.

    python tests/golden/make_hetero_golden.py [OUT]        # default: tests/golden/hetero.pt
"""
from __future__ import annotations

import importlib
import os
import sys
import types

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
for _p in (HERE, os.path.dirname(HERE), os.path.dirname(os.path.dirname(HERE))):     # make_golden, hetero_oracle, oracle
    sys.path.insert(0, _p)
import hetero_oracle as HO  # noqa: E402
import make_golden as MG  # noqa: E402

T, N, DS, H, NA = 4, 6, 14, 32, 2
CASES = {"humanoid": dict(env_name="Safety9|8HumanoidVelocity-v0", obs=(10, 10), act=(9, 8), pad=9, obs_list=False),
         "franka": dict(env_name="FreightFrankaCloseDrawer", obs=(10, 14), act=(4, 3), pad=None, obs_list=True)}
ALGOS = {"mappolag": ("MAPPO_L_Policy", "MAPPO_L_Trainer"), "happo": ("HAPPO_Policy", "HAPPO_Trainer")}
# mappolag: its yaml's mamujoco section without the sizes; happo: the mask flags and the entropy of MAPPO's mamujoco section
FLAGS = {"mappolag": dict(gamma=0.99, entropy_coef=0.01, actor_lr=5e-4, critic_lr=5e-4, max_grad_norm=10.0, use_value_active_masks=True,
                          use_policy_active_masks=True),
         "happo": dict(use_policy_active_masks=True, use_value_active_masks=True, entropy_coef=0.01)}
KEEP = ("actor_lr", "critic_lr", "opti_eps", "weight_decay", "clip_param", "huber_delta", "entropy_coef", "max_grad_norm", "gamma",
        "gae_lambda", "value_loss_coef", "layer_N", "std_x_coef", "std_y_coef", "learning_iters", "use_policy_active_masks",
        "use_value_active_masks", "cost_limit", "lagrangian_coef_rate", "lamda_lagr", "episode_length", "n_rollout_threads")


class Sp:
    def __init__(self, d):
        self.shape = (d,)


class Log:
    def store(self, **kw):
        pass


def _config(algo, **changes):
    import yaml
    cfg = yaml.safe_load(open(os.path.join(MG.REF, "safepo", "multi_agent", "marl_cfg", algo, "config.yaml")))
    cfg.update(device="cpu", algorithm_name=algo, **changes)
    return cfg


def _nets(algo):
    return ("actor", "critic", "cost_critic") if algo == "mappolag" else ("actor", "critic")


def _load(policy, init, algo):
    """Load the initial state dicts into the reference's policies (strict: the keys and shapes must be the reference's)."""
    for pol, sts in zip(policy, init):
        for n, st in zip(_nets(algo), sts):
            getattr(pol, n).load_state_dict(st)


def _states(pol, algo):
    return {n: {k: v.clone() for k, v in getattr(pol, n).state_dict().items()} for n in _nets(algo)}


def _obs(g, case):
    """One step's observations in the case's convention: stacked [N, agents, D] or one [N, D_i] tensor per agent."""
    if case["obs_list"]:
        return [torch.randn(N, d, generator=g) * 2 + 0.5 for d in case["obs"]]
    return torch.randn(N, NA, case["obs"][0], generator=g) * 2 + 0.5


def _clone(x):
    return [t.clone() for t in x] if isinstance(x, list) else x.clone()


def gen_run(algo, case_name, seed):
    """Two iterations of two agents through the reference Runner's own methods: T = 4 steps, 6 environments, hidden 32,
    learning_iters 2.  Every agent of environment 1 finishes at step 2; for HAPPO agent 1 of environment 0 also finishes alone
    at step 1.  Stored: the seed of the initial state dicts, the stream (the actions as collect hands them to the environment), the
    global-RNG seed, the buffers after compute() and after train() the factor, lamda_lagr, the PopArt state and the weights
    (every output as a fingerprint)."""
    case = CASES[case_name]
    m = importlib.import_module(f"safepo.multi_agent.{algo}")
    pcls, tcls = ALGOS[algo]
    cfg = _config(algo, env_name=case["env_name"], n_rollout_threads=N, hidden_size=H, episode_length=T, learning_iters=2, **FLAGS[algo])
    lag = algo == "mappolag"
    torch.manual_seed(seed)
    policy = [getattr(m, pcls)(cfg, Sp(D), Sp(DS), Sp(A)) for D, A in zip(case["obs"], case["act"])]
    _load(policy, HO.initial_states(seed, case["obs"], DS, case["act"], H, cfg["layer_N"], lag), algo)
    fake = types.SimpleNamespace(config=cfg, num_agents=NA, logger=Log(), policy=policy,
                                 trainer=[getattr(m, tcls)(cfg, pol) for pol in policy],
                                 buffer=[m.SeparatedReplayBuffer(cfg, Sp(D), Sp(DS), Sp(A)) for D, A in zip(case["obs"], case["act"])])
    g = torch.Generator().manual_seed(seed + 1)
    obs0, share0 = _obs(g, case), torch.randn(N, NA, DS, generator=g) * 3
    for a in range(NA):                                    # Runner.warmup, in the case's observation convention
        fake.buffer[a].share_obs[0].copy_(share0[:, a])
        fake.buffer[a].obs[0].copy_(obs0[a] if case["obs_list"] else obs0[:, a])
    stream, iters = [], []
    torch.manual_seed(seed + 2)
    train_episode_costs = torch.zeros(1, N)
    for it in range(2):
        steps = []
        for step in range(T):
            if lag:
                values, actions, logps, rnn_states, rnn_states_critic, cost_preds, rnn_states_cost = m.Runner.collect(fake, step)
            else:
                values, actions, logps, rnn_states, rnn_states_critic = m.Runner.collect(fake, step)
            env_actions = [x.clone() for x in actions]     # insert cuts the padded agent's actions back in the list itself
            obs, share_obs = _obs(g, case), torch.randn(N, NA, DS, generator=g) * 3
            rewards, costs = torch.randn(N, NA, 1, generator=g), (torch.rand(N, NA, 1, generator=g) < 0.3).float()
            dones = torch.zeros(N, NA, dtype=torch.bool)
            if step == 2:
                dones[1, :] = True
            if step == 1 and not lag:
                dones[0, 1] = True
            if lag:
                train_episode_costs += torch.mean(costs, dim=1).flatten()
                train_episode_costs[:, torch.all(dones, dim=1)] = 0
                m.Runner.insert(fake, (obs, share_obs, rewards, costs, dones, None, values, actions, logps, rnn_states, rnn_states_critic,
                                       cost_preds, rnn_states_cost, train_episode_costs.mean()))
            else:
                m.Runner.insert(fake, (obs, share_obs, rewards, dones, None, values, actions, logps, rnn_states, rnn_states_critic))
            st = dict(obs=_clone(obs), share_obs=share_obs, rewards=rewards, costs=costs, dones=dones, values=HO.digest(values),
                      actions=HO.digests(env_actions), action_log_probs=HO.digests(logps))
            if lag:
                st["cost_preds"] = HO.digest(cost_preds)
            steps.append(st)
        m.Runner.compute(fake)
        keys = ("returns", "value_preds", "masks", "active_masks", "obs", "actions") + (("cost_returns", "cost_preds") if lag else ())
        after_compute = [{k: HO.digest(getattr(b, k)) for k in keys} for b in fake.buffer]
        m.Runner.train(fake)
        res = []
        for a in range(NA):
            tr, vn = fake.trainer[a], fake.trainer[a].value_normalizer
            r = dict(factor=fake.buffer[a].factor, popart=[x.reshape(-1) for x in (vn.running_mean, vn.running_mean_sq, vn.debiasing_term)],
                     state=_states(policy[a], algo))
            if lag:
                r["lamda_lagr"] = torch.as_tensor(tr.lamda_lagr).reshape(-1)
            res.append(HO.digests(r))
        stream.append(steps)
        iters.append(dict(after_compute=after_compute, agents=res))
        if it == 0 and lag:                                  # Runner.return_aver_cost after an iteration with finished episodes
            for a in range(NA):
                fake.buffer[a].return_aver_insert(torch.tensor(31.5))
    return dict(cfg={k: cfg[k] for k in KEEP if k in cfg}, env_name=case["env_name"], obs_dims=case["obs"], act_dims=case["act"],
                pad=case["pad"], dims=(T, N, DS, H, NA), init_seed=seed, obs0=obs0, share_obs0=share0, seed=seed + 2, stream=stream,
                iters=iters, aver_cost_after_first=31.5 if lag else None)


def gen_masked_update(out):
    """Two consecutive MAPPO_L_Trainer.ppo_update calls with the mamujoco flags (policy masks on, entropy 0.01): obs 10, share_obs
    14, act 3, hidden 32, 48 rows of which about a quarter inactive, ratios spread over both sides of the clip range."""
    m = importlib.import_module("safepo.multi_agent.mappolag")
    D, A, R = 10, 3, 48
    cfg = _config("mappolag", env_name="synthetic", n_rollout_threads=4, hidden_size=H, **FLAGS["mappolag"])
    torch.manual_seed(51)
    pol = m.MAPPO_L_Policy(cfg, Sp(D), Sp(DS), Sp(A))
    _load([pol], HO.initial_states(51, [D], DS, [A], H, cfg["layer_N"], True), "mappolag")
    tr = m.MAPPO_L_Trainer(cfg, pol)
    g = torch.Generator().manual_seed(52)
    obs, share = torch.randn(R, D, generator=g) * 2 + 0.5, torch.randn(R, DS, generator=g) * 3
    import numpy as np
    rnn, masks = np.zeros((R, 1, H), dtype=np.float32), np.ones((R, 1), dtype=np.float32)
    with torch.no_grad():
        mu = pol.actor(obs, rnn, masks, deterministic=True)[0]
        std = torch.sigmoid(pol.actor.state_dict()["act.action_out.log_std"] / cfg["std_x_coef"]) * cfg["std_y_coef"]
        actions = mu + std * torch.randn(R, A, generator=g)
        logp = pol.actor.evaluate_actions(obs, rnn, actions, masks, None, None)[0]
    sample = dict(share_obs=share, obs=obs, actions=actions, value_preds=0.1 * torch.randn(R, 1, generator=g),
                  returns=torch.randn(R, 1, generator=g) * 4 + 1, old_action_log_probs=logp + 0.3 * torch.randn(R, A, generator=g),
                  adv_targ=torch.randn(R, 1, generator=g), factor=torch.rand(R, 1, generator=g) + 0.5,
                  active_masks=(torch.rand(R, 1, generator=g) >= 0.25).float(), cost_preds=0.1 * torch.randn(R, 1, generator=g),
                  cost_returns=torch.randn(R, 1, generator=g) * 2, cost_adv_targ=torch.randn(R, 1, generator=g),
                  aver_episode_costs=torch.tensor(30.0))
    calls = []
    names = ("value_loss", "critic_grad_norm", "policy_loss", "dist_entropy", "actor_grad_norm", "imp_weights", "cost_loss", "cost_grad_norm")
    for _ in range(2):
        s = sample
        tup = (s["share_obs"].numpy(), s["obs"].numpy(), rnn, rnn, s["actions"].numpy(), s["value_preds"], s["returns"], masks, s["active_masks"],
               s["old_action_log_probs"], s["adv_targ"], None, s["factor"], s["cost_preds"], s["cost_returns"], rnn, s["cost_adv_targ"],
               s["aver_episode_costs"])
        r = tr.ppo_update(tup)
        vn = tr.value_normalizer
        calls.append(HO.digests(dict(out={k: torch.as_tensor(v).detach() for k, v in zip(names, r)}, lamda_lagr=torch.as_tensor(tr.lamda_lagr).reshape(-1),
                                     popart=[x.reshape(-1) for x in (vn.running_mean, vn.running_mean_sq, vn.debiasing_term)],
                                     state=_states(pol, "mappolag"))))
    out["masked_update"] = dict(cfg={k: cfg[k] for k in KEEP if k in cfg}, dims=(D, DS, A, H, R), init_seed=51, sample=sample, calls=calls)


def main():
    path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "hetero.pt")
    sys.path.insert(0, MG.ROOT)
    MG.import_reference()
    threads = torch.get_num_threads()
    torch.set_num_threads(1)       # LayerNorm's backward reductions depend on the intra-op thread count (see make_golden.gen_ma_update)
    out = {"runs": {}}
    for i, algo in enumerate(ALGOS):
        for j, case in enumerate(CASES):
            out["runs"][(algo, case)] = gen_run(algo, case, 100 + 10 * (2 * i + j))
    gen_masked_update(out)
    torch.set_num_threads(threads)
    torch.save(out, path)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
