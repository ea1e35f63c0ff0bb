"""MAPPO-Lag on the device: the per-iteration part of the reference's ``Runner`` (safepo/multi_agent/mappolag.py:402-504,
583-597: ``collect`` / ``insert`` / ``compute`` / ``train``) around ``MultiAgentNets`` / ``MultiAgentTrainer``
(safepo/common/ma_model.py) and ``SeparatedReplayBuffer`` (safepo/common/buffer.py).  One runner holds all agents of one
GPU's environments; the environments themselves (Isaac Gym / multi-agent MuJoCo in the reference) are the caller's: it
feeds ``insert`` with what ``envs.step`` returned.  Random draws can be injected (``eps`` in ``collect``, ``agent_order`` and
``perms`` in ``train``) so that a run can be replayed against the oracle; by default they come from the device generator.
There is no CPU path."""
from __future__ import annotations

import argparse
import os
import time

import numpy as np
import torch

from safepo._lib import SpoError
from safepo.common.buffer import SeparatedReplayBuffer
from safepo.common.ma_model import MultiAgentNets, MultiAgentTrainer


def _per_agent(value, num_agents, what):
    """One int per agent from an int (every agent) or a sequence of ``num_agents`` entries."""
    if isinstance(value, (int, np.integer)):
        return [int(value)] * num_agents
    values = [int(v) for v in value]
    if len(values) != num_agents:
        raise SpoError(f"{what}: {len(values)} entries for {num_agents} agents")
    return values


def _check_agent(a, nets, obs_dim, share_obs_dim, act_dim):
    """Refuse agent ``a`` before any launch when its nets do not have its sizes or a size is outside the kernels' limits: even
    input widths (spo_ma_mlp_layer) and act_dim in 1..32.  (The hidden size, shared by the agents, is the layer kernels' to
    check.)"""
    if obs_dim < 2 or obs_dim % 2:
        raise SpoError(f"agent {a}: obs_dim={obs_dim} must be even and >= 2 (spo_ma_mlp_layer)")
    if share_obs_dim < 2 or share_obs_dim % 2:
        raise SpoError(f"agent {a}: share_obs_dim={share_obs_dim} must be even and >= 2 (spo_ma_mlp_layer)")
    if not 1 <= act_dim <= 32:
        raise SpoError(f"agent {a}: act_dim={act_dim} must be in 1..32")
    if nets.actor.D != obs_dim:
        raise SpoError(f"agent {a}: obs_dim={obs_dim}, but its actor takes {nets.actor.D} inputs")
    if nets.act_dim != act_dim:
        raise SpoError(f"agent {a}: act_dim={act_dim}, but its actor has {nets.act_dim} actions")
    for name, net in (("critic", nets.critic), ("cost_critic", nets.cost_critic)):
        if net is not None and net.D != share_obs_dim:
            raise SpoError(f"agent {a}: share_obs_dim={share_obs_dim}, but its {name} takes {net.D} inputs")


class Runner:
    trainer_class = MultiAgentTrainer
    cost_critic = True            # the agents' MultiAgentNets hold a cost critic; without it the runner skips the cost side

    def __init__(self, nets, config, obs_dim, share_obs_dim, act_dim, pad_actions_to=None):
        """``nets``: one MultiAgentNets per agent (all on the same device).  ``obs_dim`` / ``act_dim``: one int for every agent,
        or one entry per agent (the reference sizes agent i from ``envs.observation_space[i]`` / ``envs.action_space[i]``);
        ``share_obs_dim`` is one int, every agent's critic input.  ``pad_actions_to`` (opt-in): the width the environments take
        every agent's actions at; narrower actions are padded with zero columns for them and cut back to the agent's own width
        on ``insert`` (the reference's Safety9|8HumanoidVelocity-v0, whose agents have 9 and 8 actions).  Every agent is checked
        against its nets and the kernels' limits here, before anything runs on the device: SpoError naming the agent."""
        self.config, self.num_agents = dict(config), len(nets)
        self.nets = list(nets)
        self.device = nets[0].device
        self.obs_dims = _per_agent(obs_dim, self.num_agents, "obs_dim")
        self.act_dims = _per_agent(act_dim, self.num_agents, "act_dim")
        self.share_obs_dim = int(share_obs_dim)
        self.pad_actions_to = None if pad_actions_to is None else int(pad_actions_to)
        if self.pad_actions_to is not None and self.pad_actions_to < max(self.act_dims):
            raise SpoError(f"pad_actions_to={self.pad_actions_to} is narrower than the widest agent's act_dim {max(self.act_dims)}")
        for a, nets_a in enumerate(self.nets):
            _check_agent(a, nets_a, self.obs_dims[a], self.share_obs_dim, self.act_dims[a])
        self.trainer = [self.trainer_class(n, self.config) for n in self.nets]
        self.buffer = [SeparatedReplayBuffer(self.config, D, self.share_obs_dim, A, self.device) for D, A in zip(self.obs_dims, self.act_dims)]
        self.T, self.N = int(config["episode_length"]), int(config["n_rollout_threads"])
        self.iterations_done = 0

    def _dev(self, x):
        return torch.as_tensor(x).to(self.device)

    def _agent_obs(self, obs):
        """Every agent's observations [N, D_i] from either environment convention: a list with one tensor per agent (agents of
        different observation sizes; the reference's Freight-Franka branch reads ``obs[agent_id]``) or the stacked
        [N, agents, D] tensor (``obs[:, agent_id]``)."""
        if isinstance(obs, (list, tuple)):
            if len(obs) != self.num_agents:
                raise SpoError(f"{len(obs)} observation tensors for {self.num_agents} agents")
            return [self._dev(o) for o in obs]
        obs = self._dev(obs)
        return [obs[:, a] for a in range(self.num_agents)]

    def env_actions(self, actions):
        """The per-agent actions as the environments take them: the list itself, or with ``pad_actions_to`` every agent's
        actions padded with zero columns to that width (mappolag.py:428-430)."""
        W = self.pad_actions_to
        if W is None:
            return actions
        return [x if x.shape[-1] == W else torch.nn.functional.pad(x, (0, W - x.shape[-1])) for x in actions]

    def warmup(self, obs, share_obs):
        """obs [N, agents, D] or one [N, D_i] tensor per agent, share_obs [N, agents, DS] of the reset (mappolag.py:396-405)."""
        obs, share_obs = self._agent_obs(obs), self._dev(share_obs)
        for a, b in enumerate(self.buffer):
            b.share_obs[0].copy_(share_obs[:, a])
            b.obs[0].copy_(obs[a])

    @torch.no_grad()
    def collect(self, step, eps=None):
        """get_actions of every agent on its buffer's step-th observations (mappolag.py:408-445): values [N, agents, 1], the
        per-agent lists of actions / per-dimension log-probs, cost predictions [N, agents, 1] (None without a cost critic)."""
        values, actions, logps, cost_preds = [], [], [], []
        for a, nets in enumerate(self.nets):
            b = self.buffer[a]
            e = None if eps is None else self._dev(eps[a]).contiguous()
            v, act, lp, cp = nets.get_actions(b.share_obs[step], b.obs[step], eps=e)
            values.append(v), actions.append(act), logps.append(lp), cost_preds.append(cp)
        return torch.stack(values, dim=1), actions, logps, torch.stack(cost_preds, dim=1) if self.cost_critic else None

    @torch.no_grad()
    def insert(self, obs, share_obs, rewards, costs, dones, values, actions, action_log_probs, cost_preds=None):
        """One environment step into every agent's buffer (mappolag.py:447-487, mappo.py:377-406): an environment whose agents
        are all done gets mask 0 (and active mask 1); an agent done alone gets active mask 0.  Without a cost critic ``costs``
        and ``cost_preds`` are not stored.  ``obs`` in either convention of ``warmup``; actions wider than an agent's act_dim
        (padded for the environments) are cut back to it (mappolag.py:460-461)."""
        obs, share_obs, rewards = self._agent_obs(obs), self._dev(share_obs), self._dev(rewards)
        dones = self._dev(dones).bool()
        dones_env = torch.all(dones, dim=1)
        masks = torch.ones(self.N, self.num_agents, 1, device=self.device)
        masks[dones_env] = 0.0
        active_masks = torch.ones(self.N, self.num_agents, 1, device=self.device)
        active_masks[dones] = 0.0
        active_masks[dones_env] = 1.0
        if self.cost_critic:
            costs = self._dev(costs)
        for a, b in enumerate(self.buffer):
            cost = dict(costs=costs[:, a], cost_preds=cost_preds[:, a]) if self.cost_critic else {}
            act = actions[a]
            if act.shape[-1] != self.act_dims[a]:
                act = act[:, :self.act_dims[a]]
            b.insert(share_obs[:, a], obs[a], act, action_log_probs[a], values[:, a], rewards[:, a], masks[:, a], active_masks[:, a], **cost)

    @torch.no_grad()
    def compute(self):
        """Bootstrap values of the last observations and the masked GAE returns of both critics, or of the reward critic alone
        (mappolag.py:583-597, mappo.py:518-526)."""
        for nets, b, tr in zip(self.nets, self.buffer, self.trainer):
            mean, sd = tr.popart_mean_sqrt_var()
            b.compute_returns(nets.value(nets.critic, b.share_obs[-1]), mean, sd)
            if self.cost_critic:
                b.compute_cost_returns(nets.value(nets.cost_critic, b.share_obs[-1]), mean, sd)

    def train(self, agent_order=None, perms=None, collect_outputs=False):
        """Sequential update of the agents in a random order; every updated agent multiplies the importance ratio of its new
        against its old policy into the factor the following agents see (mappolag.py:489-519)."""
        T, N = self.T, self.N
        factor = torch.ones(T, N, 1, device=self.device)
        order = torch.randperm(self.num_agents).tolist() if agent_order is None else [int(a) for a in agent_order]
        outs = {}
        for a in order:
            b, tr, nets = self.buffer[a], self.trainer[a], self.nets[a]
            A = b.actions.shape[-1]
            b.update_factor(factor)
            flat_obs, flat_act = b.obs[:-1].reshape(-1, b.obs.shape[-1]), b.actions.reshape(-1, A)
            with torch.no_grad():
                old_lp = nets.evaluate_actions(flat_obs, flat_act)
            outs[a] = tr.train(b, perms=None if perms is None else perms[a])
            with torch.no_grad():
                new_lp = nets.evaluate_actions(flat_obs, flat_act)
                factor = factor * torch.prod(torch.exp(new_lp - old_lp).reshape(T, N, A), dim=-1, keepdim=True)
            b.after_update()
        return outs if collect_outputs else order

    def log_agent(self, a, out):
        """The logged values of agent a's last update (mappolag.py:228-234)."""
        value_loss, critic_norm, policy_loss, entropy, actor_norm, imp, cost_loss, cost_norm = out
        return {f"Loss/Loss_reward_critic/agent{a}": float(value_loss), f"Loss/Loss_cost_critic/agent{a}": float(cost_loss),
                f"Loss/Loss_actor/agent{a}": float(policy_loss), f"Misc/Entropy/agent{a}": float(entropy),
                f"Misc/Ratio/agent{a}": float(imp.mean()), f"Misc/Lagrange/agent{a}": float(self.trainer[a].lamda_lagr)}

    def return_aver_cost(self, aver_episode_costs):
        for b in self.buffer:
            b.return_aver_insert(aver_episode_costs)

    # ---- checkpoints and evaluation (mappolag.py:506-581; mappo.py, happo.py and macpo.py have the same three methods) ----
    def save(self, directory, train_state=False):
        """Runner.save: every agent's ``actor_agent{i}.pt`` / ``critic_agent{i}.pt`` in the reference's format (no cost critic,
        as in the reference).  ``train_state`` (an extension): also ``train_state_agent{i}.pt`` with what a resumed run needs to
        continue exactly -- the trainer's state (Adam moments and steps, PopArt, lamda_lagr), the cost critic's weights, the
        buffer's carried first step and average episode cost, and the number of iterations done.  The reference ignores it."""
        for a, nets in enumerate(self.nets):
            nets.save(directory, a)
            if train_state:
                st = dict(iterations_done=int(self.iterations_done), trainer=self.trainer[a].train_state(),
                          buffer=self.buffer[a].carried_state())
                if nets.cost_critic is not None:
                    st["cost_critic"] = nets.cost_critic.cpu_state_dict()
                torch.save(st, os.path.join(directory, f"train_state_agent{a}.pt"))

    def restore(self, directory, train_state=False):
        """Runner.restore: load every agent's actor and reward critic from ``directory`` in place.  The cost critic keeps its
        weights, as in the reference (which does not save it), unless ``train_state``: then ``train_state_agent{i}.pt``
        restores it together with the trainer's and the buffer's state and ``iterations_done``."""
        for a, nets in enumerate(self.nets):
            st = None
            if train_state:
                path = os.path.join(directory, f"train_state_agent{a}.pt")
                if not os.path.isfile(path):
                    raise SpoError(f"no training state {path}")
                st = torch.load(path, map_location="cpu", weights_only=True)
                if not isinstance(st, dict) or not isinstance(st.get("iterations_done"), int):
                    raise SpoError(f"{path}: not a training state")
                if nets.cost_critic is not None:
                    nets.cost_critic.check_state(st.get("cost_critic"), f"{path}: cost_critic")
            nets.load(directory, a)
            if st is not None:
                self.trainer[a].load_train_state(st.get("trainer"), path)
                self.buffer[a].load_carried_state(st.get("buffer"), path)
                if nets.cost_critic is not None:
                    nets.cost_critic.load_state(st["cost_critic"])
                self.iterations_done = st["iterations_done"]

    @torch.no_grad()
    def eval(self, envs, eval_episodes=1):
        """Runner.eval (mappolag.py:520-581): deterministic actions of every agent on ``envs`` (reset first), per-environment
        sums of the agents' mean reward / cost, the environments finished at a step taken in index order, until at least
        ``eval_episodes`` episodes have finished; returns the means (np.mean, float64) of the finished episodes' sums.  The sums
        stay on the device: each step reads back the number of finished environments, the finished sums are read back once at
        the end.  ``last_eval`` keeps that number and the per-episode sums."""
        obs, _, _ = envs.reset()
        ep_rew = ep_cost = None
        done_rew, done_cost, finished = [], [], 0
        while True:
            obs = self._agent_obs(obs)
            actions = [nets.act(obs[a].contiguous()) for a, nets in enumerate(self.nets)]
            obs, _, rewards, costs, dones, _, _ = envs.step(self.env_actions(actions))
            rew_env = torch.mean(self._dev(rewards), dim=1).flatten()
            cost_env = torch.mean(self._dev(costs), dim=1).flatten()
            if ep_rew is None:
                ep_rew, ep_cost = torch.zeros_like(rew_env), torch.zeros_like(cost_env)
            ep_rew += rew_env
            ep_cost += cost_env
            dones_env = torch.all(self._dev(dones).bool(), dim=1)
            k = int(dones_env.sum())
            if k:
                done_rew.append(ep_rew[dones_env])          # boolean indexing keeps the index order and copies
                done_cost.append(ep_cost[dones_env])
                ep_rew[dones_env] = 0
                ep_cost[dones_env] = 0
                finished += k
            if finished >= eval_episodes:
                rews, costs = torch.cat(done_rew).tolist(), torch.cat(done_cost).tolist()
                self.last_eval = dict(episodes=finished, rewards=rews, costs=costs)
                return np.mean(rews), np.mean(costs)

    def run(self, envs, iterations, logger=None, save_dir=None, eval_envs=None, save_train_state=False, first_iteration=0):
        """The training loop of the reference's Runner.run (mappolag.py:300-373) for ``iterations`` iterations of ``episode_length``
        steps: ``envs.reset() -> (obs [N, agents, D] or one [N, D_i] tensor per agent, share_obs [N, agents, DS], _)``,
        ``envs.step(actions) -> (obs, share_obs, rewards [N, agents, 1], costs [N, agents, 1], dones [N, agents], infos, _)`` with
        device tensors, ``actions`` one tensor per agent (padded to ``pad_actions_to`` when set); the per-environment
        episode sums live on the device, nothing is read back inside an iteration except the PopArt statistics in compute()/train()
        and the logged scalars at its end.  After each iteration, as in the reference: ``save(save_dir)`` (when given) every
        ``save_interval`` iterations and after the last one, ``eval(eval_envs)`` every ``eval_interval`` iterations when the
        config's ``use_eval`` is set; ``Eval/EpRet`` / ``Eval/EpCost`` are logged, 0.0 until the first evaluation.  Iterations
        are numbered from ``first_iteration`` (a resumed run continues its count).  Returns the list of per-iteration log rows."""
        c = self.config
        save_interval, eval_interval = int(c.get("save_interval", 1)), int(c.get("eval_interval", 25))
        use_eval = bool(c.get("use_eval", False))
        if use_eval and eval_envs is None:
            raise ValueError("use_eval needs eval_envs")
        obs, share_obs, _ = envs.reset()
        self.warmup(obs, share_obs)
        ep_rew = torch.zeros(self.N, device=self.device)
        ep_cost = torch.zeros(self.N, device=self.device)
        eval_rew, eval_cost = 0.0, 0.0
        rows, start = [], time.time()
        last = int(first_iteration) + int(iterations) - 1
        for it in range(int(first_iteration), last + 1):
            done_rew, done_cost = [], []
            for step in range(self.T):
                values, actions, logps, cost_preds = self.collect(step)
                actions = self.env_actions(actions)
                obs, share_obs, rewards, costs, dones, _infos, _ = envs.step(actions)
                dones_env = torch.all(self._dev(dones).bool(), dim=1)
                ep_rew += torch.mean(self._dev(rewards), dim=1).flatten()
                ep_cost += torch.mean(self._dev(costs), dim=1).flatten()
                done_rew.append(ep_rew[dones_env].clone())
                done_cost.append(ep_cost[dones_env].clone())
                ep_rew[dones_env] = 0
                ep_cost[dones_env] = 0
                self.insert(obs, share_obs, rewards, costs, dones, values, actions, logps, cost_preds)
            self.compute()
            outs = self.train(collect_outputs=True)
            row = {"Train/Epoch": it, "Train/TotalSteps": (it + 1) * self.T * self.N}
            finished_rew, finished_cost = torch.cat(done_rew), torch.cat(done_cost)
            if finished_rew.numel():
                row["Metrics/EpRet"] = float(finished_rew.mean())
                row["Metrics/EpCost"] = float(finished_cost.mean())
                self.return_aver_cost(finished_cost.mean())          # mappolag.py:349-351
            # the reference saves and evaluates just before return_aver_cost; neither touches the weights, and saving after
            # it puts this iteration's average episode cost into the training state
            self.iterations_done = it + 1
            if save_dir is not None and (it % save_interval == 0 or it == last):
                self.save(save_dir, train_state=save_train_state)
            if use_eval and it % eval_interval == 0:
                eval_rew, eval_cost = self.eval(eval_envs)
            row["Eval/EpRet"], row["Eval/EpCost"] = float(eval_rew), float(eval_cost)
            for a, out in outs.items():                              # the reference logs the last update of every agent's train()
                row.update(self.log_agent(a, out))
            row["Time/Total"] = time.time() - start
            row["Time/FPS"] = int(row["Train/TotalSteps"] / max(row["Time/Total"], 1e-9))
            rows.append(row)
            if logger is not None:
                for k, v in row.items():
                    logger.log_tabular(k, v)
                logger.dump_tabular()
        return rows


def init_state(in_dim, hidden_size, layer_N, head, act_dim=0, std_x_coef=1.0, actor_gain=0.01, generator=None):
    """Random weights of one MultiAgentActor / MultiAgentCritic in the reference's layout and initialisation (mlp.py:27-38: orthogonal
    with the ReLU gain, zero biases; distributions.py:21-36: fc_mean orthogonal with gain 0.01, log_std = std_x_coef; model.py:336-339:
    v_out orthogonal) -- there is no checkpoint to load offline."""
    import torch.nn as nn

    def ortho(rows, cols, gain):
        w = torch.empty(rows, cols)
        nn.init.orthogonal_(w, gain=gain, generator=generator)
        return w
    relu_gain = nn.init.calculate_gain("relu")
    st = {"base.feature_norm.weight": torch.ones(in_dim), "base.feature_norm.bias": torch.zeros(in_dim)}
    dims = [in_dim] + [hidden_size] * (1 + layer_N)
    for li, name in enumerate(["fc1"] + [f"fc2.{i}" for i in range(layer_N)]):
        st[f"base.mlp.{name}.0.weight"] = ortho(hidden_size, dims[li], relu_gain)
        st[f"base.mlp.{name}.0.bias"] = torch.zeros(hidden_size)
        st[f"base.mlp.{name}.2.weight"] = torch.ones(hidden_size)
        st[f"base.mlp.{name}.2.bias"] = torch.zeros(hidden_size)
    if head == "actor":
        st["act.action_out.log_std"] = torch.ones(act_dim) * std_x_coef
        st["act.action_out.fc_mean.weight"] = ortho(act_dim, hidden_size, actor_gain)
        st["act.action_out.fc_mean.bias"] = torch.zeros(act_dim)
    else:
        st["v_out.weight"] = ortho(1, hidden_size, 1.0)
        st["v_out.bias"] = torch.zeros(1)
    return st


# the yaml's values (safepo/multi_agent/marl_cfg/mappolag/config.yaml) that this path reads
DEFAULT_CONFIG = dict(episode_length=8, n_rollout_threads=1024, hidden_size=512, layer_N=2, gamma=0.96, gae_lambda=0.95, learning_iters=5,
                      num_mini_batch=1, actor_lr=9e-5, critic_lr=5e-3, opti_eps=1e-5, weight_decay=0.0, clip_param=0.2, huber_delta=10.0,
                      entropy_coef=0.0, max_grad_norm=10.0, cost_limit=25.0, lagrangian_coef_rate=1e-5, value_loss_coef=1.0, lamda_lagr=0.78,
                      std_x_coef=1.0, std_y_coef=0.5, actor_gain=0.01, use_policy_active_masks=False, use_value_active_masks=False,
                      save_interval=1, use_eval=False, eval_interval=25, n_eval_rollout_threads=1)
# the yaml's mamujoco section (the multi-agent MuJoCo tasks, 9|8 Humanoid among them); use_value_active_masks is read by
# nothing, as in the reference (cal_value_loss ignores the masks)
MAMUJOCO = dict(episode_length=1000, n_rollout_threads=10, n_eval_rollout_threads=10, hidden_size=128, gamma=0.99, entropy_coef=0.01,
                actor_lr=5e-4, critic_lr=5e-4, max_grad_norm=10.0, use_value_active_masks=True, use_policy_active_masks=True)


def main(argv=None):
    """`python -m safepo.multi_agent.mappolag --env synthetic [--mamujoco]`: MAPPO-Lag on a synthetic multi-agent stream of config
    5's shape (the reference's Isaac-Gym / multi-agent MuJoCo environments are not installable offline)."""
    return run_cli(argv, Runner, DEFAULT_CONFIG, "mappolag", mamujoco=MAMUJOCO)


def _int_list(text):
    return [int(x) for x in text.split(",")]


def _parser(algo, mamujoco):
    ap = argparse.ArgumentParser()
    ap.add_argument("--env", default="synthetic", choices=("synthetic",))
    ap.add_argument("--num-envs", type=int, default=1024)
    ap.add_argument("--num-agents", type=int, default=2)
    ap.add_argument("--obs-dim", type=int, default=398)
    ap.add_argument("--share-obs-dim", type=int, default=398)
    ap.add_argument("--act-dim", type=int, default=20)
    ap.add_argument("--obs-dims", type=_int_list, default=None, metavar="D0,D1,..",
                    help="one observation size per agent, for agents of different sizes (replaces --obs-dim)")
    ap.add_argument("--act-dims", type=_int_list, default=None, metavar="A0,A1,..",
                    help="one action size per agent, for agents of different sizes (replaces --act-dim)")
    ap.add_argument("--pad-actions-to", type=int, default=None, metavar="W",
                    help="hand the environments every agent's actions padded with zero columns to W (the reference's 9|8 Humanoid: 9)")
    ap.add_argument("--hidden-size", type=int, default=None)
    ap.add_argument("--iterations", type=int, default=10)
    ap.add_argument("--episode-len", type=int, default=64, help="steps after which the synthetic environments finish an episode")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--device", default="cuda:0")
    ap.add_argument("--log-dir", default=os.path.join("runs", "synthetic", algo, "seed0"))
    ap.add_argument("--agent-done-prob", type=float, default=0.0,
                    help="probability per step that an agent of the synthetic environments finishes alone (active masks)")
    if mamujoco is not None:
        ap.add_argument("--mamujoco", action="store_true", help="apply the yaml's mamujoco section (hidden size, gamma, entropy, masks)")
    ap.add_argument("--save-dir", default=None, help="where the runner saves actor_agent{i}.pt / critic_agent{i}.pt (default: "
                    "<log-dir>/models_seed<seed>, the reference's save_dir)")
    ap.add_argument("--save-interval", type=int, default=None, help="save every this many iterations (and after the last; yaml: 1)")
    ap.add_argument("--save-train-state", action="store_true", help="also save train_state_agent{i}.pt, which --resume needs")
    ap.add_argument("--model-dir", default=None, help="restore the actors and critics saved there and evaluate them instead of training")
    ap.add_argument("--resume", default=None, metavar="DIR", help="restore a run saved with --save-train-state and keep training")
    ap.add_argument("--use-eval", action="store_true", help="evaluate every --eval-interval iterations on separate environments")
    ap.add_argument("--eval-interval", type=int, default=None, help="iterations between evaluations (yaml: 25)")
    ap.add_argument("--eval-episodes", type=int, default=10, help="episodes --model-dir evaluates")
    ap.add_argument("--eval-num-envs", type=int, default=None, help="evaluation environments (yaml: n_eval_rollout_threads)")
    return ap


def run_cli(argv, runner_class, default_config, algo, mamujoco=None):
    """The synthetic-environment CLI shared by the multi-agent algorithms: builds the nets (with a cost critic when
    ``runner_class.cost_critic``), the runner and the environments.  ``mamujoco``: the yaml's ``mamujoco`` overrides, applied
    with ``--mamujoco`` (the flag exists only where they are given).  A training run writes its flags and configuration to
    ``<log-dir>/config.json`` (as the reference's Runner does), which is what safepo.evaluate rebuilds the run from."""
    from safepo.common.logger import EpochLogger
    from safepo.common.synthetic_env import SyntheticMultiAgentEnv
    ap = _parser(algo, mamujoco)
    args = ap.parse_args(argv)
    if args.model_dir is not None and args.resume is not None:
        ap.error("--model-dir evaluates, --resume trains: give one of them")
    for flag, dims in (("--obs-dims", args.obs_dims), ("--act-dims", args.act_dims)):
        if dims is not None and len(dims) != args.num_agents:
            ap.error(f"{flag} needs one entry per agent ({args.num_agents})")
    runner, cfg, env_obs, env_act, eval_envs = _setup(args, runner_class, default_config, mamujoco)
    if args.model_dir is not None:                                  # mappolag.py:634-637: restore, then evaluate only
        runner.restore(args.model_dir)
        ret, cost = runner.eval(eval_envs(), args.eval_episodes)
        row = {"Eval/EpRet": float(ret), "Eval/EpCost": float(cost), "Eval/Episodes": runner.last_eval["episodes"]}
        print(row)
        return [row]
    if args.resume is not None:
        runner.restore(args.resume, train_state=True)
    envs = SyntheticMultiAgentEnv(args.num_envs, args.num_agents, env_obs, args.share_obs_dim, env_act, args.episode_len, args.seed,
                                  runner.device, agent_done_prob=args.agent_done_prob)
    save_dir = args.save_dir if args.save_dir is not None else os.path.join(args.log_dir, f"models_seed{args.seed}")
    logger = EpochLogger(args.log_dir, seed=args.seed, use_tensorboard=False)
    logger.save_config(dict(vars(args), **cfg, algorithm_name=algo, env_name="synthetic"))
    rows = runner.run(envs, args.iterations, logger=logger, save_dir=save_dir, eval_envs=eval_envs() if args.use_eval else None,
                      save_train_state=args.save_train_state, first_iteration=runner.iterations_done)
    logger.close()
    return rows


def evaluate_run(config, model_dir, eval_episodes, runner_class, default_config, algo, mamujoco=None):
    """Restore the run that ``config`` (its config.json) describes from ``model_dir`` and evaluate it like ``--model-dir``:
    returns Runner.eval's (reward, cost) means over ``eval_episodes`` episodes."""
    ap = _parser(algo, mamujoco)
    args = ap.parse_args([])
    for key in vars(args):
        if key in config:
            setattr(args, key, config[key])
    runner, _, _, _, eval_envs = _setup(args, runner_class, default_config, mamujoco)
    runner.restore(model_dir)
    return runner.eval(eval_envs(), eval_episodes)


def _setup(args, runner_class, default_config, mamujoco):
    """The nets, the runner and the evaluation environments' factory of the parsed flags ``args``."""
    from safepo.common.synthetic_env import SyntheticMultiAgentEnv
    obs_dims = args.obs_dims if args.obs_dims is not None else [args.obs_dim] * args.num_agents
    act_dims = args.act_dims if args.act_dims is not None else [args.act_dim] * args.num_agents
    # the synthetic environments take every agent's actions at the padded width when there is one
    env_obs = args.obs_dim if args.obs_dims is None else obs_dims
    env_act = args.pad_actions_to if args.pad_actions_to is not None else (args.act_dim if args.act_dims is None else act_dims)
    cfg = dict(default_config)
    if mamujoco is not None and args.mamujoco:
        cfg.update(mamujoco)
    # the CLI's sizes win over the yaml's (--hidden-size defaults to the yaml's value of the chosen section)
    hidden = args.hidden_size if args.hidden_size is not None else cfg["hidden_size"]
    cfg.update(n_rollout_threads=args.num_envs, hidden_size=hidden)
    for key, value in (("save_interval", args.save_interval), ("eval_interval", args.eval_interval),
                       ("n_eval_rollout_threads", args.eval_num_envs)):
        if value is not None:
            cfg[key] = value
    cfg["use_eval"] = bool(args.use_eval)
    g = torch.Generator().manual_seed(args.seed)
    nets = []
    for D, A in zip(obs_dims, act_dims):
        nets.append(MultiAgentNets(init_state(D, cfg["hidden_size"], cfg["layer_N"], "actor", A, cfg["std_x_coef"], cfg["actor_gain"], g),
                                   init_state(args.share_obs_dim, cfg["hidden_size"], cfg["layer_N"], "critic", generator=g),
                                   init_state(args.share_obs_dim, cfg["hidden_size"], cfg["layer_N"], "critic", generator=g)
                                   if runner_class.cost_critic else None,
                                   args.device, layer_N=cfg["layer_N"], std_x_coef=cfg["std_x_coef"], std_y_coef=cfg["std_y_coef"]))
    runner = runner_class(nets, cfg, obs_dims, args.share_obs_dim, act_dims, pad_actions_to=args.pad_actions_to)

    def eval_envs():
        # the reference's evaluation environments: n_eval_rollout_threads of them, seeded seed + 10000 (mappolag.py:609-617)
        return SyntheticMultiAgentEnv(int(cfg.get("n_eval_rollout_threads", 1)), args.num_agents, env_obs, args.share_obs_dim,
                                      env_act, args.episode_len, args.seed + 10000, runner.device, agent_done_prob=args.agent_done_prob)
    return runner, cfg, env_obs, env_act, eval_envs


__all__ = ["Runner", "MultiAgentNets", "MultiAgentTrainer", "SeparatedReplayBuffer", "init_state", "DEFAULT_CONFIG", "MAMUJOCO", "main"]


if __name__ == "__main__":
    main()
