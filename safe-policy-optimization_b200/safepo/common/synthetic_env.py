"""Synthetic vector environment of Safety-Gymnasium shape (no MuJoCo, no host cost).

``env.step`` stays on host cores in the real pipeline (safepo/common/env.py:58-69 in the
reference forks SafetyAsyncVectorEnv workers); Safety-Gymnasium is not installable
offline, and BASELINE.json defines the headline metric on *synthetic observations of the
task's shape*.  This class produces that stream with the same step/reset signature and
autoreset + ``final_observation`` convention the reference's rollout loop consumes
(ppo_lag.py:166-186), at ~zero cost per step: every quantity is read from a small
pre-generated pool of frames so that the trainer, not the generator, is what is timed.

Stream definition (SURVEY.md section 8d): obs ~ N(0,1) fp32, reward ~ 0.01*N(0,1),
cost ~ Bernoulli(0.05), time-limit truncation every ``episode_len`` steps (optionally
staggered per env), optional Bernoulli termination.
"""
from __future__ import annotations

import numpy as np
import torch

TASK_DIMS = {
    # obs_dim, act_dim of the tasks BASELINE.json names (upstream Safety-Gymnasium values)
    "SafetyPointGoal1-v0": (60, 2),
    "SafetyCarButton1-v0": (88, 2),
    "SafetyAntVelocity-v1": (27, 8),
    # Doggo (12 actuators; [64, 64] nets like every non-Isaac task, ppo_lag.py:46).  104 is the upstream Safety-Gymnasium
    # observation size of this task, not checked here (safety_gymnasium is not a dependency); the other seven Doggo
    # tasks are left out until their sizes can be cited.
    "SafetyDoggoGoal1-v0": (104, 12),
}


class _Box:
    def __init__(self, dim):
        self.shape = (dim,)


class _ObsRms:
    """Placeholder for the running normaliser the reference checkpoints (ppo_lag.py:381-386)."""

    def __init__(self, dim):
        self.mean, self.var, self.count = np.zeros(dim), np.ones(dim), 1e-4


class SyntheticVecEnv:
    def __init__(self, num_envs, obs_dim, act_dim, episode_len=1000, seed=0, pool=64,
                 stagger=False, p_terminate=0.0):
        rng = np.random.default_rng(seed)
        self.num_envs, self.obs_dim, self.act_dim = num_envs, obs_dim, act_dim
        self.episode_len = int(episode_len)
        self.observation_space = _Box(obs_dim)
        self.action_space = _Box(act_dim)
        self.single_observation_space = self.observation_space
        self.single_action_space = self.action_space
        self.obs_rms = _ObsRms(obs_dim)
        self._pool = pool
        self._obs = rng.standard_normal((pool, num_envs, obs_dim)).astype(np.float32)
        self._final = rng.standard_normal((pool, num_envs, obs_dim)).astype(np.float32)
        self._rew = (0.01 * rng.standard_normal((pool, num_envs))).astype(np.float64)
        self._cost = (rng.random((pool, num_envs)) < 0.05).astype(np.float64)
        self._term = rng.random((pool, num_envs)) < p_terminate
        self._phase = (rng.integers(0, self.episode_len, num_envs) if stagger
                       else np.zeros(num_envs, dtype=np.int64))
        self._age = self._phase.copy()
        self._k = 0

    def reset(self, seed=None):
        self._age = self._phase.copy()
        self._k = 0
        return self._obs[0].copy(), {}

    def step(self, action):
        self._k += 1
        k = self._k % self._pool
        self._age += 1
        terminated = self._term[k].copy()
        truncated = (self._age >= self.episode_len) & ~terminated
        done = terminated | truncated
        info = {}
        if done.any():
            fin = np.empty(self.num_envs, dtype=object)
            for i in np.nonzero(done)[0]:
                fin[i] = self._final[k, i]
            info["final_observation"] = fin
            info["_final_observation"] = done.copy()
            info["final_observation_dense"] = self._final[k]
            self._age[done] = 0
        return self._obs[k], self._rew[k], self._cost[k], terminated, truncated, info

    def close(self):
        pass


def make_synthetic_env(num_envs, env_id="SafetyPointGoal1-v0", seed=0, episode_len=1000, **kw):
    """Same return triple as make_sa_mujoco_env (safepo/common/env.py:35-80)."""
    obs_dim, act_dim = TASK_DIMS[env_id]
    env = SyntheticVecEnv(num_envs, obs_dim, act_dim, episode_len=episode_len,
                          seed=0 if seed is None else seed, **kw)
    return env, env.observation_space, env.action_space


class SyntheticMultiAgentEnv:
    """A synthetic multi-agent vector environment with the interface the reference's multi-agent Runner uses
    (safepo/multi_agent/mappolag.py:300-345: ``reset() -> obs, share_obs, _`` and ``step(actions) -> obs, share_obs, rewards,
    costs, dones, infos, _``), on the device: observations ~ N(0, 1), rewards ~ 0.01 N(0, 1), costs ~ Bernoulli(0.05) like the
    single-agent synthetic stream (SURVEY 8d), all agents of an environment finish together every ``episode_len`` steps.
    ``agent_done_prob`` > 0 (opt-in) also lets every agent finish alone with that probability per step, so that the active
    masks (an agent done while its environment goes on) occur; at 0 the stream draws exactly the numbers it always drew.
    ``obs_dim`` / ``act_dim`` may also give one size per agent.  Equal observation sizes keep the stacked [N, agents, D]
    observations and their draws; different ones come as one [N, D_i] tensor per agent, drawn agent by agent (the reference's
    Freight-Franka convention).  ``step`` checks every agent's actions against that agent's width."""

    def __init__(self, num_envs, num_agents, obs_dim, share_obs_dim, act_dim, episode_len, seed, device, agent_done_prob=0.0):
        self.num_envs, self.num_agents = int(num_envs), int(num_agents)
        self.obs_dims = _sizes(obs_dim, self.num_agents, "obs_dim")
        self.act_dims = _sizes(act_dim, self.num_agents, "act_dim")
        self.obs_dim = self.obs_dims[0] if len(set(self.obs_dims)) == 1 else None      # None: the per-agent list form
        self.act_dim = self.act_dims[0] if len(set(self.act_dims)) == 1 else None
        self.share_obs_dim = int(share_obs_dim)
        self.episode_len, self.device = int(episode_len), torch.device(device)
        self.agent_done_prob = float(agent_done_prob)
        self._g = torch.Generator(device=self.device).manual_seed(int(seed))
        self._t = 0

    def _obs(self):
        n, a = self.num_envs, self.num_agents
        if self.obs_dim is not None:
            obs = torch.randn(n, a, self.obs_dim, generator=self._g, device=self.device)
        else:
            obs = [torch.randn(n, d, generator=self._g, device=self.device) for d in self.obs_dims]
        return obs, torch.randn(n, a, self.share_obs_dim, generator=self._g, device=self.device)

    def reset(self):
        self._t = 0
        obs, share_obs = self._obs()
        return obs, share_obs, None

    def step(self, actions):
        if len(actions) != self.num_agents or any(x.shape != (self.num_envs, d) for x, d in zip(actions, self.act_dims)):
            raise ValueError("one [num_envs, act_dim] action tensor per agent expected")
        n, a = self.num_envs, self.num_agents
        self._t += 1
        obs, share_obs = self._obs()
        rewards = 0.01 * torch.randn(n, a, 1, generator=self._g, device=self.device)
        costs = (torch.rand(n, a, 1, generator=self._g, device=self.device) < 0.05).float()
        done = self._t % self.episode_len == 0
        dones = torch.full((n, a), bool(done), dtype=torch.bool, device=self.device)
        if self.agent_done_prob > 0.0:
            dones |= torch.rand(n, a, generator=self._g, device=self.device) < self.agent_done_prob
        return obs, share_obs, rewards, costs, dones, None, None


def _sizes(value, num_agents, what):
    if isinstance(value, (int, np.integer)):
        return [int(value)] * num_agents
    sizes = [int(v) for v in value]
    if len(sizes) != num_agents:
        raise ValueError(f"{what}: {len(sizes)} entries for {num_agents} agents")
    return sizes
