"""TEST INFRASTRUCTURE ONLY: the multi-agent Runner's save / restore / eval (safepo/multi_agent/mappolag.py:506-581 of the
reference; mappo.py, happo.py and macpo.py have the same three methods) restated on the oracle runner
(oracle/ma_oracle.py: OracleMARunner), and the deterministic stand-in environment that tests/golden/make_ma_ckpt_golden.py
drives the reference's own methods with.  Pinned bit for bit by tests/golden/ma_ckpt.pt (tests/test_ma_checkpoint.py)."""
import os

import numpy as np
import torch

from oracle import ma_oracle as MA


class StubMAEnv:
    """A deterministic multi-agent vector environment with the reference Runner's interface (``reset() -> obs, share_obs, _``,
    ``step(actions) -> obs, share_obs, rewards, costs, dones, infos, _``).  Every draw comes from a CPU generator re-seeded by
    reset(), so two evaluations see the same stream.  Environment i finishes every ``periods[i]`` steps (all its agents done);
    ``alone`` = (env, agent, step) lets one agent finish alone at that step of every episode (the environment goes on).  The
    rewards and costs depend smoothly on the actions, so an evaluation checks the policy, while the finishing schedule does not."""

    def __init__(self, num_agents, obs_dim, share_obs_dim, periods, seed, alone=(0, 1, 2), device="cpu"):
        self.num_envs, self.num_agents = len(periods), int(num_agents)
        self.obs_dim, self.share_obs_dim = int(obs_dim), int(share_obs_dim)
        self.periods, self.seed, self.alone, self.device = [int(p) for p in periods], int(seed), alone, torch.device(device)
        self.reset()

    def _obs(self):
        n, a = self.num_envs, self.num_agents
        obs = torch.randn(n, a, self.obs_dim, generator=self._g) * 2 + 0.3
        share = torch.randn(n, a, self.share_obs_dim, generator=self._g) * 3
        return obs.to(self.device), share.to(self.device)

    def reset(self):
        self._g = torch.Generator().manual_seed(self.seed)
        self._age = [0] * self.num_envs
        obs, share = self._obs()
        return obs, share, None

    def step(self, actions):
        n, a = self.num_envs, self.num_agents
        obs, share = self._obs()
        base_r = (0.1 * torch.randn(n, a, 1, generator=self._g)).to(self.device)
        base_c = (torch.rand(n, a, 1, generator=self._g) < 0.3).float().to(self.device)
        act = torch.stack([x.to(self.device) for x in actions], dim=1)                       # [n, agents, A]
        rewards = base_r - 0.5 * (act ** 2).mean(-1, keepdim=True)
        costs = base_c + 0.1 * act.abs().mean(-1, keepdim=True)
        dones = torch.zeros(n, a, dtype=torch.bool)
        for i in range(n):
            self._age[i] += 1
            if self._age[i] == self.periods[i]:
                dones[i] = True
                self._age[i] = 0
        e, ag, s = self.alone
        if self._age[e] == s:
            dones[e, ag] = True
        return obs, share, rewards, costs, dones.to(self.device), None, None


class OracleMACkptRunner(MA.OracleMARunner):
    """OracleMARunner with the reference Runner's save / restore / eval.  ``last_eval`` keeps the finished-episode count and the
    per-episode sums of the last eval()."""

    def save(self, directory):
        """Runner.save (mappolag.py:506-511): the actor and the reward critic of every agent, no cost critic."""
        os.makedirs(directory, exist_ok=True)
        for a, (actor, critic, _) in enumerate(self.nets):
            torch.save(actor.state(), os.path.join(directory, f"actor_agent{a}.pt"))
            torch.save(critic.state(), os.path.join(directory, f"critic_agent{a}.pt"))

    def restore(self, directory):
        """Runner.restore (mappolag.py:513-518): load_state_dict (strict) of the actor and the reward critic."""
        for a, (actor, critic, _) in enumerate(self.nets):
            for net, name in ((actor, "actor"), (critic, "critic")):
                st = torch.load(os.path.join(directory, f"{name}_agent{a}.pt"))
                assert set(st) == set(net.p), (name, a)
                with torch.no_grad():
                    for k, v in st.items():
                        net.p[k].copy_(v)

    @torch.no_grad()
    def eval(self, envs, eval_episodes=1):
        """Runner.eval (mappolag.py:520-581) without the recurrent states (MLP policies): deterministic actions, per-environment
        sums of the agents' mean reward / cost, finished environments in index order, np.mean of the finished sums."""
        eval_episode = 0
        eval_episode_rewards, eval_episode_costs = [], []
        eval_obs, _, _ = envs.reset()
        n = eval_obs.shape[0]
        one_episode_rewards, one_episode_costs = torch.zeros(1, n), torch.zeros(1, n)
        while True:
            eval_actions_collector = [MA.ma_actor_dist(actor, eval_obs[:, a], self.cfg["std_x_coef"], self.cfg["std_y_coef"]).mean
                                      for a, (actor, _, _) in enumerate(self.nets)]
            eval_obs, _, eval_rewards, eval_costs, eval_dones, _, _ = envs.step(eval_actions_collector)
            reward_env = torch.mean(eval_rewards, dim=1).flatten()
            cost_env = torch.mean(eval_costs, dim=1).flatten()
            one_episode_rewards += reward_env
            one_episode_costs += cost_env
            eval_dones_env = torch.all(eval_dones, dim=1)
            for eval_i in range(n):
                if eval_dones_env[eval_i]:
                    eval_episode += 1
                    eval_episode_rewards.append(one_episode_rewards[:, eval_i].mean().item())
                    one_episode_rewards[:, eval_i] = 0
                    eval_episode_costs.append(one_episode_costs[:, eval_i].mean().item())
                    one_episode_costs[:, eval_i] = 0
            if eval_episode >= eval_episodes:
                self.last_eval = dict(episodes=eval_episode, rewards=eval_episode_rewards, costs=eval_episode_costs)
                return np.mean(eval_episode_rewards), np.mean(eval_episode_costs)
