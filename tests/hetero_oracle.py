"""TEST INFRASTRUCTURE ONLY: the oracle runners of oracle/ma_oracle.py (MAPPO-Lag) and oracle/ppo_oracle.py (MAPPO / HAPPO) for
agents of different observation and action sizes, and MAPPO-Lag's ppo_update with use_policy_active_masks.

Restates the reference's per-agent handling in its runners (safepo/multi_agent/mappolag.py:277-297: agent i built from
``observation_space[i]`` / ``action_space[i]``; :428-430 and :460-461: the 9|8 Humanoid's actions padded with a zero column for
the environment in collect and cut back in insert; :462-465: the Freight-Franka observations as one tensor per agent; mappo.py,
happo.py and macpo.py do the same) and MAPPO_L_Trainer.ppo_update's masked surrogate and entropy (mappolag.py:146-170,
act.py:69-72), with the reference's torch ops in its order.  Pinned bit for bit by tests/golden/hetero.pt
(tests/golden/make_hetero_golden.py) through tests/test_ma_hetero.py.  The fixture keeps its inputs as tensors and the
reference's outputs as ``digest`` fingerprints, and its initial weights are ``random_state`` of recorded seeds, which keeps it
small; a fingerprint matches only a bit-identical tensor."""
import hashlib

import torch

from oracle import ma_oracle as MA
from oracle import ppo_oracle as PO


def random_state(g, din, H, A, head, layer_N):
    """A MultiAgentActor / MultiAgentCritic state dict with non-trivial LayerNorm parameters and biases."""
    st = {"base.feature_norm.weight": 1 + 0.1 * torch.randn(din, generator=g), "base.feature_norm.bias": 0.1 * torch.randn(din, generator=g)}
    for li, name in enumerate(["fc1"] + [f"fc2.{i}" for i in range(layer_N)]):
        k = din if li == 0 else H
        st[f"base.mlp.{name}.0.weight"] = torch.randn(H, k, generator=g) * (1.4 / k ** 0.5)
        st[f"base.mlp.{name}.0.bias"] = 0.1 * torch.randn(H, generator=g)
        st[f"base.mlp.{name}.2.weight"] = 1 + 0.1 * torch.randn(H, generator=g)
        st[f"base.mlp.{name}.2.bias"] = 0.1 * torch.randn(H, generator=g)
    if head == "actor":
        st["act.action_out.log_std"] = torch.ones(A) + 0.3 * torch.randn(A, generator=g)
        st["act.action_out.fc_mean.weight"] = torch.randn(A, H, generator=g) * 0.05
        st["act.action_out.fc_mean.bias"] = 0.1 * torch.randn(A, generator=g)
    else:
        st["v_out.weight"] = torch.randn(1, H, generator=g) * 0.1
        st["v_out.bias"] = 0.1 * torch.randn(1, generator=g)
    return st



def initial_states(seed, obs_dims, share_obs_dim, act_dims, H, layer_N, cost_critic):
    """The initial weights of the fixture's agents: per agent (actor, critic[, cost_critic]) ``random_state`` dicts drawn in
    that order from one generator seeded ``seed``."""
    g = torch.Generator().manual_seed(seed)
    return [[random_state(g, D, H, A, "actor", layer_N)] + [random_state(g, share_obs_dim, H, 0, "critic", layer_N)
                                                            for _ in range(2 if cost_critic else 1)]
            for D, A in zip(obs_dims, act_dims)]


def digest(t):
    """A bit-exact fingerprint of a tensor: its dtype, its shape and the SHA-256 of its bytes."""
    t = torch.as_tensor(t).detach().contiguous().cpu()
    return str(t.dtype), tuple(t.shape), hashlib.sha256(t.numpy().tobytes()).hexdigest()


def digests(obj):
    """``digest`` of every tensor in nested dicts / lists / tuples."""
    if torch.is_tensor(obj):
        return digest(obj)
    if isinstance(obj, dict):
        return {k: digests(v) for k, v in obj.items()}
    if isinstance(obj, (list, tuple)):
        return type(obj)(digests(v) for v in obj)
    return obj


class OracleMaskedMATrainer(MA.OracleMATrainer):
    """OracleMATrainer with use_policy_active_masks honoured: the surrogate rows weighted m_r / sum m, the entropy
    (entropy [n, A] * m).sum() / m.sum().  The Lagrange step and both value losses ignore the masks, as in the reference."""

    def ppo_update(self, s):
        c = self.cfg
        if not c.get("use_policy_active_masks"):
            return super().ppo_update(s)
        am = s["active_masks"]
        dist = MA.ma_actor_dist(self.actor, s["obs"])
        action_log_probs = dist.log_prob(s["actions"])
        dist_entropy = (dist.entropy() * am).sum() / am.sum()
        values = MA.ma_critic_value(self.critic, s["share_obs"])
        cost_values = MA.ma_critic_value(self.cost_critic, s["share_obs"])
        adv_targ_hybrid = s["adv_targ"] - self.lamda_lagr * s["cost_adv_targ"]
        imp_weights = torch.prod(torch.exp(action_log_probs - s["old_action_log_probs"]), dim=-1, keepdim=True)
        surr1 = imp_weights * adv_targ_hybrid
        surr2 = torch.clamp(imp_weights, 1.0 - c["clip_param"], 1.0 + c["clip_param"]) * adv_targ_hybrid
        policy_loss = (-torch.sum(s["factor"] * torch.min(surr1, surr2), dim=-1, keepdim=True) * am).sum() / am.sum()
        self.opt_a.zero_grad()
        (policy_loss - dist_entropy * c["entropy_coef"]).backward()
        actor_grad_norm = torch.nn.utils.clip_grad_norm_(self.actor.params(), c["max_grad_norm"])
        self.opt_a.step()
        delta = -((s["aver_episode_costs"].mean() - c["cost_limit"]) * (1 - c["gamma"]) + (imp_weights * s["cost_adv_targ"])).mean().detach()
        self.lamda_lagr = torch.nn.ReLU()(self.lamda_lagr - (delta * c["lagrangian_coef_rate"]))
        value_loss = self.cal_value_loss(values, s["value_preds"], s["returns"])
        self.opt_c.zero_grad()
        (value_loss * c["value_loss_coef"]).backward()
        critic_grad_norm = torch.nn.utils.clip_grad_norm_(self.critic.params(), c["max_grad_norm"])
        self.opt_c.step()
        cost_loss = self.cal_value_loss(cost_values, s["cost_preds"], s["cost_returns"])
        self.opt_k.zero_grad()
        (cost_loss * c["value_loss_coef"]).backward()
        cost_grad_norm = torch.nn.utils.clip_grad_norm_(self.cost_critic.params(), c["max_grad_norm"])
        self.opt_k.step()
        return dict(value_loss=value_loss.detach(), critic_grad_norm=critic_grad_norm, policy_loss=policy_loss.detach(),
                    dist_entropy=dist_entropy.detach(), actor_grad_norm=actor_grad_norm, imp_weights=imp_weights.detach(),
                    cost_loss=cost_loss.detach(), cost_grad_norm=cost_grad_norm)


class OracleMaskedMABuffer(MA.OracleMABuffer):
    """OracleMABuffer whose sample also carries the active masks of the rows' own steps (buffer.py:417-418)."""

    def whole_batch_sample(self, advantages, cost_adv, perm=None):
        idx = torch.randperm(self.T * self.N) if perm is None else perm
        flat = lambda t: t.reshape(-1, t.shape[-1])[idx]        # noqa: E731
        return dict(share_obs=flat(self.share_obs[:-1]), obs=flat(self.obs[:-1]), actions=flat(self.actions),
                    value_preds=flat(self.value_preds[:-1]), returns=flat(self.returns[:-1]),
                    old_action_log_probs=flat(self.action_log_probs), adv_targ=flat(advantages), factor=flat(self.factor),
                    cost_preds=flat(self.cost_preds[:-1]), cost_returns=flat(self.cost_returns[:-1]), cost_adv_targ=flat(cost_adv),
                    aver_episode_costs=self.aver_episode_costs, active_masks=flat(self.active_masks[:-1]))


class _PerAgent:
    """The reference runners' two environment conventions: observations as the stacked [N, agents, D] tensor or one [N, D_i]
    tensor per agent; with ``pad_to`` every agent's actions padded with zero columns to that width after collect and cut back
    to its own width on insert."""

    def _setup(self, obs_dims, act_dims, pad_to):
        self.obs_dims, self.act_dims, self.pad_to = list(obs_dims), list(act_dims), pad_to

    def _obs(self, obs):
        return list(obs) if isinstance(obs, (list, tuple)) else [obs[:, a] for a in range(self.num_agents)]

    def _pad(self, actions):
        if self.pad_to is None:
            return actions
        return [x if x.shape[1] == self.pad_to else torch.cat((x, torch.zeros(x.shape[0], self.pad_to - x.shape[1])), dim=1) for x in actions]

    def _trim(self, actions):
        return [x[:, :A] for x, A in zip(actions, self.act_dims)]

    def warmup(self, obs, share_obs):
        for a, (b, o) in enumerate(zip(self.buffer, self._obs(obs))):
            b.share_obs[0].copy_(share_obs[:, a])
            b.obs[0].copy_(o)


class OracleHeteroMARunner(_PerAgent, MA.OracleMARunner):
    """OracleMARunner (MAPPO-Lag) with per-agent sizes and the masked trainer."""

    def __init__(self, nets, cfg, T, N, obs_dims, share_obs_dim, act_dims, pad_to=None):
        self.cfg, self.T, self.N, self.num_agents = cfg, T, N, len(nets)
        self.nets = nets
        self._setup(obs_dims, act_dims, pad_to)
        self.trainer = [OracleMaskedMATrainer(a, c, k, cfg) for a, c, k in nets]
        self.buffer = [OracleMaskedMABuffer(T, N, D, share_obs_dim, A, cfg["gamma"], cfg["gae_lambda"]) for D, A in zip(obs_dims, act_dims)]

    def collect(self, step, eps=None):
        values, actions, logps, cost_preds = super().collect(step, eps)
        return values, self._pad(actions), logps, cost_preds

    def insert(self, obs, share_obs, rewards, costs, dones, values, actions, action_log_probs, cost_preds):
        dones_env = torch.all(dones, dim=1)
        masks = torch.ones(self.N, self.num_agents, 1)
        masks[dones_env] = 0.0
        active_masks = torch.ones(self.N, self.num_agents, 1)
        active_masks[dones] = 0.0
        active_masks[dones_env] = 1.0
        for a, (b, o, act) in enumerate(zip(self.buffer, self._obs(obs), self._trim(actions))):
            b.insert(share_obs[:, a], o, act, action_log_probs[a], values[:, a], rewards[:, a], masks[:, a], active_masks[:, a], costs[:, a],
                     cost_preds[:, a])


class OracleHeteroTwoNetRunner(_PerAgent, PO.OracleTwoNetRunner):
    """OracleTwoNetRunner (MAPPO / HAPPO) with per-agent sizes."""

    def __init__(self, nets, cfg, T, N, obs_dims, share_obs_dim, act_dims, trainer_class, pad_to=None):
        self.cfg, self.T, self.N, self.num_agents = cfg, T, N, len(nets)
        self.nets = nets
        self._setup(obs_dims, act_dims, pad_to)
        self.trainer = [trainer_class(a, c, cfg) for a, c in nets]
        self.buffer = [PO.OracleTwoNetBuffer(T, N, D, share_obs_dim, A, cfg["gamma"], cfg["gae_lambda"]) for D, A in zip(obs_dims, act_dims)]

    def collect(self, step, eps=None):
        values, actions, logps = super().collect(step, eps)
        return values, self._pad(actions), logps

    def insert(self, obs, share_obs, rewards, dones, values, actions, action_log_probs):
        dones_env = torch.all(dones, dim=1)
        masks = torch.ones(self.N, self.num_agents, 1)
        masks[dones_env] = 0.0
        active_masks = torch.ones(self.N, self.num_agents, 1)
        active_masks[dones] = 0.0
        active_masks[dones_env] = 1.0
        for a, (b, o, act) in enumerate(zip(self.buffer, self._obs(obs), self._trim(actions))):
            b.insert(share_obs[:, a], o, act, action_log_probs[a], values[:, a], rewards[:, a], masks[:, a], active_masks[:, a])


class OracleHeteroMACPORunner(OracleHeteroMARunner):
    """tests/macpo_oracle.py's OracleMACPORunner (MAPPO-Lag's iteration with MACPO's trainer) with per-agent sizes."""

    def __init__(self, nets, cfg, T, N, obs_dims, share_obs_dim, act_dims, pad_to=None):
        import macpo_oracle as MO
        super().__init__(nets, dict(cfg, lamda_lagr=cfg.get("lamda_lagr", 0.0)), T, N, obs_dims, share_obs_dim, act_dims, pad_to)
        self.cfg = cfg
        self.trainer = [MO.OracleMACPOTrainer(a, c, k, cfg) for a, c, k in nets]

    def train(self, agent_order=None, perms=None):
        import macpo_oracle as MO
        return MO.OracleMACPORunner.train(self, agent_order, perms)
