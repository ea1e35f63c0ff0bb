"""TEST INFRASTRUCTURE ONLY (see oracle/__init__.py): CPU restatement of MAPPO and HAPPO, the two-net multi-agent algorithms.

Restates safepo/multi_agent/mappo.py:96-186 (MAPPO_Trainer: cal_value_loss, ppo_update, train) and happo.py:96-194
(HAPPO_Trainer), with safepo/utils/act.py:62-77 (evaluate_actions: the masked entropy (entropy() * m).sum() / m.sum() over
the [n, A] entropies) and the runners' collect / insert / compute / train (mappo.py:347-437, 518-526; happo.py's are the
same), with the reference's torch ops in its order, fp32, and the same draws from torch's global generator.  Both mask
flags are honoured where the reference honours them: MAPPO's value loss is always a plain mean (mappo.py:117).  The networks,
PopArt, the masked GAE and the buffer are oracle/ma_oracle.py's.  Pinned by tests/golden/mappo.pt (outputs of the reference's
own MAPPO_Trainer / HAPPO_Trainer and Runners) through tests/test_mappo_happo.py."""
import torch

from oracle.ma_oracle import OracleMABuffer, OraclePopArt, huber_loss, ma_actor_dist, ma_critic_value, masked_gae


class OracleTwoNetTrainer:
    """MAPPO_Trainer / HAPPO_Trainer around two OracleMANets (actor, critic): Adam(lr, eps=opti_eps) x 2 and one PopArt that
    every cal_value_loss call updates twice."""

    PRODUCT_RATIO = None      # subclasses: False = MAPPO's per-dimension clip, True = HAPPO's product ratio x factor

    def __init__(self, actor, critic, cfg):
        self.actor, self.critic, self.cfg = actor, critic, cfg
        self.opt_a = torch.optim.Adam(actor.params(), lr=cfg["actor_lr"], eps=cfg["opti_eps"], weight_decay=cfg["weight_decay"])
        self.opt_c = torch.optim.Adam(critic.params(), lr=cfg["critic_lr"], eps=cfg["opti_eps"], weight_decay=cfg["weight_decay"])
        self.popart = OraclePopArt(1)

    def value_masks_used(self):
        return self.PRODUCT_RATIO and self.cfg["use_value_active_masks"]

    def cal_value_loss(self, values, value_preds_batch, return_batch, active_masks_batch):
        c = self.cfg
        value_pred_clipped = value_preds_batch + (values - value_preds_batch).clamp(-c["clip_param"], c["clip_param"])
        error_clipped = self.popart.normalize(return_batch) - value_pred_clipped
        error_original = self.popart.normalize(return_batch) - values
        value_loss = torch.max(huber_loss(error_original, c["huber_delta"]), huber_loss(error_clipped, c["huber_delta"]))
        if self.value_masks_used():
            return (value_loss * active_masks_batch).sum() / active_masks_batch.sum()
        return value_loss.mean()

    def ppo_update(self, s):
        """s: dict with share_obs, obs, actions, value_preds, returns, active_masks, old_action_log_probs [N,A], adv_targ and
        (HAPPO) factor.  Returns the reference's six values."""
        c = self.cfg
        am = s["active_masks"]
        dist = ma_actor_dist(self.actor, s["obs"], c["std_x_coef"], c["std_y_coef"])
        action_log_probs = dist.log_prob(s["actions"])
        if c["use_policy_active_masks"]:
            dist_entropy = (dist.entropy() * am).sum() / am.sum()
        else:
            dist_entropy = dist.entropy().mean()
        values = ma_critic_value(self.critic, s["share_obs"])
        imp_weights = torch.exp(action_log_probs - s["old_action_log_probs"])
        if self.PRODUCT_RATIO:
            imp_weights = torch.prod(imp_weights, dim=-1, keepdim=True)
        surr1 = imp_weights * s["adv_targ"]
        surr2 = torch.clamp(imp_weights, 1.0 - c["clip_param"], 1.0 + c["clip_param"]) * s["adv_targ"]
        inner = s["factor"] * torch.min(surr1, surr2) if self.PRODUCT_RATIO else torch.min(surr1, surr2)
        if c["use_policy_active_masks"]:
            policy_loss = (-torch.sum(inner, dim=-1, keepdim=True) * am).sum() / am.sum()
        else:
            policy_loss = -torch.sum(inner, dim=-1, keepdim=True).mean()
        self.opt_a.zero_grad()
        (policy_loss - dist_entropy * c["entropy_coef"]).backward()
        actor_grad_norm = torch.nn.utils.clip_grad_norm_(self.actor.params(), c["max_grad_norm"])
        self.opt_a.step()
        value_loss = self.cal_value_loss(values, s["value_preds"], s["returns"], am)
        self.opt_c.zero_grad()
        (value_loss * c["value_loss_coef"]).backward()
        critic_grad_norm = torch.nn.utils.clip_grad_norm_(self.critic.params(), c["max_grad_norm"])
        self.opt_c.step()
        return dict(value_loss=value_loss.detach(), critic_grad_norm=critic_grad_norm, policy_loss=policy_loss.detach(),
                    dist_entropy=dist_entropy.detach(), actor_grad_norm=actor_grad_norm, imp_weights=imp_weights.detach())

    def train(self, buf, perms=None):
        """mappo.py:165-186: advantages standardised with std + 1e-5 over every entry, learning_iters whole-batch updates."""
        advantages = buf.returns[:-1] - self.popart.denormalize(buf.value_preds[:-1])
        advantages_copy = advantages.clone()
        mean_advantages = torch.mean(advantages_copy)
        std_advantages = torch.std(advantages_copy)
        advantages = (advantages - mean_advantages) / (std_advantages + 1e-5)
        out = None
        for it in range(self.cfg["learning_iters"]):
            out = self.ppo_update(buf.whole_batch_sample(advantages, None, None if perms is None else perms[it]))
        return out


class OracleMAPPOTrainer(OracleTwoNetTrainer):
    PRODUCT_RATIO = False


class OracleHAPPOTrainer(OracleTwoNetTrainer):
    PRODUCT_RATIO = True


class OracleTwoNetBuffer(OracleMABuffer):
    """SeparatedReplayBuffer without the cost side (mappo.py:402-406 inserts None costs)."""

    def insert(self, share_obs, obs, actions, action_log_probs, value_preds, rewards, masks, active_masks, costs=None, cost_preds=None):
        s = self.step
        self.share_obs[s + 1].copy_(share_obs)
        self.obs[s + 1].copy_(obs)
        self.actions[s].copy_(actions)
        self.action_log_probs[s].copy_(action_log_probs)
        self.value_preds[s].copy_(value_preds)
        self.rewards[s].copy_(rewards)
        self.masks[s + 1].copy_(masks)
        self.active_masks[s + 1].copy_(active_masks)
        self.step = (s + 1) % self.T

    def whole_batch_sample(self, advantages, cost_adv=None, perm=None):
        idx = torch.randperm(self.T * self.N) if perm is None else perm
        flat = lambda t: t.reshape(-1, t.shape[-1])[idx]        # noqa: E731
        return dict(share_obs=flat(self.share_obs[:-1]), obs=flat(self.obs[:-1]), actions=flat(self.actions),
                    value_preds=flat(self.value_preds[:-1]), returns=flat(self.returns[:-1]),
                    old_action_log_probs=flat(self.action_log_probs), adv_targ=flat(advantages), factor=flat(self.factor),
                    active_masks=flat(self.active_masks[:-1]))


class OracleTwoNetRunner:
    """The per-iteration part of MAPPO's / HAPPO's Runner (mappo.py:261-291 without environments and logging): agents = list
    of (actor, critic) OracleMANets; ``trainer_class`` = OracleMAPPOTrainer or OracleHAPPOTrainer."""

    def __init__(self, nets, cfg, T, N, obs_dim, share_obs_dim, act_dim, trainer_class):
        self.cfg, self.T, self.N, self.num_agents = cfg, T, N, len(nets)
        self.nets = nets
        self.trainer = [trainer_class(a, c, cfg) for a, c in nets]
        self.buffer = [OracleTwoNetBuffer(T, N, obs_dim, share_obs_dim, act_dim, cfg["gamma"], cfg["gae_lambda"]) for _ in nets]

    def warmup(self, obs, share_obs):
        for a, b in enumerate(self.buffer):
            b.share_obs[0].copy_(share_obs[:, a])
            b.obs[0].copy_(obs[:, a])

    def collect(self, step, eps=None):
        """eps: per-agent standard-normal draws replacing Normal.sample()."""
        c = self.cfg
        values, actions, logps = [], [], []
        with torch.no_grad():
            for a, (actor, critic) in enumerate(self.nets):
                b = self.buffer[a]
                dist = ma_actor_dist(actor, b.obs[step], c["std_x_coef"], c["std_y_coef"])
                act = dist.sample() if eps is None else dist.mean + dist.stddev * eps[a]
                values.append(ma_critic_value(critic, b.share_obs[step])), actions.append(act), logps.append(dist.log_prob(act))
        return torch.transpose(torch.stack(values), 1, 0), actions, logps

    def insert(self, obs, share_obs, rewards, dones, values, actions, action_log_probs):
        dones_env = torch.all(dones, dim=1)
        masks = torch.ones(self.N, self.num_agents, 1)
        masks[dones_env] = 0.0
        active_masks = torch.ones(self.N, self.num_agents, 1)
        active_masks[dones] = 0.0
        active_masks[dones_env] = 1.0
        for a, b in enumerate(self.buffer):
            b.insert(share_obs[:, a], obs[:, a], actions[a], action_log_probs[a], values[:, a], rewards[:, a], masks[:, a], active_masks[:, a])

    def compute(self):
        with torch.no_grad():
            for (actor, critic), b, tr in zip(self.nets, self.buffer, self.trainer):
                b.value_preds[-1] = ma_critic_value(critic, b.share_obs[-1])
                b.returns[:-1] = masked_gae(b.rewards, b.value_preds, b.masks, tr.popart, b.gamma, b.gae_lambda)

    def train(self, agent_order=None, perms=None):
        """The cross-agent factor loop (mappo.py:408-437); returns {agent: its last update's values}."""
        c = self.cfg
        factor = torch.ones(self.T, self.N, 1)
        outs = {}
        for agent_id in (torch.randperm(self.num_agents) if agent_order is None else agent_order):
            a = int(agent_id)
            b, tr, actor = self.buffer[a], self.trainer[a], self.nets[a][0]
            A = b.actions.shape[-1]
            b.factor.copy_(factor)
            flat_obs, flat_act = b.obs[:-1].reshape(-1, b.obs.shape[-1]), b.actions.reshape(-1, A)
            with torch.no_grad():
                old_lp = ma_actor_dist(actor, flat_obs, c["std_x_coef"], c["std_y_coef"]).log_prob(flat_act)
            outs[a] = tr.train(b, None if perms is None else perms[a])
            with torch.no_grad():
                new_lp = ma_actor_dist(actor, flat_obs, c["std_x_coef"], c["std_y_coef"]).log_prob(flat_act)
            factor = factor * torch.prod(torch.exp(new_lp - old_lp).reshape(self.T, self.N, A), dim=-1, keepdim=True)
            b.after_update()
        return outs
