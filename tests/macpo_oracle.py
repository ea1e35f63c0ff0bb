"""TEST INFRASTRUCTURE ONLY: CPU restatement of MACPO_Trainer (safepo/multi_agent/macpo.py:96-415) on the oracle's multi-agent
nets (oracle/ma_oracle.py: OracleMANet, ma_actor_dist, OracleMATrainer.cal_value_loss), same torch ops in the same order,
autograd for every derivative -- the yardstick of safepo/common/ma_model.py: MACPOTrainer.

Restated quirks of the reference, each cited where it happens:
- the KL has ``1e-8 +`` in its denominator (:163-164), so its Hessian along log_std is not the textbook one;
- CG (:168-185): ``+1e-8`` on p.Ap only, beta without eps, the break tests rdotr itself against 1e-10 (not its square root);
- ``rescale_constraint_val`` 0 is replaced by the float 1e-8 (:236-237), r / s 0 by 1e-8 (:282-285), and the recovery value 0
  by 1e-8 after the case split (:299-300);
- the line search rescales x to norm 0.5 before EVERY trial (:343-345) and applies the improvement test only when
  optim_case > 1 (:370); when no trial passes, the old weights come back (:376-378);
- train() standardises with std + 1e-5 and no NaN masking (:383-395) and runs one trpo_update (num_mini_batch = 1);
- the value the reference logs as "Loss_cost_critic" is the actor's cost surrogate (:248, :326, :405).
Parameters are flattened in state_dict order without padding, like Module.parameters()."""
import math

import torch

from oracle import ma_oracle as MA


class OracleMACPOTrainer(MA.OracleMATrainer):
    """MACPO_Trainer around three OracleMANets; the critic optimisers, PopArt and cal_value_loss are OracleMATrainer's
    (macpo.py:58-66,103,106-117 are the same as mappolag.py's)."""

    def __init__(self, actor, critic, cost_critic, cfg):
        super().__init__(actor, critic, cost_critic, dict(cfg, lamda_lagr=cfg.get("lamda_lagr", 0.0)))
        self.cfg = cfg

    # ---- macpo.py:119-151 ----
    def flat_params(self):
        return torch.cat([p.data.view(-1) for p in self.actor.params()])

    def update_model(self, net, flat):
        i = 0
        for p in net.params():
            k = p.numel()
            p.data.copy_(flat[i:i + k].view(p.size()))
            i += k

    def _eval(self, net, obs, actions):
        """MultiAgentActor.evaluate_actions -> evaluate_actions_trpo (act.py:76-97).  The yaml's use_policy_active_masks is False,
        so the actor gets no active masks and the entropy is entropy().mean() over rows AND dimensions (act.py:93-96)."""
        dist = MA.ma_actor_dist(net, obs, self.cfg["std_x_coef"], self.cfg["std_y_coef"])
        return dist.log_prob(actions), dist.entropy().mean(), dist.mean, dist.stddev

    def kl_divergence(self, obs, actions, new_actor, old_actor):
        """macpo.py:153-166."""
        _, _, mu, std = self._eval(new_actor, obs, actions)
        _, _, mu_old, std_old = self._eval(old_actor, obs, actions)
        logstd = torch.log(std)
        mu_old, std_old = mu_old.detach(), std_old.detach()
        logstd_old = torch.log(std_old)
        kl = logstd_old - logstd + (std_old.pow(2) + (mu_old - mu).pow(2)) / (1e-8 + 2.0 * std.pow(2)) - 0.5
        return kl.sum(1, keepdim=True)

    def fisher_vector_product(self, obs, actions, p):
        """macpo.py:187-198: double backprop of the mean KL of the actor against itself, plus 0.1 p."""
        kl = self.kl_divergence(obs, actions, self.actor, self.actor).mean()
        g = torch.cat([x.view(-1) for x in torch.autograd.grad(kl, self.actor.params(), create_graph=True)])
        hp = torch.autograd.grad((g * p).sum(), self.actor.params())
        return torch.cat([x.contiguous().view(-1) for x in hp]).data + 0.1 * p

    def conjugate_gradient(self, obs, actions, b, nsteps, residual_tol=1e-10):
        """macpo.py:168-185.  Also returns the number of iterations run."""
        x = torch.zeros(b.size())
        r, p = b.clone(), b.clone()
        rdotr = torch.dot(r, r)
        it = 0
        for _ in range(nsteps):
            it += 1
            Avp = self.fisher_vector_product(obs, actions, p)
            alpha = rdotr / (torch.dot(p, Avp) + 1e-8)
            x += alpha * p
            r -= alpha * Avp
            new_rdotr = torch.dot(r, r)
            betta = new_rdotr / rdotr
            p = r + betta * p
            rdotr = new_rdotr
            if rdotr < residual_tol:
                break
        return x, it

    def trpo_update(self, s):
        """macpo.py:200-380 on a sample dict (the oracle's keys).  Returns a dict of every intermediate the fixture pins."""
        c = self.cfg
        obs, actions = s["obs"], s["actions"]
        old_lp, adv, factor, cost_adv = s["old_action_log_probs"], s["adv_targ"], s["factor"], s["cost_adv_targ"]
        action_log_probs, dist_entropy, _, _ = self._eval(self.actor, obs, actions)          # :215-218
        values = MA.ma_critic_value(self.critic, s["share_obs"])
        cost_values = MA.ma_critic_value(self.cost_critic, s["share_obs"])
        value_loss = self.cal_value_loss(values, s["value_preds"], s["returns"])              # :220-224
        self.opt_c.zero_grad()
        (value_loss * c["value_loss_coef"]).backward()
        critic_grad_norm = torch.nn.utils.clip_grad_norm_(self.critic.params(), c["max_grad_norm"])
        self.opt_c.step()
        cost_critic_loss = self.cal_value_loss(cost_values, s["cost_preds"], s["cost_returns"])   # :226-231
        self.opt_k.zero_grad()
        (cost_critic_loss * c["value_loss_coef"]).backward()
        cost_grad_norm = torch.nn.utils.clip_grad_norm_(self.cost_critic.params(), c["max_grad_norm"])
        self.opt_k.step()

        rescale = (s["aver_episode_costs"].mean() - c["cost_limit"]) * (1 - c["gamma"])     # :234-237
        if rescale == 0:
            rescale = 1e-8
        ratio = torch.prod(torch.exp(action_log_probs - old_lp), dim=-1, keepdim=True)     # :239-240
        reward_loss = -torch.sum(ratio * factor * adv, dim=-1, keepdim=True).mean()
        g = torch.cat([x.view(-1) for x in torch.autograd.grad(reward_loss, self.actor.params(), retain_graph=True)])
        cost_loss = torch.sum(ratio * factor * cost_adv, dim=-1, keepdim=True).mean()
        b = torch.cat([x.view(-1) for x in torch.autograd.grad(cost_loss, self.actor.params(), retain_graph=True)])
        nsteps = c["conjugate_gradient_iters"]
        xg, it_g = self.conjugate_gradient(obs, actions, g.data, nsteps)                      # :255-262
        xb, it_b = self.conjugate_gradient(obs, actions, b.data, nsteps)
        q = (g * xg).sum(0, keepdim=True)                                                     # :264-266
        r = (g * xb).sum(0, keepdim=True)
        s_ = (b * xb).sum(0, keepdim=True)
        fraction = c["step_fraction"]
        bb = torch.dot(b, b)
        if bb <= 1e-8 and rescale < 0:                                                        # :272-278
            xb_used, r, s_ = torch.tensor(0), torch.tensor(0), torch.tensor(0)
            pos_cauchy, recover = torch.tensor(0), torch.tensor(0)
            optim_case = 4
        else:
            xb_used = xb
            r = (g * xb).sum(0, keepdim=True)
            s_ = (b * xb).sum(0, keepdim=True)
            if r == 0:
                r = 1e-8
            if s_ == 0:
                s_ = 1e-8
            pos_cauchy = q - (r ** 2) / (1e-8 + s_)
            recover = 2 * c["target_kl"] - (rescale ** 2) / (1e-8 + s_)
            if rescale < 0 and recover < 0:
                optim_case = 3
            elif rescale < 0 and recover >= 0:
                optim_case = 2
            elif rescale >= 0 and recover >= 0:
                optim_case = 1
            else:
                optim_case = 0
        if recover == 0:                                                                      # :299-300
            recover = 1e-8
        if optim_case in [3, 4]:                                                              # :302-321
            lam = torch.sqrt(q / (2 * c["target_kl"]))
            nu = torch.tensor(0)
        elif optim_case in [1, 2]:
            LA, LB = [0, r / rescale], [r / rescale, math.inf]
            LA, LB = (LA, LB) if rescale < 0 else (LB, LA)
            proj = lambda x, L: max(L[0], min(L[1], x))          # noqa: E731
            lam_a = proj(torch.sqrt(pos_cauchy / recover), LA)
            lam_b = proj(torch.sqrt(q / torch.tensor(2 * c["target_kl"])), LB)
            f_a = lambda lam: -0.5 * (pos_cauchy / (1e-8 + lam) + recover * lam) - r * rescale / (1e-8 + s_)   # noqa: E731
            f_b = lambda lam: -0.5 * (q / (1e-8 + lam) + 2 * c["target_kl"] * lam)                            # noqa: E731
            lam = lam_a if f_a(lam_a) >= f_b(lam_b) else lam_b
            nu = max(0, lam * rescale - r) / (1e-8 + s_)
        else:
            lam = torch.tensor(0)
            nu = torch.sqrt(torch.tensor(2 * c["target_kl"]) / (1e-8 + s_))
        x = (1. / (lam + 1e-8)) * (xg + nu * xb_used) if optim_case > 0 else nu * xb_used     # :323-325
        x0 = x.clone()
        reward_loss, cost_loss = reward_loss.detach(), cost_loss.detach()
        params = self.flat_params()
        old_actor = MA.OracleMANet(self.actor.state(), self.actor.layer_N)                  # :329-335
        expected_improve = (-torch.dot(x, g).sum(0, keepdim=True)).detach()
        flag, accepted = False, -1
        kl = loss_improve = None
        with torch.no_grad():
            for i in range(c["searching_steps"]):                                             # :342-374
                x_norm = torch.norm(x)
                if x_norm > 0.5:
                    x = x * 0.5 / x_norm
                self.update_model(self.actor, params - c["fraction_coef"] * (fraction ** i) * x)
                action_log_probs, dist_entropy, _, _ = self._eval(self.actor, obs, actions)
                ratio = torch.prod(torch.exp(action_log_probs - old_lp), dim=-1, keepdim=True)
                new_reward_loss = -torch.sum(ratio * factor * adv, dim=-1, keepdim=True).mean()
                new_cost_loss = torch.sum(ratio * factor * cost_adv, dim=-1, keepdim=True).mean()
                loss_improve = new_reward_loss - reward_loss
                kl = self.kl_divergence(obs, actions, self.actor, old_actor).mean()
                if (kl < c["target_kl"]) and (loss_improve < 0 if optim_case > 1 else True) and \
                        (new_cost_loss.mean() - cost_loss.mean() <= max(-rescale, 0)):
                    flag, accepted = True, i
                    break
                expected_improve *= fraction
            if not flag:                                                                      # :376-378
                self.update_model(self.actor, torch.cat([p.data.view(-1) for p in old_actor.params()]))
        return dict(value_loss=value_loss.detach(), critic_grad_norm=critic_grad_norm, cost_critic_loss=cost_critic_loss.detach(),
                    cost_grad_norm=cost_grad_norm, kl=kl, loss_improve=loss_improve, expected_improve=expected_improve,
                    dist_entropy=dist_entropy.detach(), ratio=ratio.detach(), cost_loss=cost_loss, reward_loss=reward_loss,
                    rescale=torch.as_tensor(rescale), g=g.detach(), b=b.detach(), xg=xg, xb=xb, cg_iters=(it_g, it_b),
                    q=q.detach(), r=torch.as_tensor(r).detach(), s=torch.as_tensor(s_).detach(), bb=bb.detach(), optim_case=optim_case,
                    lam=torch.as_tensor(lam).detach(), nu=torch.as_tensor(nu).detach(), x=x0.detach(), x_final=x.detach(),
                    accepted=accepted)

    def train(self, buf, perm=None):
        """macpo.py:382-400: standardise with std + 1e-5 (no NaN masking), one trpo_update on the whole batch."""
        def standardise(ret, pred):
            a = ret[:-1] - self.popart.denormalize(pred[:-1])
            cp = a.clone()
            return (a - torch.mean(cp)) / (torch.std(cp) + 1e-5)
        advantages = standardise(buf.returns, buf.value_preds)
        cost_adv = standardise(buf.cost_returns, buf.cost_preds)
        return self.trpo_update(buf.whole_batch_sample(advantages, cost_adv, perm))


class OracleMACPORunner(MA.OracleMARunner):
    """The MAPPO-Lag runner's iteration (oracle/ma_oracle.py: OracleMARunner) with MACPO's trainer: macpo.py's Runner shares
    collect / insert / compute / the cross-agent factor with mappolag.py; its train() calls MACPO_Trainer.train once per agent."""

    def __init__(self, nets, cfg, T, N, obs_dim, share_obs_dim, act_dim):
        super().__init__(nets, dict(cfg, lamda_lagr=cfg.get("lamda_lagr", 0.0)), T, N, obs_dim, share_obs_dim, act_dim)
        self.cfg = cfg
        self.trainer = [OracleMACPOTrainer(a, c, k, cfg) for a, c, k in nets]

    def train(self, agent_order=None, perms=None):
        factor = torch.ones(self.T, self.N, 1)
        outs = {}
        for agent_id in (torch.randperm(self.num_agents) if agent_order is None else agent_order):
            a = int(agent_id)
            b, tr, actor = self.buffer[a], self.trainer[a], self.nets[a][0]
            A = b.actions.shape[-1]
            b.factor.copy_(factor)
            flat_obs, flat_act = b.obs[:-1].reshape(-1, b.obs.shape[-1]), b.actions.reshape(-1, A)
            with torch.no_grad():
                old_lp = MA.ma_actor_dist(actor, flat_obs).log_prob(flat_act)
            outs[a] = tr.train(b, None if perms is None else perms[a][0])
            with torch.no_grad():
                new_lp = MA.ma_actor_dist(actor, flat_obs).log_prob(flat_act)
            factor = factor * torch.prod(torch.exp(new_lp - old_lp).reshape(self.T, self.N, A), dim=-1, keepdim=True)
            b.after_update()
        return outs
