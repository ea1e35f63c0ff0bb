"""GPU parity at BASELINE.json's FULL sizes, and the kernel-level cases the round-1 review found missing.

* config 2 (PPO-Lag, 1024 envs x 1000 steps: S = 1 024 000, 16 000 minibatch steps per pass): one whole pass of the
  update kernel against the oracle's loop on the same permutation.  Two views:
    - teacher-forced: every CHUNK steps the device weights / Adam state are re-loaded from the oracle, so the numbers
      are per-CHUNK-step errors without the chaotic amplification of a 16 000-step Adam chain;
    - free-running: a second device policy runs the whole pass on its own; its drift from the oracle is reported
      (and bounded loosely): two fp32 implementations of a 16 000-step chain cannot agree to 1e-5.
  The measured errors are printed (run with -s) and bounded; see DESIGN.md section "Numerics" for the per-quantity bars.
* config 3 (CPO, obs 88, S = 1 024 000): Fisher-vector product, conjugate gradient, line-search evaluation.
* SPO_LOSS_CRITIC_ONLY at kernel level (cpo.py:543-571), with gradients large enough to trigger the joint clip, with
  and without a stale actor gradient in the norm.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import spo_oracle as O

pytestmark = pytest.mark.gpu


def _cuda():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    return torch.device("cuda:0")


def policy_state(pol):
    return {n: {k: v.detach().cpu().clone() for k, v in getattr(pol, n).state_dict().items()}
            for n in ("actor", "reward_critic", "cost_critic")}


def load_oracle_state(pol, adam, opol, opt):
    """Device weights, Adam moments and step counters <- the oracle's (packed layout = parameter order of the nets)."""
    flat, m, v, t = [], [], [], []
    for name, o in (("actor", opt.actor), ("reward_critic", opt.reward_critic), ("cost_critic", opt.cost_critic)):
        step = 0
        for p in opol.params(name):
            flat.append(p.detach().reshape(-1))
            st = o.state.get(p, {})
            m.append(st["exp_avg"].reshape(-1) if st else torch.zeros(p.numel()))
            v.append(st["exp_avg_sq"].reshape(-1) if st else torch.zeros(p.numel()))
            if st:
                step = int(st["step"])
        t.append(step)
    dev = pol.flat.device
    with torch.no_grad():
        pol.flat.copy_(torch.cat(flat).to(dev))
    adam.m.copy_(torch.cat(m).to(dev))
    adam.v.copy_(torch.cat(v).to(dev))
    adam.t.copy_(torch.tensor(t, dtype=torch.int32, device=dev))


def oracle_flat(opol):
    # packed order of libspo (include/spo.h): actor | reward critic | cost critic -- NOT O.NET_ORDER (the RNG construction order)
    return torch.cat([p.detach().reshape(-1) for n in ("actor", "reward_critic", "cost_critic") for p in opol.params(n)])


def test_update_full_config2_pass_vs_oracle():
    from safepo import _lib as L
    from safepo.common.model import ActorVCritic
    from safepo.single_agent._engine import PolicyGradientUpdate
    dev = _cuda()
    D, A, N, T, B, CHUNK = 60, 2, 1024, 1000, 64, 100
    S = N * T
    torch.manual_seed(2)
    torch.set_num_threads(4)
    pol = ActorVCritic(D, A, [64, 64]).to(dev)
    free = ActorVCritic(D, A, [64, 64]).to(dev)
    with torch.no_grad():
        free.flat.copy_(pol.flat)
    opol = O.OraclePolicy(D, A)
    opol.load(policy_state(pol))
    g = torch.Generator().manual_seed(S)
    obs = torch.randn(S, D, generator=g)
    with torch.no_grad():
        mean, std = O.actor_mean_std(opol, obs)
        act = mean + std * torch.randn(S, A, generator=g)
        logp = O.normal_log_prob(act, mean, std).sum(-1) + 0.05 * torch.randn(S, generator=g)
    data_cpu = {"obs": obs, "act": act, "log_prob": logp, "target_value_r": torch.randn(S, generator=g),
                "target_value_c": torch.randn(S, generator=g).abs(), "adv": torch.randn(S, generator=g)}
    perm = torch.randperm(S, generator=g)
    # loss_pi = -mean(min(ratio * adv, clip(ratio) * adv)) is a mean of SIGNED terms of magnitude ~|adv| that nearly cancel
    # (|loss_pi| ~ 0.05 here): the 1e-5 bar applies relative to the mean magnitude of its terms, not to the cancelled sum
    pi_scale = float(data_cpu["adv"].abs().mean())
    cfg = dict(hidden_sizes=[64, 64], gamma=0.99, target_kl=1e9, batch_size=B, learning_iters=1, max_grad_norm=40.0)
    upd = PolicyGradientUpdate(pol, cfg, L.LOSS_PPO_CLIP, epochs=10 ** 9, host_rng=False, device=dev)
    upd_free = PolicyGradientUpdate(free, cfg, L.LOSS_PPO_CLIP, epochs=10 ** 9, host_rng=False, device=dev)
    data = {k: v.to(dev).contiguous() for k, v in data_cpu.items()}
    opt = O.OracleOptim(opol)
    n_steps = S // B
    assert n_steps == 16000
    loss_rel, w_abs, w_rel, free_abs = [], [], [], []
    for c0 in range(0, n_steps, CHUNK):
        idx = perm[c0 * B:(c0 + CHUNK) * B]
        res = upd.run(data, perms=[idx], refresh_old=(c0 == 0))
        res_f = upd_free.run(data, perms=[idx], refresh_old=(c0 == 0))
        assert res["steps"] == CHUNK and res_f["steps"] == CHUNK
        losses = []
        for s in range(CHUNK):
            ii = idx[s * B:(s + 1) * B]
            losses.append(O.minibatch_step(opol, opt, {k: v[ii] for k, v in data_cpu.items()}, "ppo"))
        want = torch.tensor(losses, dtype=torch.float64).mean(0)
        got = torch.tensor([res["loss_r"], res["loss_c"], res["loss_pi"]], dtype=torch.float64)
        den = torch.maximum(want.abs(), torch.tensor([0.0, 0.0, pi_scale], dtype=torch.float64))
        loss_rel.append(((got - want).abs() / den).max().item())
        of = oracle_flat(opol)
        err = (pol.flat.detach().cpu() - of).abs()
        w_abs.append(err.max().item())
        w_rel.append((err.norm() / of.norm()).item())
        free_abs.append((free.flat.detach().cpu() - of).abs().max().item())
        load_oracle_state(pol, upd.adam, opol, opt)       # teacher forcing: next chunk starts from the oracle's state
    loss_rel, w_abs, w_rel, free_abs = map(np.array, (loss_rel, w_abs, w_rel, free_abs))
    print(f"\nconfig 2 full pass (16000 steps, S={S}), teacher-forced every {CHUNK} steps:"
          f"\n  chunk-mean losses, max rel error over r/c/pi: median {np.median(loss_rel):.2e}  p90 {np.percentile(loss_rel, 90):.2e}  max {loss_rel.max():.2e}"
          f"\n  weights after {CHUNK} steps: max |dtheta| median {np.median(w_abs):.2e}  max {w_abs.max():.2e};  ||dtheta||/||theta|| max {w_rel.max():.2e}"
          f"\nfree-running device chain vs oracle: max |dtheta| after 1000 / 4000 / 16000 steps: "
          f"{free_abs[9]:.2e} / {free_abs[39]:.2e} / {free_abs[-1]:.2e}")
    # the weight bound allows a handful of near-zero-gradient coordinates where Adam's m / sqrt(v) flips sign
    assert loss_rel.max() < 1e-5, loss_rel.max()
    assert w_abs.max() < 6e-5 and w_rel.max() < 1e-5 and np.median(w_abs) < 1e-6, (w_abs.max(), w_rel.max(), np.median(w_abs))
    assert free_abs[-1] < 0.05, free_abs[-1]                   # sanity only: the chains stay in the same basin


def test_update_per_step_error_histogram_config2_shape():
    """Per-STEP losses, one launch per minibatch step, device state re-loaded from the oracle before every step:
    the error of one forward/loss evaluation at identical weights (north_star: 1e-5 relative on losses)."""
    from safepo import _lib as L
    from safepo.common.model import ActorVCritic
    from safepo.single_agent._engine import PolicyGradientUpdate
    dev = _cuda()
    D, A, B, S, STEPS = 60, 2, 64, 64 * 256, 256
    torch.manual_seed(3)
    pol = ActorVCritic(D, A, [64, 64]).to(dev)
    opol = O.OraclePolicy(D, A)
    opol.load(policy_state(pol))
    g = torch.Generator().manual_seed(11)
    obs = torch.randn(S, D, generator=g)
    with torch.no_grad():
        mean, std = O.actor_mean_std(opol, obs)
        act = mean + std * torch.randn(S, A, generator=g)
        logp = O.normal_log_prob(act, mean, std).sum(-1) + 0.05 * torch.randn(S, generator=g)
    data_cpu = {"obs": obs, "act": act, "log_prob": logp, "target_value_r": torch.randn(S, generator=g),
                "target_value_c": torch.randn(S, generator=g).abs(), "adv": torch.randn(S, generator=g)}
    perm = torch.randperm(S, generator=g)
    pi_scale = float(data_cpu["adv"].abs().mean())     # loss_pi relative to the mean magnitude of its signed terms (see the test above)
    cfg = dict(hidden_sizes=[64, 64], gamma=0.99, target_kl=1e9, batch_size=B, learning_iters=1, max_grad_norm=40.0)
    upd = PolicyGradientUpdate(pol, cfg, L.LOSS_PPO_CLIP, epochs=10 ** 9, host_rng=False, device=dev)
    data = {k: v.to(dev).contiguous() for k, v in data_cpu.items()}
    opt = O.OracleOptim(opol)
    rel = []
    wstep = []
    for s in range(STEPS):
        idx = perm[s * B:(s + 1) * B]
        res = upd.run(data, perms=[idx], refresh_old=(s == 0))
        want = O.minibatch_step(opol, opt, {k: v[idx] for k, v in data_cpu.items()}, "ppo")
        got = (res["loss_r"], res["loss_c"], res["loss_pi"])
        rel.append([abs(a - b) / max(abs(b), sc) for a, b, sc in zip(got, want, (0.0, 0.0, pi_scale))])
        wstep.append((pol.flat.detach().cpu() - oracle_flat(opol)).abs().max().item())
        load_oracle_state(pol, upd.adam, opol, opt)
    rel = np.array(rel)
    wstep = np.array(wstep)
    print(f"\nper-step loss error at identical weights ({STEPS} steps, batch 64, obs 60): rel error (r, c, pi)"
          f"\n  median {np.median(rel, 0)}  p99 {np.percentile(rel, 99, 0)}  max {rel.max(0)}"
          f"\n  one Adam step: max |dtheta| vs oracle median {np.median(wstep):.2e} max {wstep.max():.2e} (lr 3e-4)")
    assert rel.max() < 1e-5, rel.max(0)
    assert wstep.max() < 1e-6, wstep.max()


@pytest.mark.parametrize("extra", [0.0, 900.0])
def test_critic_only_mode_vs_oracle(extra):
    """cpo.py:543-571 at kernel level: batch 128 (two tiles per step), lr 1e-3, the critics' joint clip active
    (targets scaled so that the gradient norm exceeds 40), actor untouched.  extra > 0: a stale actor gradient with that
    squared norm joins the clip (ctrl->extra_sumsq), as torch's clip_grad_norm_ over policy.parameters() would see it."""
    from safepo.common.model import ActorVCritic
    from safepo.single_agent._engine import CriticRegression
    dev = _cuda()
    D, A, S, B = 88, 2, 128 * 6 + 37, 128
    torch.manual_seed(4)
    pol = ActorVCritic(D, A, [64, 64]).to(dev)
    opol = O.OraclePolicy(D, A)
    opol.load(policy_state(pol))
    opol0 = opol.clone()
    g = torch.Generator().manual_seed(5)
    data_cpu = {"obs": torch.randn(S, D, generator=g), "target_value_r": 60.0 * torch.randn(S, generator=g),
                "target_value_c": 45.0 * torch.randn(S, generator=g).abs()}
    perms = [torch.randperm(S, generator=g) for _ in range(2)]
    cfg = dict(hidden_sizes=[64, 64], gamma=0.99, target_kl=0.01, batch_size=B, learning_iters=2, max_grad_norm=40.0)
    crit = CriticRegression(pol, cfg, host_rng=False, device=dev)
    data = {k: v.to(dev).contiguous() for k, v in data_cpu.items()}
    actor_before = pol.flat[: pol.n_actor].clone()
    res = crit.run(data, stale_actor_grad_sumsq=extra, perms=perms)
    opt = O.OracleOptim(opol, lr=3e-4, critic_lr=1e-3)
    losses = []
    for perm in perms:
        for s0 in range(0, S, B):
            idx = perm[s0:s0 + B]
            if extra > 0:       # the stale actor gradient: sqrt(extra) on one coordinate (clip_grad_norm_ rescales it in place each step)
                for p in opol.params("actor"):
                    p.grad = torch.zeros_like(p)
                opol.params("actor")[0].grad[0] = extra ** 0.5
            lr_, lc_, _ = O.minibatch_step(opol, opt, {k: v[idx] for k, v in data_cpu.items()}, "critic")
            losses.append((lr_, lc_))
    want = torch.tensor(losses, dtype=torch.float64).mean(0)
    assert res["steps"] == len(losses)
    for name, got, w in (("loss_r", res["loss_r"], want[0]), ("loss_c", res["loss_c"], want[1])):
        assert abs(got - float(w)) <= 2e-5 * abs(float(w)), (name, got, float(w))
    final = policy_state(pol)
    worst = 0.0
    for net in ("reward_critic", "cost_critic"):
        for k, v in opol.state()[net].items():
            worst = max(worst, float((final[net][k] - v).abs().max()))
    assert worst < 1e-4, worst              # 14 Adam steps of lr 1e-3
    assert torch.equal(pol.flat[: pol.n_actor], actor_before)       # the actor is not touched in this mode
    # the first step really is clipped (otherwise the test would not exercise the clip path)
    first = {k: v[perms[0][:B]] for k, v in data_cpu.items()}
    l_r, l_c = O.critic_losses(opol0, first["obs"], first["target_value_r"], first["target_value_c"])
    (l_r + l_c).backward()
    gn0 = torch.sqrt(sum((p.grad ** 2).sum() for n in ("reward_critic", "cost_critic") for p in opol0.params(n)))
    assert float(gn0) > 40.0, float(gn0)


def test_trust_region_pieces_at_config3_size():
    """CPO config 3 (SafetyCarButton1 shape: obs 88, act 2; 1024 envs x 1000 steps): FVP, CG and the line-search
    evaluation on S = 1 024 000 samples against the oracle (the closed-form FVP of the oracle is pinned against the
    reference's double backprop in tests/test_oracle_golden.py)."""
    from safepo.common.model import ActorVCritic
    from safepo.single_agent._engine import TrustRegionUpdate
    dev = _cuda()
    D, A, S = 88, 2, 1024 * 1000
    torch.manual_seed(6)
    torch.set_num_threads(8)
    pol = ActorVCritic(D, A, [64, 64]).to(dev)
    with torch.no_grad():
        pol.actor.log_std.copy_(torch.tensor([-0.3, 0.1]))
    opol = O.OraclePolicy(D, A)
    opol.load(policy_state(pol))
    g = torch.Generator().manual_seed(7)
    obs = torch.randn(S, D, generator=g)
    with torch.no_grad():
        mean, std = O.actor_mean_std(opol, obs)
        act = mean + std * torch.randn(S, A, generator=g)
        logp = O.normal_log_prob(act, mean, std).sum(-1)
    data_cpu = {"obs": obs, "act": act, "log_prob": logp, "adv_r": torch.randn(S, generator=g), "adv_c": torch.randn(S, generator=g)}
    cfg = dict(hidden_sizes=[64, 64], gamma=0.99, target_kl=0.01, batch_size=128, learning_iters=10, max_grad_norm=40.0)
    tr = TrustRegionUpdate(pol, cfg, dev)
    data = {k: v.to(dev).contiguous() for k, v in data_cpu.items()}
    P = pol.n_actor
    v = torch.randn(P, generator=g)
    # surrogate gradient
    loss = tr._grad(data, data["adv_r"], tr.g)
    for p in opol.params("actor"):
        p.grad = None
    want_loss = O.surrogate_loss(opol, obs, act, logp, data_cpu["adv_r"])
    want_loss.backward()
    want_g = O.flat_grads(opol)
    assert abs(float(loss) - float(want_loss.detach())) <= 1e-5 * abs(float(want_loss.detach())) + 1e-7
    eg = float((tr.g.cpu() - want_g).norm() / want_g.norm())
    # FVP
    tr._old_dist(data)
    tr._fvp(data, v.to(dev), tr.Fx)
    want_Fv = O.fvp_analytic(opol, obs, v)
    ef = float((tr.Fx.cpu() - want_Fv).norm() / want_Fv.norm())
    # CG on b = surrogate gradient
    tr._cg(data, tr.g, tr.x)
    want_x = O.conjugate_gradients(lambda z: O.fvp_analytic(opol, obs, z), want_g)
    ex = float((tr.x.cpu() - want_x).norm() / want_x.norm())
    r_mine = float((O.fvp_analytic(opol, obs, tr.x.cpu()) - want_g).norm())
    r_ref = float((O.fvp_analytic(opol, obs, want_x) - want_g).norm())
    # line-search evaluation at a trial point
    with torch.no_grad():
        om, os_ = O.actor_mean_std(opol, obs)
        om, os_ = om.clone(), os_.clone()
    step = 0.01 * torch.randn(P, generator=g)
    pol.actor_flat().add_(step.to(dev))
    O.set_flat_params(opol, O.flat_params(opol) + step)
    out = tr._eval(data, data["adv_r"], data["adv_c"])
    with torch.no_grad():
        w0 = O.surrogate_loss(opol, obs, act, logp, data_cpu["adv_r"])
        w1 = O.surrogate_loss(opol, obs, act, logp, data_cpu["adv_c"])
        m, s = O.actor_mean_std(opol, obs)
        w2 = O.normal_kl(om, os_, m, s).mean()
    els = [abs(float(a) - float(b)) / (abs(float(b)) + 1e-9) for a, b in zip(out, (w0, w1, w2))]
    print(f"\nconfig 3 size (obs 88, S={S}): surrogate grad rel {eg:.2e}, FVP rel {ef:.2e}, CG x rel {ex:.2e} "
          f"(residuals {r_mine:.3e} vs oracle {r_ref:.3e}), line-search evals rel {els}")
    assert eg < 1e-5 and ef < 1e-5, (eg, ef)
    assert ex < 5e-3 and r_mine <= 1.5 * r_ref + 1e-6, (ex, r_mine, r_ref)
    assert els[2] < 2e-5 and max(els[:2]) < 1e-3, els        # means of 1e6 signed terms (|mean| ~ 1e-3): absolute error ~1e-8
