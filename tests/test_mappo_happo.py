"""MAPPO and HAPPO on the device (csrc/spo_ma_ppo.cu, safepo/common/ma_model.py: MAPPOTrainer / HAPPOTrainer,
safepo/multi_agent/mappo.py / happo.py).

CPU: argument validation of the new entry points, the synthetic environment's opt-in lone finishes, and the host path of both
trainers and runners through an emulated C-ABI (tests/ppo_emulator.py) against oracle/ppo_oracle.py.
GPU: each new entry point against float64 autograd of the reference's formulas (both ratio modes, act_dim 1 / 20 / 32, n 1 / 33 /
4097, masks with zero rows and the all-zero NaN case, every per-dimension clip branch including the bounds themselves), the
product mode against MAPPO-Lag's spo_ma_actor_loss bit for bit, whole ppo_update calls and a runner iteration of each
algorithm against the oracle, and both CLIs.  Run with ``-s`` to see the measured maxima."""
import math
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F
from torch.distributions import Normal

from oracle import ma_oracle as MA
from oracle import ppo_oracle as PO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# Bars: error / scale (the tensor's max |float64| or the named scale), each at most 4x the largest error measured over this
# file's matrix on one H100 80GB HBM3 (in brackets).
BAR = dict(
    actor=3e-5,           # dmean, importance weights, g_b, g_log_std
    actor_loss=9e-6,      # policy loss (relative to the mean |term|), entropy, mean ratio
    value=2.4e-7,         # dv, its sum and the loss of spo_ma_value_loss_masked
)
MEASURED = {}
X_COEF, Y_COEF = 1.7, 0.4
PRODUCT, PER_DIM = 0, 1


def _check(key, got, want, scale=None):
    got = torch.as_tensor(got).detach().double().cpu().reshape(-1)
    want = torch.as_tensor(want).detach().double().cpu().reshape(-1)
    assert got.shape == want.shape, (key, got.shape, want.shape)
    assert bool(torch.isfinite(got).all()), key
    zero = want == 0
    assert bool((got[zero] == 0).all()), (key, "nonzero where float64 is exactly 0")
    if scale is None:
        scale = float(want.abs().max())
    err = float((got - want).abs().max()) / scale if scale > 0 else float((got - want).abs().max())
    MEASURED[key] = max(MEASURED.get(key, 0.0), err)
    assert err <= BAR[key], (key, err, BAR[key])
    return err


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if MEASURED:
        print("\nmeasured maxima (error / scale) and bars:\n" + "\n".join(f"  {k:12s} {v:.2e}  bar {BAR[k]:.0e}" for k, v in sorted(MEASURED.items())))


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs CUDA")
    return torch.device("cuda:0")


def _call(name, *args):
    from safepo import _lib as L
    L.check(getattr(L.lib(), name)(*args), name)


def _ptr(t):
    from safepo import _lib as L
    return L.ptr(t)


def _stream():
    from safepo import _lib as L
    return L.stream()


# ======================================================= float64 reference =======================================================
def ref_policy_loss(log_probs, old_log_probs, adv, factor, masks, clip, per_dim):
    """mappo.py:137-147 (per_dim) / happo.py:144-155: returns (policy loss, importance weights).  ``clip``: the clip parameter,
    or the pair (1 - clip, 1 + clip) itself."""
    lo, hi = clip if isinstance(clip, tuple) else (1.0 - clip, 1.0 + clip)
    imp = torch.exp(log_probs - old_log_probs)
    if not per_dim:
        imp = torch.prod(imp, dim=-1, keepdim=True)
    surr1 = imp * adv
    surr2 = torch.clamp(imp, lo, hi) * adv
    inner = torch.min(surr1, surr2) if factor is None else factor * torch.min(surr1, surr2)
    if masks is not None:
        return (-torch.sum(inner, dim=-1, keepdim=True) * masks).sum() / masks.sum(), imp
    return -torch.sum(inner, dim=-1, keepdim=True).mean(), imp


def ref_entropy(dist, masks):
    """act.py:69-72."""
    return dist.entropy().mean() if masks is None else (dist.entropy() * masks).sum() / masks.sum()


def huber(e, d):
    a = (abs(e) <= d).to(e.dtype)
    b = (e > d).to(e.dtype)
    return a * e ** 2 / 2 + b * d * (abs(e) - d / 2)


def ref_value_loss(values, value_preds, ret_c, ret_o, clip, delta, masks):
    """happo.py:106-122 with the two normalised returns given."""
    vpc = value_preds + (values - value_preds).clamp(-clip, clip)
    L = torch.max(huber(ret_o - values, delta), huber(ret_c - vpc, delta))
    return (L * masks).sum() / masks.sum()


# ============================================================ CPU ============================================================
def test_new_entry_points_reject_bad_arguments_before_touching_the_device():
    """Null arguments, unpaired optional arguments, a bad ratio mode and act_dim > 32 return a status and a message."""
    from safepo import _lib as L
    lib, OK, x = L.lib(), 0, 0x1000         # x: a dummy non-null address; nothing is launched on a rejected call
    args = [x, 4, 128, x, x, x, 3, x, x, x, None, None, None, None, None, PRODUCT, 0.8, 1.2, 1.0, 0.5, x, x, x, None]

    def call(**over):
        a = list(args)
        for k, v in over.items():
            a[int(k[1:])] = v
        return lib.spo_ma_ppo_actor_loss(*a)
    assert call(_0=None) != OK and b"spo_ma_ppo_actor_loss" in lib.spo_last_error()
    assert call(_1=0) != OK
    assert call(_10=x) != OK and b"lamda" in lib.spo_last_error()              # cost_adv without lamda
    assert call(_13=x) != OK and b"mask_sum" in lib.spo_last_error()          # masks without their sum
    assert call(_15=2) != OK and b"ratio_mode" in lib.spo_last_error()
    assert call(_6=33) != OK and b"act_dim" in lib.spo_last_error()
    assert call(_6=0) != OK
    assert lib.spo_ma_ppo_actor_finalize(None, 1, 4, None, PRODUCT, x, 3, 1.0, 0.5, 0.01, x, x, x, None) != OK
    assert lib.spo_ma_ppo_actor_finalize(x, 1, 4, None, 5, x, 3, 1.0, 0.5, 0.01, x, x, x, None) != OK
    assert lib.spo_ma_ppo_actor_finalize(x, 2, 4, None, PRODUCT, x, 3, 1.0, 0.5, 0.01, x, x, x, None) != OK and b"nblk" in lib.spo_last_error()
    assert lib.spo_ma_ppo_actor_finalize(x, 1, 4, None, PRODUCT, x, 40, 1.0, 0.5, 0.01, x, x, x, None) != OK
    assert lib.spo_ma_value_loss_masked(x, x, x, x, None, x, 4, 0.2, 10.0, 1.0, x, x, None) != OK
    assert b"spo_ma_value_loss_masked" in lib.spo_last_error()
    assert lib.spo_ma_value_loss_masked(x, x, x, x, x, x, 0, 0.2, 10.0, 1.0, x, x, None) != OK


def test_synthetic_env_lone_finishes_are_opt_in():
    """agent_done_prob = 0 draws exactly the old stream (the same generator calls in the same order); > 0 lets agents finish alone."""
    from safepo.common.synthetic_env import SyntheticMultiAgentEnv
    acts = [torch.zeros(5, 2), torch.zeros(5, 2)]
    e0 = SyntheticMultiAgentEnv(5, 2, 3, 4, 2, episode_len=3, seed=9, device="cpu")
    g = torch.Generator().manual_seed(9)
    obs, share, _ = e0.reset()
    assert torch.equal(obs, torch.randn(5, 2, 3, generator=g)) and torch.equal(share, torch.randn(5, 2, 4, generator=g))
    for t in range(1, 7):
        o, s, r, c, d, _, _ = e0.step(acts)
        assert torch.equal(o, torch.randn(5, 2, 3, generator=g)) and torch.equal(s, torch.randn(5, 2, 4, generator=g))
        assert torch.equal(r, 0.01 * torch.randn(5, 2, 1, generator=g))
        assert torch.equal(c, (torch.rand(5, 2, 1, generator=g) < 0.05).float())
        assert bool((d == (t % 3 == 0)).all())
    e1 = SyntheticMultiAgentEnv(64, 2, 3, 4, 2, episode_len=100, seed=9, device="cpu", agent_done_prob=0.2)
    e1.reset()
    lone = 0
    for _ in range(5):
        d = e1.step([torch.zeros(64, 2)] * 2)[4]
        lone += int((d.any(1) & ~d.all(1)).sum())
    assert lone > 10


def _two_net_states(g, D, DS, A, H, layer_N=2):
    return MA_state(g, D, H, A, "actor", layer_N), MA_state(g, DS, H, A, "critic", layer_N)


def MA_state(g, din, H, A, head, layer_N=2):
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


BASE_CFG = dict(actor_lr=9e-5, critic_lr=5e-3, opti_eps=1e-5, weight_decay=0.0, clip_param=0.2, huber_delta=10.0, entropy_coef=0.0,
                max_grad_norm=10.0, value_loss_coef=1.0, learning_iters=2, gamma=0.96, gae_lambda=0.95, layer_N=2, std_x_coef=1.0,
                std_y_coef=0.5, use_policy_active_masks=False, use_value_active_masks=False)
MASKED = dict(use_policy_active_masks=True, use_value_active_masks=True, entropy_coef=0.01)


def _update_sample(g, N, D, DS, A, oa, oc, cfg, inactive=0.2):
    """A whole-batch sample with inactive rows whose importance weights fall on every side of the clip range per dimension."""
    obs, share = torch.randn(N, D, generator=g) * 2 + 0.5, torch.randn(N, DS, generator=g) * 3
    with torch.no_grad():
        dist = MA.ma_actor_dist(oa, obs, cfg["std_x_coef"], cfg["std_y_coef"])
        actions = dist.mean + dist.stddev * torch.randn(N, A, generator=g)
        logp = dist.log_prob(actions)
        v0 = MA.ma_critic_value(oc, share)
    return dict(share_obs=share, obs=obs, actions=actions, value_preds=v0 + 0.1 * torch.randn(N, 1, generator=g),
                returns=torch.randn(N, 1, generator=g) * 4 + 1, old_action_log_probs=logp + 0.3 * torch.randn(N, A, generator=g),
                adv_targ=torch.randn(N, 1, generator=g), factor=torch.rand(N, 1, generator=g) + 0.5,
                active_masks=(torch.rand(N, 1, generator=g) >= inactive).float())


ALGOS = {"mappo": ("MAPPOTrainer", PO.OracleMAPPOTrainer), "happo": ("HAPPOTrainer", PO.OracleHAPPOTrainer)}


def _compare_update(algo, cfg, N, D, DS, A, H, dev, seed, rtol, atol, gtol, names_only=False):
    """Two consecutive ppo_update calls through the package's trainer and the oracle; returns the worst gradient error."""
    from safepo.common import ma_model
    g = torch.Generator().manual_seed(seed)
    sa, sc = _two_net_states(g, D, DS, A, H, cfg["layer_N"])
    oa, oc = MA.OracleMANet(sa, cfg["layer_N"]), MA.OracleMANet(sc, cfg["layer_N"])
    sample = _update_sample(g, N, D, DS, A, oa, oc, cfg)
    otr = ALGOS[algo][1](oa, oc, cfg)
    nets = ma_model.MultiAgentNets(sa, sc, None, dev, layer_N=cfg["layer_N"], std_x_coef=cfg["std_x_coef"], std_y_coef=cfg["std_y_coef"])
    tr = getattr(ma_model, ALGOS[algo][0])(nets, cfg)
    names = ("value_loss", "critic_grad_norm", "policy_loss", "dist_entropy", "actor_grad_norm", "imp_weights")
    worst = 0.0
    for it in range(2):
        want = otr.ppo_update(sample)
        ds = dict(sample) if it == 0 else tuple(sample.get(k) for k in ma_model._PPO_SAMPLE_KEYS)      # the reference's 13-tuple too
        got = dict(zip(names, tr.ppo_update(ds)))
        slack = 1.0 if it == 0 else 10.0
        for k in names:
            gv, wv = got[k].detach().cpu().reshape(-1).double(), want[k].reshape(-1).double()
            assert gv.shape == wv.shape, (k, gv.shape, wv.shape)
            err = float((gv - wv).abs().max())
            assert err <= (rtol * float(wv.abs().max()) + atol) * slack, (algo, it, k, err, float(wv.abs().max()))
        assert float(tr.last_ratio) == pytest.approx(float(want["imp_weights"].mean()), rel=rtol * slack, abs=atol * slack)
        for net, onet, nk in ((nets.actor, oa, "actor_grad_norm"), (nets.critic, oc, "critic_grad_norm")):
            coef = min(1.0, float(cfg["max_grad_norm"]) / (float(want[nk]) + 1e-6))
            for k, pt in onet.p.items():
                wg = pt.grad / coef
                err = float((net.g[k].cpu() - wg).abs().max())
                scale = float(wg.abs().max())
                worst = max(worst, err / (scale + 1e-12))
                assert err <= (gtol * scale + 1e-7) * slack, (algo, it, k, err, scale)
        pst = tr.popart_state.cpu()
        for got_s, want_s in zip(pst, (otr.popart.running_mean, otr.popart.running_mean_sq, otr.popart.debiasing_term)):
            assert abs(float(got_s) - float(want_s)) <= 1e-5 * abs(float(want_s)) + 1e-12
        for net, onet, lr in ((nets.actor, oa, cfg["actor_lr"]), (nets.critic, oc, cfg["critic_lr"])):
            for k, pt in onet.p.items():
                err = float((net.p[k].cpu() - pt.detach()).abs().max())
                assert err < 0.05 * lr + 1e-6, (algo, it, k, err, lr)
    return worst


@pytest.mark.parametrize("algo", ["mappo", "happo"])
@pytest.mark.parametrize("masked", [False, True], ids=["defaults", "mamujoco_flags"])
def test_trainer_host_path_through_emulated_abi_vs_oracle(monkeypatch, algo, masked):
    """MAPPOTrainer / HAPPOTrainer.ppo_update host logic (which buffer goes where, the masked critic call, the partial layouts,
    the 13-tuple) through the emulated C-ABI against the oracle: two consecutive updates, flags on and off."""
    import ppo_emulator
    ppo_emulator.install(monkeypatch)
    cfg = dict(BASE_CFG, **(MASKED if masked else {}))
    _compare_update(algo, cfg, 96, 6, 8, 3, 16, "cpu", 11 + masked, rtol=2e-5, atol=1e-6, gtol=5e-5)


def _runner_pair(algo, cfg, T, N, D, DS, A, H, NA, dev, seed):
    from safepo.common.ma_model import MultiAgentNets
    from safepo.multi_agent import happo, mappo
    g = torch.Generator().manual_seed(seed)
    states = [_two_net_states(g, D, DS, A, H, cfg["layer_N"]) for _ in range(NA)]
    onets = [(MA.OracleMANet(a, cfg["layer_N"]), MA.OracleMANet(c, cfg["layer_N"])) for a, c in states]
    orun = PO.OracleTwoNetRunner(onets, cfg, T, N, D, DS, A, ALGOS[algo][1])
    nets = [MultiAgentNets(a, c, None, dev, layer_N=cfg["layer_N"], std_x_coef=cfg["std_x_coef"], std_y_coef=cfg["std_y_coef"]) for a, c in states]
    run = {"mappo": mappo, "happo": happo}[algo].Runner(nets, dict(cfg, episode_length=T, n_rollout_threads=N), D, DS, A)
    return orun, run, onets, g


def _run_iterations(orun, run, g, T, N, D, DS, A, NA, dev, iters=2):
    """Two whole iterations on the same inputs (the same eps, agent order and row orders): agent 1 of env 0 finishes alone at
    step 1, every agent of env 1 at step 2.  Returns the per-iteration outputs of both."""
    obs, share = torch.randn(N, NA, D, generator=g), torch.randn(N, NA, DS, generator=g)
    orun.warmup(obs, share)
    run.warmup(obs.to(dev), share.to(dev))
    outs = []
    for it in range(iters):
        for step in range(T):
            eps = [torch.randn(N, A, generator=g) for _ in range(NA)]
            ov, oact, olp = orun.collect(step, eps)
            v, act, lp, cp = run.collect(step, [e.to(dev) for e in eps])
            assert cp is None
            for a in range(NA):
                assert float((act[a].cpu() - oact[a]).abs().max()) < 1e-4
            obs, share = torch.randn(N, NA, D, generator=g), torch.randn(N, NA, DS, generator=g)
            rew = 0.1 * torch.randn(N, NA, 1, generator=g)
            dones = torch.zeros(N, NA, dtype=torch.bool)
            if step == 1:
                dones[0, 1] = True
            if step == 2:
                dones[1, :] = True
            orun.insert(obs, share, rew, dones, ov, oact, olp)
            # the device runner stores its own actions / log-probs (equal to the oracle's to fp32 noise, checked above)
            run.insert(obs.to(dev), share.to(dev), rew.to(dev), torch.zeros(N, NA, 1, device=dev), dones.to(dev), v, act, lp, None)
        orun.compute()
        run.compute()
        order = torch.randperm(NA, generator=g).tolist()
        perms = {a: [torch.randperm(T * N, generator=g) for _ in range(orun.cfg["learning_iters"])] for a in range(NA)}
        want = orun.train(order, perms)
        got = run.train(order, {a: [p.to(dev) for p in ps] for a, ps in perms.items()}, collect_outputs=True)
        outs.append((got, want))
    return outs


@pytest.mark.parametrize("algo", ["mappo", "happo"])
def test_runner_host_path_through_emulated_abi_vs_oracle(monkeypatch, algo):
    """Two runner iterations of two agents (collect / insert / compute / train with the cross-agent factor) through the emulated
    C-ABI against the oracle runner, masks on, an agent finishing alone."""
    import ppo_emulator
    ppo_emulator.install(monkeypatch)
    cfg = dict(BASE_CFG, **MASKED)
    T, N, D, DS, A, H, NA = 4, 6, 10, 14, 3, 16, 2
    orun, run, onets, g = _runner_pair(algo, cfg, T, N, D, DS, A, H, NA, "cpu", 5)
    for got, want in _run_iterations(orun, run, g, T, N, D, DS, A, NA, "cpu"):
        for a in range(NA):
            for gv, wk in zip(got[a], ("value_loss", "critic_grad_norm", "policy_loss", "dist_entropy", "actor_grad_norm", "imp_weights")):
                wv = want[a][wk]
                assert torch.allclose(gv.reshape(-1).double(), wv.reshape(-1).double(), rtol=1e-3, atol=1e-5), (a, wk)
    assert float(run.buffer[1].active_masks.min()) == 0.0         # agent 1 of env 0 finished alone
    for a in range(NA):
        for k, pt in onets[a][0].p.items():
            assert torch.allclose(run.nets[a].actor.p[k], pt.detach(), rtol=1e-4, atol=1e-6), (a, k)


# ============================================================ GPU: kernels ============================================================
def _actor_case(g, n, A, H, clip, with_masks, zero_mask_rows=True):
    """Head inputs whose per-dimension ratios lie below / inside / above the clip range with a margin, or exactly on its bounds,
    for both advantage signs; masks with zero rows."""
    feat = torch.randn(n, H, generator=g)
    W, b = torch.randn(A, H, generator=g) * 0.05, 0.1 * torch.randn(A, generator=g)
    ls = 0.5 * torch.randn(A, generator=g)
    with torch.no_grad():
        mean64 = F.linear(feat.double(), W.double(), b.double())
        dist = Normal(mean64, torch.sigmoid(ls.double() / X_COEF) * Y_COEF)
        actions = (dist.mean + dist.stddev * torch.randn(n, A, generator=g, dtype=torch.float64)).float()
        lp32 = Normal(F.linear(feat, W, b), torch.sigmoid(ls / X_COEF) * Y_COEF).log_prob(actions)
        lp64 = dist.log_prob(actions.double())
    lo, hi = 1 - clip, 1 + clip
    # per dimension: region 0 below, 1 inside, 2 above, 3 on a bound (old = logp exactly: ratio 1 -- the bounds themselves come
    # from clip = 0 in the bound test); the product mode sees the row product
    region = (torch.arange(n)[:, None] + torch.arange(A)[None, :]) % 3
    u = torch.rand(n, A, generator=g, dtype=torch.float64)
    target = torch.where(region == 0, lo - 0.25 + 0.2 * u, torch.where(region == 1, lo + 0.05 + (hi - lo - 0.1) * u, hi + 0.05 + 0.3 * u))
    old = (lp64 - torch.log(target)).float()
    adv = torch.where(torch.arange(n) % 2 == 0, 1.0, -1.0) * (0.3 + torch.rand(n, generator=g))
    factor = torch.rand(n, generator=g) + 0.5
    masks = (torch.rand(n, generator=g) >= 0.3).float() if with_masks else None
    if with_masks:
        masks[-1] = 1.0                                      # at least one active row (the all-inactive case has its own test)
        if zero_mask_rows and n > 1:
            masks[0] = 0.0
    return feat, W, b, ls, actions, old, adv, factor, masks, region, lp32


def _run_actor(dev, feat, W, b, ls, actions, old, adv, factor, masks, mode, clip, ec, cost_adv=None, lam=None):
    n, H = feat.shape
    A = W.shape[0]
    t = [x.to(dev).contiguous() if x is not None else None for x in (feat, W, b, ls, actions, old, adv, factor, masks, cost_adv)]
    msum = t[8].sum().reshape(1) if masks is not None else None
    lamd = torch.tensor([lam], device=dev) if lam is not None else None
    nb = (n + 31) // 32
    dmean, imp, part = torch.empty(n, A, device=dev), torch.empty(n * (A if mode == PER_DIM else 1), device=dev), torch.empty(nb * 66, device=dev)
    lo, hi = clip if isinstance(clip, tuple) else (1.0 - clip, 1.0 + clip)
    _call("spo_ma_ppo_actor_loss", _ptr(t[0]), n, H, _ptr(t[1]), _ptr(t[2]), _ptr(t[3]), A, _ptr(t[4]), _ptr(t[5]), _ptr(t[6]), _ptr(t[9]),
          _ptr(lamd), _ptr(t[7]), _ptr(t[8]), _ptr(msum), mode, lo, hi, X_COEF, Y_COEF, _ptr(dmean), _ptr(imp), _ptr(part), _stream())
    gb, gls, scal = torch.empty(A, device=dev), torch.empty(A, device=dev), torch.empty(3, device=dev)
    _call("spo_ma_ppo_actor_finalize", _ptr(part), nb, n, _ptr(msum), mode, _ptr(t[3]), A, X_COEF, Y_COEF, ec, _ptr(gb), _ptr(gls), _ptr(scal),
          _stream())
    torch.cuda.synchronize()
    return dmean.cpu(), imp.cpu(), part.cpu(), gb.cpu(), gls.cpu(), scal.cpu()


def _ref_actor(feat, W, b, ls, actions, old, adv, factor, masks, mode, clip, ec):
    mean = F.linear(feat.double(), W.double(), b.double()).requires_grad_(True)
    ls64 = ls.double().requires_grad_(True)
    dist = Normal(mean, torch.sigmoid(ls64 / X_COEF) * Y_COEF)
    m = None if masks is None else masks.double()[:, None]
    pl, imp = ref_policy_loss(dist.log_prob(actions.double()), old.double(), adv.double()[:, None],
                              None if factor is None else factor.double()[:, None], m, clip, mode == PER_DIM)
    ent = ref_entropy(dist, m)
    (dm,) = torch.autograd.grad(pl, mean, retain_graph=True)
    (gls,) = torch.autograd.grad(pl - ent * ec, ls64)
    return pl.detach(), imp.detach(), ent.detach(), dm, gls


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [PRODUCT, PER_DIM], ids=["product", "per_dim"])
@pytest.mark.parametrize("A", [1, 20, 32])
@pytest.mark.parametrize("with_masks", [False, True], ids=["no_masks", "masks"])
def test_ppo_actor_loss_vs_float64(mode, A, with_masks):
    """spo_ma_ppo_actor_loss + finalize: dmean, importance weights, g_b, g_log_std (entropy term included; masked: sum_j e_j and its
    A-fold gradient), policy loss, entropy and mean ratio at n in {1, 33, 4097}; HAPPO's factor in product mode, MAPPO's none per
    dimension; per-dimension clip branches counted."""
    dev = _cuda()
    g = torch.Generator().manual_seed(700 + 10 * A + mode + 2 * with_masks)
    clip, ec, H = 0.2, 0.013, 256
    for n in (1, 33, 4097):
        feat, W, b, ls, actions, old, adv, factor, masks, region, _ = _actor_case(g, n, A, H, clip, with_masks)
        if mode == PER_DIM:
            factor = None
        dmean, imp, _, gb, gls, scal = _run_actor(dev, feat, W, b, ls, actions, old, adv, factor, masks, mode, clip, ec)
        pl, imp64, ent, dm64, gls64 = _ref_actor(feat, W, b, ls, actions, old, adv, factor, masks, mode, clip, ec)
        cat = lambda t: (t < 1 - clip).int() + 2 * (t > 1 + clip).int()      # noqa: E731
        assert torch.equal(cat(imp.double().reshape(imp64.shape)), cat(imp64))
        if mode == PER_DIM:
            assert torch.equal(cat(imp64), torch.tensor([1, 0, 2], dtype=torch.int32)[region])
            if n == 4097:
                for reg in (0, 1, 2):         # row x dimension count of each branch, for both advantage signs
                    for sgn in (adv > 0, adv < 0):
                        assert int(((region == reg) & sgn[:, None]).sum()) >= n * A // 8, (reg, n, A)
        if masks is not None and n > 1:
            assert int((masks == 0).sum()) >= 1
        _check("actor", dmean, dm64)
        _check("actor", imp, imp64)
        _check("actor", gb, dm64.sum(0))
        _check("actor", gls, gls64)
        terms = (imp64 * adv.double()[:, None]).abs()
        _check("actor_loss", scal[0:1], pl.reshape(1), scale=float(terms.mean()) * (A if mode == PER_DIM else 1) + 1e-30)
        _check("actor_loss", scal[1:2], ent.reshape(1))
        _check("actor_loss", scal[2:3], imp64.mean().reshape(1))


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [PRODUCT, PER_DIM], ids=["product", "per_dim"])
def test_ppo_actor_loss_exactly_on_the_clip_bounds(mode):
    """Every importance weight (every row x dimension per dimension) exactly on the lower, then on the upper clip bound, for both
    advantage signs: clamp's backward passes the gradient there and torch.min's tie gives the same total, the full gradient of
    imp * adv.  Equal inputs in every row and dimension (mean 0 from zero head weights) make all ratios one fp32 value r; the
    bounds are then set to r (the float64 side to its own r)."""
    dev = _cuda()
    g = torch.Generator().manual_seed(91 + mode)
    n, A, H = 33, 20, 128
    feat, W, b = torch.randn(n, H, generator=g), torch.zeros(A, H), torch.zeros(A)
    ls, actions, old = torch.full((A,), 0.4), torch.full((n, A), 0.3), torch.full((n, A), -0.2)
    adv = torch.where(torch.arange(n) % 2 == 0, 1.0, -1.0) * (0.3 + torch.rand(n, generator=g))
    factor = torch.rand(n, generator=g) + 0.5
    _, imp, _, _, _, _ = _run_actor(dev, feat, W, b, ls, actions, old, adv, factor, None, mode, (0.0, 100.0), 0.0)
    r = float(imp[0])
    assert bool((imp == r).all())
    _, imp64, _, _, _ = _ref_actor(feat, W, b, ls, actions, old, adv, factor, None, mode, (0.0, 100.0), 0.0)
    r64 = float(imp64[0, 0])
    for side, (lo, hi), (lo64, hi64) in (("low", (r, r + 0.1), (r64, r64 + 0.1)), ("high", (r - 0.1, r), (r64 - 0.1, r64))):
        dmean, imp, _, gb, gls, scal = _run_actor(dev, feat, W, b, ls, actions, old, adv, factor, None, mode, (lo, hi), 0.0)
        on = int((imp == (lo if side == "low" else hi)).sum())
        assert on == n * (A if mode == PER_DIM else 1), (side, on)
        pl, _, ent, dm64, gls64 = _ref_actor(feat, W, b, ls, actions, old, adv, factor, None, mode, (lo64, hi64), 0.0)
        full = _ref_actor(feat, W, b, ls, actions, old, adv, factor, None, mode, (0.0, 100.0), 0.0)[3]
        assert torch.equal(dm64, full)                   # on the bound the float64 gradient is the unclipped one
        _check("actor", dmean, dm64)
        _check("actor", gb, dm64.sum(0))
        _check("actor", gls, gls64)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [PRODUCT, PER_DIM], ids=["product", "per_dim"])
def test_ppo_actor_loss_all_rows_inactive_is_nan(mode):
    """sum m = 0: the reference divides 0 by 0, so the loss, the entropy and the gradients are NaN -- not a silent 0."""
    dev = _cuda()
    g = torch.Generator().manual_seed(5)
    feat, W, b, ls, actions, old, adv, factor, masks, _, _ = _actor_case(g, 40, 3, 128, 0.2, True)
    masks.zero_()
    dmean, imp, _, gb, gls, scal = _run_actor(dev, feat, W, b, ls, actions, old, adv, factor, masks, mode, 0.2, 0.01)
    assert bool(torch.isnan(scal[0])) and bool(torch.isnan(scal[1])) and bool(torch.isnan(gls).all()) and bool(torch.isnan(gb).all())
    assert bool(torch.isfinite(scal[2]))                     # the logged mean ratio is unmasked, as imp_weights.mean()
    pl, _, ent, _, _ = _ref_actor(feat, W, b, ls, actions, old, adv, factor, masks, mode, 0.2, 0.01)
    assert bool(torch.isnan(pl)) and bool(torch.isnan(ent))


@pytest.mark.gpu
@pytest.mark.parametrize("A", [1, 20, 32])
def test_ppo_actor_loss_equals_mappolag_kernel_bit_for_bit(A):
    """Product ratio, factor, lambda and no masks is MAPPO-Lag's configuration: dmean, the importance weights, the partials,
    g_b, g_log_std, the policy loss and the entropy equal spo_ma_actor_loss + spo_ma_actor_finalize bit for bit."""
    dev = _cuda()
    g = torch.Generator().manual_seed(33 + A)
    clip, ec, lam = 0.2, 0.01, 0.78
    for n in (1, 33, 4097):
        feat, W, b, ls, actions, old, adv, factor, _, _, _ = _actor_case(g, n, A, 512, clip, False)
        cadv = torch.randn(n, generator=g)
        dmean, imp, part, gb, gls, scal = _run_actor(dev, feat, W, b, ls, actions, old, adv, factor, None, PRODUCT, clip, ec, cadv, lam)
        t = [x.to(dev).contiguous() for x in (feat, W, b, ls, actions, old, adv, cadv, factor)]
        lamd = torch.tensor([lam], device=dev)
        nb = (n + 31) // 32
        dm2, imp2, part2 = torch.empty(n, A, device=dev), torch.empty(n, device=dev), torch.empty(nb * 66, device=dev)
        _call("spo_ma_actor_loss", _ptr(t[0]), n, 512, _ptr(t[1]), _ptr(t[2]), _ptr(t[3]), A, _ptr(t[4]), _ptr(t[5]), _ptr(t[6]), _ptr(t[7]),
              _ptr(t[8]), _ptr(lamd), 1.0 - clip, 1.0 + clip, X_COEF, Y_COEF, _ptr(dm2), _ptr(imp2), _ptr(part2), _stream())
        gb2, gls2, sc2 = torch.empty(A, device=dev), torch.empty(A, device=dev), torch.empty(2, device=dev)
        _call("spo_ma_actor_finalize", _ptr(part2), nb, n, _ptr(t[3]), A, X_COEF, Y_COEF, ec, _ptr(gb2), _ptr(gls2), _ptr(sc2), _stream())
        torch.cuda.synchronize()
        p2 = part2.cpu().view(nb, 66)
        p1 = part.view(nb, 66)
        assert torch.equal(dmean, dm2.cpu()) and torch.equal(imp, imp2.cpu())
        assert torch.equal(p1[:, 0], p2[:, 0]) and torch.equal(p1[:, 2:], p2[:, 2:])
        assert torch.equal(gb, gb2.cpu()) and torch.equal(gls, gls2.cpu()) and torch.equal(scal[:2], sc2.cpu())


def _value_case(g, n):
    """Exactly representable rows (multiples of 1/8): the value clip on both sides and at +-clip, every Huber piece, ties."""
    dlts = torch.tensor([-0.75, -0.25, -0.125, 0.0, 0.125, 0.25, 0.75], dtype=torch.float64)
    errs = torch.tensor([-3.0, -2.5, -2.0, -1.5, -0.5, 0.0, 0.5, 1.5, 2.0, 2.5, 3.0], dtype=torch.float64)
    dlt = dlts[torch.randint(0, 7, (n,), generator=g)]
    ec, eo = errs[torch.randint(0, 11, (n,), generator=g)], errs[torch.randint(0, 11, (n,), generator=g)]
    vp = torch.randint(-8, 9, (n,), generator=g).double() / 8
    v = vp + dlt
    return v, vp, vp + dlt.clamp(-0.25, 0.25) + ec, v + eo


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 33, 4097])
def test_value_loss_masked_vs_float64(n):
    """spo_ma_value_loss_masked: dv, its sum and the loss of (max(huber(eo), huber(ec)) * m).sum() / m.sum() times
    value_loss_coef, masks with zero rows; all rows inactive gives NaN."""
    dev = _cuda()
    g = torch.Generator().manual_seed(n)
    clip, d, coef = 0.25, 2.0, 0.7
    v, vp, rn_c, rn_o = _value_case(g, n)
    m = (torch.rand(n, generator=g) >= 0.3).double()
    m[-1] = 1.0
    if n > 1:
        m[0] = 0.0
    for masks in (m, torch.zeros(n, dtype=torch.float64)):
        ins = [t.float().to(dev) for t in (v, vp, rn_c, rn_o, masks)]
        msum = ins[4].sum().reshape(1)
        nb = (n + 255) // 256
        dv, part = torch.empty(n, device=dev), torch.empty(nb * 2, device=dev)
        _call("spo_ma_value_loss_masked", *[_ptr(t) for t in ins], _ptr(msum), n, clip, d, coef, _ptr(dv), _ptr(part), _stream())
        torch.cuda.synchronize()
        tot = part.cpu().view(nb, 2).sum(0)
        if float(masks.sum()) == 0:
            assert bool(torch.isnan(tot[0])) and bool(torch.isnan(dv.cpu()).all())
            continue
        v64 = v.clone().requires_grad_(True)
        L = ref_value_loss(v64, vp, rn_c, rn_o, clip, d, masks)
        (dv64,) = torch.autograd.grad(L * coef, v64)
        _check("value", dv.cpu(), dv64)
        _check("value", tot[1:2], dv64.sum().reshape(1), scale=float(dv64.abs().sum()) + 1e-30)
        _check("value", tot[0:1], L.detach().reshape(1))


# ============================================================ GPU: whole steps ============================================================
SHAPES = [(300, 10, 14, 3, 128), (777, 66, 130, 32, 256), (2048, 398, 398, 20, 512)]


@pytest.mark.gpu
@pytest.mark.parametrize("algo", ["mappo", "happo"])
@pytest.mark.parametrize("masked", [False, True], ids=["defaults", "mamujoco_flags"])
@pytest.mark.parametrize("shape", SHAPES, ids=[f"n{s[0]}_obs{s[1]}_act{s[3]}_h{s[4]}" for s in SHAPES])
def test_trainer_ppo_update_vs_oracle(algo, masked, shape):
    """Two consecutive MAPPOTrainer / HAPPOTrainer.ppo_update calls against OracleMAPPOTrainer / OracleHAPPOTrainer: every
    tensor's gradient before the clip, the six returned values (imp_weights [n, A] or [n, 1]), the PopArt state and all weights,
    on a sample with inactive rows; the last shape is config 5's layers (obs 398, act 20, hidden 512)."""
    dev = _cuda()
    N, D, DS, A, H = shape
    cfg = {**BASE_CFG, "entropy_coef": 0.01, **(MASKED if masked else {})}
    worst = _compare_update(algo, cfg, N, D, DS, A, H, dev, 3 * N + D + masked, rtol=1e-4, atol=2e-6, gtol=5e-5)
    print(f"\n{algo} ppo_update {shape} masks={masked}: worst relative gradient error per tensor {worst:.2e}")


@pytest.mark.gpu
@pytest.mark.parametrize("algo", ["mappo", "happo"])
def test_runner_iteration_vs_oracle(algo):
    """Two iterations of two agents through mappo.Runner / happo.Runner against the oracle runner, masks on, an agent finishing
    alone: returned values, the factor each agent saw and the weights after the iteration."""
    dev = _cuda()
    cfg = dict(BASE_CFG, **MASKED)
    T, N, D, DS, A, H, NA = 5, 64, 18, 36, 3, 128, 2
    orun, run, onets, g = _runner_pair(algo, cfg, T, N, D, DS, A, H, NA, dev, 21)
    for got, want in _run_iterations(orun, run, g, T, N, D, DS, A, NA, dev):
        for a in range(NA):
            for gv, wk in zip(got[a], ("value_loss", "critic_grad_norm", "policy_loss", "dist_entropy", "actor_grad_norm", "imp_weights")):
                wv = want[a][wk].reshape(-1).double()
                err = float((gv.detach().cpu().reshape(-1).double() - wv).abs().max())
                assert err <= 1e-3 * float(wv.abs().max()) + 1e-5, (a, wk, err)
    for a in range(NA):
        assert float(run.buffer[a].active_masks.min()) == 0.0 or a == 0
        assert torch.allclose(run.buffer[a].factor.cpu(), orun.buffer[a].factor, rtol=1e-3, atol=1e-6)
        for k, pt in onets[a][0].p.items():
            assert float((run.nets[a].actor.p[k].cpu() - pt.detach()).abs().max()) < 0.05 * cfg["actor_lr"] + 1e-6, (a, k)


@pytest.mark.gpu
@pytest.mark.parametrize("algo", ["mappo", "happo"])
@pytest.mark.parametrize("mamujoco", [False, True], ids=["yaml", "mamujoco"])
def test_cli_synthetic(algo, mamujoco, tmp_path):
    """`python -m safepo.multi_agent.{mappo,happo} --env synthetic --iterations 2 --num-envs 64 --hidden-size 128 [--mamujoco]`
    writes finite log rows with the reference's columns (agents finishing alone, so the masks are live)."""
    _cuda()
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "safe-policy-optimization_b200")]))
    cmd = [sys.executable, "-m", f"safepo.multi_agent.{algo}", "--env", "synthetic", "--iterations", "2", "--num-envs", "64",
           "--hidden-size", "128", "--obs-dim", "18", "--share-obs-dim", "36", "--act-dim", "3", "--agent-done-prob", "0.01",
           "--episode-len", "7", "--log-dir", str(tmp_path)] + (["--mamujoco"] if mamujoco else [])
    out = subprocess.run(cmd, capture_output=True, text=True, env=env, timeout=900)
    assert out.returncode == 0, out.stderr[-3000:]
    import csv
    rows = list(csv.DictReader(open(tmp_path / "progress.csv")))
    assert len(rows) == 2
    for col in ("Loss/Loss_reward_critic", "Loss/Loss_actor", "Misc/Reward_critic_norm", "Misc/Entropy", "Misc/Ratio"):
        for a in range(2):
            vals = [float(r[f"{col}/agent{a}"]) for r in rows]
            assert all(math.isfinite(x) for x in vals), (col, vals)


# ============================================================ CPU: the fixture ============================================================
def _single_thread():
    threads = torch.get_num_threads()
    torch.set_num_threads(1)        # the fixture was written with one intra-op thread (LayerNorm's backward reductions)
    return threads


@pytest.mark.parametrize("algo", ["mappo", "happo"])
@pytest.mark.parametrize("flags", ["defaults", "mamujoco"])
def test_oracle_trainer_matches_reference_fixture_bit_for_bit(golden, algo, flags):
    """OracleMAPPOTrainer / OracleHAPPOTrainer replay the reference's two consecutive ppo_update calls of mappo.pt exactly: every
    returned value, the PopArt state and both state dicts, at the yaml's defaults and with the mamujoco mask flags."""
    fx = golden("mappo")["updates"]["cases"][(algo, flags)]
    threads = _single_thread()
    try:
        cfg = dict(fx["cfg"])
        oa, oc = MA.OracleMANet(fx["init"]["actor"], cfg["layer_N"]), MA.OracleMANet(fx["init"]["critic"], cfg["layer_N"])
        tr = ALGOS[algo][1](oa, oc, cfg)
        for call in fx["calls"]:
            out = tr.ppo_update(fx["sample"])
            for k, v in call["out"].items():
                assert torch.equal(torch.as_tensor(out[k]), torch.as_tensor(v)), (algo, flags, k)
            for got_s, want_s in zip((tr.popart.running_mean, tr.popart.running_mean_sq, tr.popart.debiasing_term), call["popart"]):
                assert torch.equal(got_s, want_s)
            for net, name in ((oa, "actor"), (oc, "critic")):
                for k, v in call["state"][name].items():
                    assert torch.equal(net.p[k].detach(), v), (algo, flags, name, k)
        if flags == "mamujoco":
            am = fx["sample"]["active_masks"]
            assert 0 < int((am == 0).sum()) < am.numel()
    finally:
        torch.set_num_threads(threads)


@pytest.mark.parametrize("algo", ["mappo", "happo"])
def test_oracle_runner_matches_reference_fixture_bit_for_bit(golden, algo):
    """OracleTwoNetRunner replays the reference Runner's two iterations of mappo.pt exactly (same global-RNG draws): actions,
    log-probs, values, returns, masks, the factor, the PopArt state and every state dict, with an agent finishing alone."""
    fx = golden("mappo")["epochs"]
    T, N, D, DS, A, H, NA = fx["dims"]
    run = fx["runs"][algo]
    threads = _single_thread()
    try:
        cfg = dict(run["cfg"])
        nets = [(MA.OracleMANet(s["actor"], cfg["layer_N"]), MA.OracleMANet(s["critic"], cfg["layer_N"])) for s in run["init"]]
        orun = PO.OracleTwoNetRunner(nets, cfg, T, N, D, DS, A, ALGOS[algo][1])
        orun.warmup(run["obs0"], run["share_obs0"])
        torch.manual_seed(run["seed"])
        for steps, it in zip(run["stream"], run["iters"]):
            for step, st in enumerate(steps):
                values, actions, logps = orun.collect(step)
                assert torch.equal(values, st["values"])
                assert all(torch.equal(x, y) for x, y in zip(actions, st["actions"]))
                assert all(torch.equal(x, y) for x, y in zip(logps, st["action_log_probs"]))
                orun.insert(st["obs"], st["share_obs"], st["rewards"], st["dones"], values, actions, logps)
            orun.compute()
            for b, want in zip(orun.buffer, it["after_compute"]):
                for k in ("returns", "value_preds", "masks", "active_masks"):
                    assert torch.equal(getattr(b, k), want[k]), k
            orun.train()
            for a, want in enumerate(it["agents"]):
                tr = orun.trainer[a]
                assert torch.equal(orun.buffer[a].factor, want["factor"])
                for got_s, want_s in zip((tr.popart.running_mean, tr.popart.running_mean_sq, tr.popart.debiasing_term), want["popart"]):
                    assert torch.equal(got_s, want_s)
                for net, name in zip(nets[a], ("actor", "critic")):
                    for k, v in want["state"][name].items():
                        assert torch.equal(net.p[k].detach(), v), (a, name, k)
        assert float(run["iters"][0]["after_compute"][1]["active_masks"].min()) == 0.0      # agent 1 finished alone
    finally:
        torch.set_num_threads(threads)


def test_mappo_fixture_regenerates_identically(tmp_path):
    """make_mappo_golden.py writes the committed mappo.pt byte for byte (only where the reference is checked out)."""
    gen = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "make_mappo_golden.py")
    sys.path.insert(0, os.path.dirname(gen))
    import make_golden
    if not os.path.isdir(make_golden.REF):
        pytest.skip("the reference checkout is not present")
    out = tmp_path / "mappo.pt"
    r = subprocess.run([sys.executable, gen, str(out)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    with open(out, "rb") as f1, open(os.path.join(os.path.dirname(gen), "mappo.pt"), "rb") as f2:
        assert f1.read() == f2.read()
