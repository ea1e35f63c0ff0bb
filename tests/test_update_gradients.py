"""Per-tensor gradients of the minibatch update (spo_pg_update) and of the trust-region kernels against float64.

The update kernel writes its Adam moments back for every parameter, and Adam's first moment is
``m = fmaf(1 - beta1, g - m, m)``.  With beta1 = 0, zeroed moments and lr = 0 for all three nets, one step
leaves ``adam_m`` equal to the step's clipped gradient bit for bit and the weights unchanged, so the gradient of
every parameter tensor can be compared with float64 autograd of the same loss.  With lr = 0 a K-step launch
evaluates every step at the initial weights, so m and v after it are float64-computable EMAs of the per-step
gradients.  With betas (0, 0) and adam_eps far above |g| each step is nearly SGD, and the weights after a
K-step launch respond linearly to gradient errors.

The float64 reference (``ref_step``) restates the five loss kinds with their hyperparameters as arguments; in
float32, at the reference's hyperparameters, it reproduces oracle/spo_oracle.py bit for bit (CPU tests below),
and so inherits the oracle's pin to the reference.  Run the GPU part with ``-s`` to see the measured maxima."""
import ctypes as C
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import spo_oracle as O

H = 64
NETS = ("actor", "reward_critic", "cost_critic")          # packed order (include/spo.h)
ACTIVE = {"ppo": NETS, "pg": NETS, "focops": NETS, "critic": NETS[1:], "cup": NETS[:1]}
# reference hyperparameters (ppo_lag.py / focops.py defaults as the oracle states them)
HP_REF = dict(clip_lo=0.8, clip_hi=1.2, critic_l2=0.001, value_coef=1.0, focops_lam=1.5, focops_kl=0.02, cup_coef=0.0,
              extra_sumsq=0.0, max_grad_norm=40.0)

# Bars (error / scale of the quantity), each at most 4x the largest error measured over this file's matrix on one
# H100 80 GB: grad 2.5e-6, loss 5.2e-7, ema_m 1.0e-6, ema_v 1.9e-6, weights 4.8e-5 (rounding of the fp32 weights
# against their 8-step movement), tr_grad 3.2e-6 (atomic flush order varies), tr_fvp 5.2e-7, tr_loss 1.4e-7, tr_kl 1.7e-6.
BAR = dict(grad=1e-5, loss=2e-6, ema_m=4e-6, ema_v=7e-6, weights=1e-4, tr_grad=1e-5, tr_fvp=2e-6, tr_loss=5e-7, tr_kl=6e-6)
MEASURED = {}


def _record(key, err):
    MEASURED[key] = max(MEASURED.get(key, 0.0), float(err))


def _names(net):
    p = "mean" if net == "actor" else "critic"
    return (["log_std"] if net == "actor" else []) + [f"{p}.{i}.{w}" for i in (0, 2, 4) for w in ("weight", "bias")]


def _shapes(net, D, A):
    O_ = A if net == "actor" else 1
    s = [(H, D), (H,), (H, H), (H,), (O_, H), (O_,)]
    return ([(A,)] if net == "actor" else []) + s


def tensor_slices(D, A, nets=NETS):
    """[(net, name, slice of the packed buffer, shape)] in packed order."""
    out, off = [], 0
    for net in NETS:
        for name, shp in zip(_names(net), _shapes(net, D, A)):
            n = int(np.prod(shp))
            if net in nets:
                out.append((net, name, slice(off, off + n), shp))
            off += n
    return out


def packed_size(D, A):
    return tensor_slices(D, A)[-1][2].stop


def unpack(flat, D, A):
    """An OraclePolicy whose leaves are copies of the packed vector's tensors (dtype of `flat`)."""
    pol = O.OraclePolicy.__new__(O.OraclePolicy)
    pol.obs_dim, pol.act_dim, pol.hidden_sizes = D, A, [H, H]
    pol.nets = {n: {} for n in NETS}
    for net, name, sl, shp in tensor_slices(D, A):
        pol.nets[net][name] = flat[sl].detach().clone().view(shp).requires_grad_(True)
    return pol


def pack(pol):
    return torch.cat([p.detach().reshape(-1) for n in NETS for p in pol.params(n)])


# ---------------------------------------------------------------------------------------------------------------
# float64 reference of one minibatch step
# ---------------------------------------------------------------------------------------------------------------

def ref_step(pol, b, kind, hp):
    """One minibatch step's losses and gradients (ppo_lag.py:298-336, pg.py:303-315, focops.py:309-357,
    cup.py:355-404, cpo.py:543-571), in the dtype of `pol` / `b`.  kind: ppo | pg | focops | cup | critic.
    The joint-norm clip runs over the three nets, over the actor alone (cup) or over the critics plus
    hp["extra_sumsq"] (critic).  Returns losses (loss_r, loss_c, loss_pi; None where the kind has none), the raw and
    the clipped gradients {net: [tensor]}, the joint norm, the clip coefficient and the mean |row term| of loss_pi."""
    for p in pol.all_params():
        p.grad = None
    obs = b["obs"]
    loss_r = loss_c = loss_pi = None
    scale_pi = None
    if kind != "cup":
        loss_r = F.mse_loss(O.critic_value(pol, "reward_critic", obs), b["target_value_r"])
        loss_c = F.mse_loss(O.critic_value(pol, "cost_critic", obs), b["target_value_c"])
        if hp["critic_l2"]:
            for p in pol.params("reward_critic"):
                loss_r = loss_r + p.pow(2).sum() * hp["critic_l2"]
            for p in pol.params("cost_critic"):
                loss_c = loss_c + p.pow(2).sum() * hp["critic_l2"]
    if kind != "critic":
        mean, std = O.actor_mean_std(pol, obs)
        logp = O.normal_log_prob(b["act"], mean, std).sum(dim=-1)
        ratio = torch.exp(logp - b["log_prob"])
        adv = b["adv"]
        if kind == "ppo":
            mins = torch.min(ratio * adv, torch.clamp(ratio, hp["clip_lo"], hp["clip_hi"]) * adv)
            loss_pi = -mins.mean()
            scale_pi = mins.detach().abs().mean()
        elif kind == "pg":
            loss_pi = -(ratio * adv).mean()
            scale_pi = (ratio * adv).detach().abs().mean()
        else:
            temp_kl = O.normal_kl(mean, std, b["old_mean"], b["old_std"]).sum(-1, keepdim=True)   # [B,1]
            if kind == "focops":
                mask = (temp_kl.detach() <= hp["focops_kl"]).to(temp_kl.dtype)
                terms = (temp_kl - (1 / hp["focops_lam"]) * ratio * adv) * mask                   # [B,B]
            else:
                terms = hp["cup_coef"] * ratio * adv + temp_kl                                     # [B,B]
            loss_pi = terms.mean()
            scale_pi = terms.detach().abs().mean()
    if kind != "cup":
        weighted_r = loss_r if hp["value_coef"] == 1 else hp["value_coef"] * loss_r   # 2*loss_r under use_value_coefficient
    if kind == "cup":
        total = loss_pi
    elif kind == "critic":
        total = weighted_r + loss_c
    else:
        total = loss_pi + weighted_r + loss_c
    total.backward()
    active = ACTIVE[kind]
    params = [p for n in active for p in pol.params(n)]
    raw = {n: [p.grad.detach().clone() for p in pol.params(n)] for n in active}
    sq = sum(float((g.double() ** 2).sum()) for gs in raw.values() for g in gs) + hp["extra_sumsq"]
    norm = math.sqrt(sq)
    coef = min(hp["max_grad_norm"] / (norm + 1e-6), 1.0)
    if hp["extra_sumsq"] == 0.0:
        torch.nn.utils.clip_grad_norm_(params, hp["max_grad_norm"])      # clip_grad_norm_ as the reference calls it
    elif coef < 1.0:
        for p in params:
            p.grad.mul_(coef)
    clipped = {n: [p.grad.detach().clone() for p in pol.params(n)] for n in active}
    item = lambda x: None if x is None else float(x.item())
    return dict(losses=(item(loss_r), item(loss_c), item(loss_pi)), raw=raw, grads=clipped, norm=norm, coef=coef,
                scale_pi=item(scale_pi))


# ---------------------------------------------------------------------------------------------------------------
# CPU: the reference against the oracle, and the readout algebra
# ---------------------------------------------------------------------------------------------------------------

def _cpu_batch(pol, B, g, D, A):
    obs = torch.randn(B, D, generator=g)
    with torch.no_grad():
        mean, std = O.actor_mean_std(pol, obs)
        act = mean + std * torch.randn(B, A, generator=g)
        logp = O.normal_log_prob(act, mean, std).sum(-1) + 0.2 * torch.randn(B, generator=g)
        old_mean = mean + 0.12 * torch.randn(B, A, generator=g)
        old_std = (std * torch.exp(0.05 * torch.randn(B, A, generator=g))).contiguous()
    return {"obs": obs, "act": act, "log_prob": logp, "target_value_r": torch.randn(B, generator=g),
            "target_value_c": torch.randn(B, generator=g).abs(), "adv": torch.randn(B, generator=g),
            "old_mean": old_mean, "old_std": old_std}


@pytest.mark.parametrize("kind", ["ppo", "pg", "focops", "critic"])
def test_reference_step_matches_oracle_bit_for_bit(kind):
    D, A, B = 17, 3, 48
    torch.manual_seed(11)
    pol = O.OraclePolicy(D, A)
    with torch.no_grad():
        pol.nets["actor"]["log_std"].copy_(torch.tensor([-0.4, 0.1, 0.3]))
    b = _cpu_batch(pol, B, torch.Generator().manual_seed(3), D, A)
    mine = unpack(pack(pol), D, A)
    got = ref_step(mine, b, kind, HP_REF)
    want = O.minibatch_step(pol, O.OracleOptim(pol), b, kind, max_grad_norm=40.0, target_kl=HP_REF["focops_kl"])
    for w, g_ in zip(want, got["losses"]):
        if g_ is not None:
            assert w == g_, (kind, w, g_)
    if kind == "focops":     # the KL mask takes both values
        with torch.no_grad():
            m, s = O.actor_mean_std(mine, b["obs"])
            kl = O.normal_kl(m, s, b["old_mean"], b["old_std"]).sum(-1)
        assert 0 < int((kl <= HP_REF["focops_kl"]).sum()) < B
    for net in ACTIVE[kind]:
        for p, g_ in zip(pol.params(net), got["grads"][net]):
            assert torch.equal(p.grad, g_), (kind, net)
    assert got["coef"] == 1.0


def test_reference_cup_step_matches_oracle_bit_for_bit():
    D, A, B = 9, 2, 40
    torch.manual_seed(12)
    pol = O.OraclePolicy(D, A)
    g = torch.Generator().manual_seed(4)
    data = _cpu_batch(pol, B, g, D, A)
    data["adv_c"] = data["adv"]
    lam, gamma = 0.7, 0.99
    mine = unpack(pack(pol), D, A)
    with torch.no_grad():
        om, os_ = O.actor_mean_std(mine, data["obs"])
    b = dict(data, old_mean=om.clone(), old_std=os_.expand_as(om).clone())
    c = lam * ((1 - gamma * 0.95) / (1 - gamma))
    got = ref_step(mine, b, "cup", dict(HP_REF, cup_coef=c))
    O.cup_second_stage(pol, O.OracleOptim(pol), data, lam, gamma=gamma, batch_size=B, learning_iters=1, target_kl=1e9,
                       perms=[torch.arange(B)])
    for p, g_ in zip(pol.params("actor"), got["grads"]["actor"]):
        assert torch.equal(p.grad, g_)
    assert all(p.grad is None for n in NETS[1:] for p in pol.params(n))


def test_adam_readout_algebra():
    """beta1 = 0, zero moments, lr = 0: one step leaves exp_avg == grad and the parameters equal, bit for bit; with
    lr = 0 and beta1 = beta2 = 0.5 K steps give the float64 EMAs of the gradients (to float32 rounding) at fixed
    parameters."""
    g = torch.Generator().manual_seed(0)
    p0 = torch.randn(200, generator=g)
    grad = torch.randn(200, generator=g) * torch.pow(10.0, torch.randint(-7, 3, (200,), generator=g).float())
    grad[:5] = 0.0
    p = p0.clone().requires_grad_(True)
    p.grad = grad.clone()
    opt = torch.optim.Adam([p], lr=0.0, betas=(0.0, 0.999))
    opt.step()
    assert torch.equal(opt.state[p]["exp_avg"], grad)
    assert torch.equal(p.detach(), p0)
    p = p0.clone().requires_grad_(True)
    opt = torch.optim.Adam([p], lr=0.0, betas=(0.5, 0.5))
    m64 = torch.zeros(200, dtype=torch.float64)
    v64 = torch.zeros(200, dtype=torch.float64)
    for k in range(5):
        gk = torch.randn(200, generator=g)
        p.grad = gk.clone()
        opt.step()
        m64 = m64 + 0.5 * (gk.double() - m64)
        v64 = 0.5 * v64 + 0.5 * gk.double() ** 2
    assert torch.equal(p.detach(), p0)
    assert float((opt.state[p]["exp_avg"].double() - m64).abs().max()) <= 1e-6 * float(m64.abs().max())
    assert float((opt.state[p]["exp_avg_sq"].double() - v64).abs().max()) <= 1e-6 * float(v64.abs().max())


def test_packed_slices_match_the_library_layout():
    """The per-tensor slices used below follow the packed layout of include/spo.h."""
    for D, A in ((1, 1), (17, 6), (128, 8)):
        sl = {(n, k): s for n, k, s, _ in tensor_slices(D, A)}
        assert sl[("actor", "log_std")] == slice(0, A)
        assert sl[("actor", "mean.0.weight")].start == A
        actor = A + H * D + H + H * H + H + A * H + A
        critic = H * D + H + H * H + H + H + 1
        assert sl[("reward_critic", "critic.0.weight")].start == actor
        assert packed_size(D, A) == actor + 2 * critic


# ---------------------------------------------------------------------------------------------------------------
# GPU harness
# ---------------------------------------------------------------------------------------------------------------

def _dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    return torch.device("cuda:0")


def _L():
    from safepo import _lib as L
    return L


KIND_ID = {"ppo": 0, "focops": 1, "critic": 2, "pg": 3, "cup": 4}


def make_hp(**kw):
    h = dict(lr=(0.0, 0.0, 0.0), beta1=0.0, beta2=0.999, adam_eps=1e-8, max_grad_norm=1e6, critic_l2=0.001, clip_lo=0.8,
             clip_hi=1.2, focops_lam=1.5, focops_kl=0.02, value_coef=1.0, cup_coef=0.7, extra_sumsq=0.0)
    h.update(kw)
    return h


def _hparams(L, kind, h):
    lam = h["cup_coef"] if kind == "cup" else h["focops_lam"]
    return L.HParams(*h["lr"], h["beta1"], h["beta2"], h["adam_eps"], h["max_grad_norm"], h["critic_l2"], h["clip_lo"],
                     h["clip_hi"], lam, h["focops_kl"], h["value_coef"])


def make_state(flat, m=None, v=None, t=None):
    dev = _dev()
    return dict(flat=flat.float().to(dev).contiguous(),
                m=(torch.zeros_like(flat) if m is None else m).float().to(dev).contiguous(),
                v=(torch.zeros_like(flat) if v is None else v).float().to(dev).contiguous(),
                t=(torch.zeros(3, dtype=torch.int32) if t is None else t).to(dev).contiguous(),
                ctrl=torch.zeros(64, dtype=torch.uint8, device=dev))


def launch(D, A, st, data, perm, batch, kind, h, stop=0):
    L = _L()
    dev = _dev()
    dd = {k: (None if v is None else v.to(dev).contiguous()) for k, v in data.items()}
    st["ctrl"].zero_()
    st["ctrl"].view(torch.float32)[L.CTRL_EXTRA_SUMSQ_F32_INDEX] = h["extra_sumsq"]
    st["ctrl"].view(torch.int32)[10] = stop
    uses_actor = kind != "critic"
    uses_old = kind in ("focops", "cup")
    bt = L.Batch(L.ptr(dd["obs"]), L.ptr(dd["act"]) if uses_actor else None, L.ptr(dd["log_prob"]) if uses_actor else None,
                 L.ptr(dd["target_value_r"]), L.ptr(dd["target_value_c"]), L.ptr(dd["adv"]) if uses_actor else None,
                 L.ptr(dd["old_mean"]) if uses_old else None, L.ptr(dd["old_std"]) if uses_old else None, dd["obs"].shape[0])
    hp = _hparams(L, kind, h)
    d = L.dims(D, A)
    perm_d = perm.to(dev).contiguous()
    L.check(L.lib().spo_pg_update(C.byref(d), L.ptr(st["flat"]), L.ptr(st["m"]), L.ptr(st["v"]), L.ptr(st["t"]), C.byref(bt),
                                  L.ptr(perm_d), perm_d.numel(), batch, KIND_ID[kind], C.byref(hp), L.ptr(st["ctrl"]), L.stream()),
            "spo_pg_update")
    torch.cuda.synchronize()
    c = st["ctrl"].cpu().numpy().view(L.CTRL_DTYPE)[0]
    return dict(loss_sum=[float(x) for x in c["loss_sum"]], steps=int(c["steps"]))


def make_case(kind, D, A, B, seed, h):
    """Float32 policy and data built in float64 from target values.  PPO: each of ratio < lo, lo <= ratio <= hi,
    ratio > hi gets a third of the rows, with both signs of adv in each band.  FOCOPS: KL(new || old) of a row
    lies below the threshold for half the rows and above it for the other half.  Returns (flat, data, idx) with
    idx the B selected rows (of B + 7) in step order."""
    torch.manual_seed(seed)
    pol = O.OraclePolicy(D, A)
    with torch.no_grad():
        pol.nets["actor"]["log_std"].copy_(torch.linspace(-0.6, 0.4, A) if A > 1 else torch.tensor([-0.2]))
    flat = pack(pol)
    p64 = unpack(flat.double(), D, A)
    g = torch.Generator().manual_seed(seed + 1)
    S = B + 7
    idx = torch.randperm(S, generator=g)[:B]
    obs = torch.randn(S, D, generator=g)
    with torch.no_grad():
        mean, std = O.actor_mean_std(p64, obs.double())
        act = (mean + std * torch.randn(S, A, generator=g, dtype=torch.float64)).float()
        logp = O.normal_log_prob(act.double(), mean, std).sum(-1)
    pos = torch.empty(S, dtype=torch.long)          # position of a row in step order (unselected rows last)
    pos[idx] = torch.arange(B)
    rest = torch.ones(S, dtype=torch.bool)
    rest[idx] = False
    pos[rest] = torch.arange(B, S)
    band = pos % 3
    u = torch.rand(S, generator=g, dtype=torch.float64)
    lo, hi = h["clip_lo"], h["clip_hi"]
    if kind == "ppo":
        r = torch.where(band == 0, lo * (0.5 + 0.45 * u), torch.where(band == 1, lo * 1.02 + (hi * 0.98 - lo * 1.02) * u,
                                                                       hi * (1.03 + 0.5 * u)))
    else:
        r = torch.exp(0.4 * torch.randn(S, generator=g, dtype=torch.float64))
    logp_old = (logp - torch.log(r)).float()
    sign = torch.where((pos // 3) % 2 == 0, 1.0, -1.0)
    adv = (sign * (0.2 + torch.randn(S, generator=g).abs())).float()
    data = {"obs": obs, "act": act, "log_prob": logp_old, "adv": adv,
            "target_value_r": torch.randn(S, generator=g), "target_value_c": torch.randn(S, generator=g).abs(),
            "old_mean": None, "old_std": None}
    if kind in ("focops", "cup"):
        delta = h["focops_kl"] if kind == "focops" else 0.05
        os64 = std * torch.exp(0.02 * torch.randn(S, A, generator=g, dtype=torch.float64))
        vr = (std / os64) ** 2
        base = 0.5 * (vr - 1 - vr.log()).sum(-1)
        below = pos % 2 == 0
        k = torch.where(below, torch.maximum(delta * (0.1 + 0.7 * u), base + 0.05 * delta), delta * (1.25 + 2 * u))
        dirn = torch.randn(S, A, generator=g, dtype=torch.float64)
        dirn = dirn / dirn.norm(dim=-1, keepdim=True)
        om64 = mean - os64 * dirn * torch.sqrt(2 * (k - base)).unsqueeze(-1)
        data["old_mean"], data["old_std"] = om64.float(), os64.float()
    if kind == "critic":
        data.update(act=None, log_prob=None, adv=None)
    return flat, data, idx


def _rows64(data, rows):
    return {k: (None if v is None else v[rows].double()) for k, v in data.items()}


def check_case_inputs(kind, D, A, flat, data, rows, h):
    """Counts of the decision branches over the selected rows, and their distance from every boundary."""
    if kind == "critic" or len(rows) < 30:
        return
    p64 = unpack(flat.double(), D, A)
    b = _rows64(data, rows)
    with torch.no_grad():
        mean, std = O.actor_mean_std(p64, b["obs"])
        ratio = torch.exp(O.normal_log_prob(b["act"], mean, std).sum(-1) - b["log_prob"])
    n = len(rows)
    if kind == "ppo":
        lo, hi = h["clip_lo"], h["clip_hi"]
        for m in (ratio < lo, (ratio >= lo) & (ratio <= hi), ratio > hi):
            assert int((m & (b["adv"] > 0)).sum()) >= 1 and int((m & (b["adv"] < 0)).sum()) >= 1
            assert int(m.sum()) >= 0.1 * n
        assert float(torch.minimum((ratio / lo - 1).abs(), (ratio / hi - 1).abs()).min()) > 1e-3
    if kind in ("focops", "cup"):
        with torch.no_grad():
            kl = O.normal_kl(mean, std, b["old_mean"], b["old_std"]).sum(-1)
        delta = h["focops_kl"] if kind == "focops" else 0.05
        assert int((kl < delta).sum()) >= 0.2 * n and int((kl > delta).sum()) >= 0.2 * n
        assert float((kl / delta - 1).abs().min()) > 1e-3


def reference(kind, D, A, flat, data, rows, h):
    p64 = unpack(flat.double(), D, A)
    return ref_step(p64, _rows64(data, rows), kind, h)


def compare_grads(tag, D, A, m_flat, ref, coef_expected=None, key="grad", bar=None):
    """Per tensor: max |m - g64| <= bar * max |g64|; tensors whose float64 gradient is exactly 0 must read 0."""
    bar = BAR[key] if bar is None else bar
    m_flat = m_flat.double().cpu()
    worst = 0.0
    for net, name, sl, shp in tensor_slices(D, A, ACTIVE[tag[0]]):
        i = _names(net).index(name)
        g64 = ref[net][i].reshape(-1).double()
        got = m_flat[sl]
        scale = float(g64.abs().max())
        if scale == 0.0:
            assert float(got.abs().max()) == 0.0, (tag, net, name)
            continue
        err = float((got - g64).abs().max()) / scale
        worst = max(worst, err)
        assert err <= bar, (tag, net, name, err)
    _record(key, worst)
    return worst


def compare_losses(tag, kind, loss_sum, want, scale_pi, key="loss"):
    slots = {"critic": (0, 1), "cup": (2,)}.get(kind, (0, 1, 2))
    worst = 0.0
    for s in slots:
        w = want[s]
        scale = max(abs(w), 1e-6) if s < 2 else max(scale_pi, 1e-6)
        err = abs(loss_sum[s] - w) / scale
        worst = max(worst, err)
        assert err <= BAR[key], (tag, s, loss_sum[s], w, err)
    _record(key, worst)


def untouched(st, st0, D, A, nets):
    """Parameters and moments of `nets` and their step counters are bit-identical to the copies in st0."""
    for net, name, sl, _ in tensor_slices(D, A, nets):
        for k in ("flat", "m", "v"):
            assert torch.equal(st[k][sl].cpu(), st0[k][sl]), (net, name, k)
    for i, net in enumerate(NETS):
        if net in nets:
            assert int(st["t"][i]) == int(st0["t"][i]), net


# ---------------------------------------------------------------------------------------------------------------
# 1. one-step gradient readout
# ---------------------------------------------------------------------------------------------------------------

READOUT = [
    ("ppo", 60, 2, 64, dict()),
    ("ppo", 1, 1, 1, dict(clip_lo=0.7, clip_hi=1.3, critic_l2=0.1, value_coef=2.0)),
    ("ppo", 17, 6, 64, dict(clip_lo=0.7, clip_hi=1.3, critic_l2=0.0, value_coef=2.0)),
    ("ppo", 63, 3, 65, dict(critic_l2=0.1)),
    ("ppo", 64, 8, 128, dict(clip_lo=0.7, clip_hi=1.3, value_coef=2.0)),
    ("ppo", 65, 5, 100, dict(critic_l2=0.0, value_coef=2.0)),
    ("ppo", 104, 3, 192, dict(clip_lo=0.7, clip_hi=1.3, critic_l2=0.1)),
    ("ppo", 128, 8, 256, dict(value_coef=2.0)),
    ("ppo", 27, 8, 129, dict(clip_lo=0.7, clip_hi=1.3, critic_l2=0.1, value_coef=2.0)),
    ("pg", 60, 2, 64, dict()),
    ("pg", 17, 6, 100, dict(critic_l2=0.1, value_coef=2.0)),
    ("focops", 60, 2, 64, dict(focops_kl=0.05)),
    ("focops", 27, 8, 48, dict(focops_lam=0.3, focops_kl=0.05, critic_l2=0.1, value_coef=2.0)),
    ("focops", 128, 1, 1, dict(focops_lam=0.3, focops_kl=0.05, critic_l2=0.0, value_coef=2.0)),
    ("focops", 65, 7, 17, dict(focops_kl=0.05, critic_l2=0.1)),
    ("cup", 60, 2, 64, dict(cup_coef=0.7)),
    ("cup", 88, 2, 37, dict(cup_coef=2.5)),
    ("critic", 60, 2, 128, dict(value_coef=2.0)),
    ("critic", 88, 2, 129, dict(critic_l2=0.1)),
    ("critic", 1, 1, 256, dict(critic_l2=0.0, value_coef=2.0)),
]


def run_readout(kind, D, A, B, extra, seed=None):
    """One step at lr = 0, beta1 = 0 from zero moments.  Returns (state, state before, launch result, reference)."""
    h = make_hp(**extra)
    seed = 1000 * D + 10 * A + B + KIND_ID[kind] if seed is None else seed
    flat, data, idx = make_case(kind, D, A, B, seed, h)
    check_case_inputs(kind, D, A, flat, data, idx, h)
    st = make_state(flat)
    st0 = {k: v.cpu().clone() for k, v in st.items()}
    res = launch(D, A, st, data, idx, B, kind, h)
    ref = reference(kind, D, A, flat, data, idx, h)
    return st, st0, res, ref


@pytest.mark.gpu
@pytest.mark.parametrize("kind,D,A,B,extra", READOUT, ids=[f"{k}-{d}-{a}-{b}" for k, d, a, b, _ in READOUT])
def test_update_gradient_readout_vs_float64(kind, D, A, B, extra):
    st, st0, res, ref = run_readout(kind, D, A, B, extra)
    tag = (kind, D, A, B)
    assert res["steps"] == 1
    assert torch.equal(st["flat"].cpu(), st0["flat"])                       # lr = 0: the weights do not move
    assert ref["coef"] == 1.0
    worst = compare_grads(tag, D, A, st["m"], ref["grads"])
    compare_losses(tag, kind, res["loss_sum"], ref["losses"], ref["scale_pi"])
    inactive = tuple(n for n in NETS if n not in ACTIVE[kind])
    untouched(st, st0, D, A, inactive)
    t = st["t"].cpu().tolist()
    assert t == [1 if n in ACTIVE[kind] else 0 for n in NETS], t
    print(f"readout {tag}: max grad err {worst:.3g}")


# ---------------------------------------------------------------------------------------------------------------
# 2. clip coefficient
# ---------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("kind,D,A,B,extra", [
    ("ppo", 60, 2, 64, dict()),
    ("ppo", 104, 3, 100, dict(value_coef=2.0)),
    ("cup", 60, 2, 64, dict(cup_coef=0.7)),
    ("critic", 88, 2, 129, dict(extra_sumsq=900.0)),
])
def test_update_clip_coefficient_vs_float64(kind, D, A, B, extra):
    """max_grad_norm below the joint norm (all three nets; the actor alone for CUP; the critics plus extra_sumsq for
    critic-only): adam_m == clip * g64 with clip = max / (|g| + 1e-6) computed in float64."""
    h = make_hp(**extra)
    seed = 7 * D + A + B
    flat, data, idx = make_case(kind, D, A, B, seed, h)
    free = reference(kind, D, A, flat, data, idx, h)
    h["max_grad_norm"] = 0.3 * free["norm"]
    st = make_state(flat)
    res = launch(D, A, st, data, idx, B, kind, h)
    ref = reference(kind, D, A, flat, data, idx, h)
    assert 0.29 < ref["coef"] < 0.31 and res["steps"] == 1
    want = {n: [ref["coef"] * g.double() for g in gs] for n, gs in free["raw"].items()}
    compare_grads((kind, D, A, B), D, A, st["m"], want)


# ---------------------------------------------------------------------------------------------------------------
# 3. several steps at fixed weights
# ---------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("kind,D,A,batch,K,extra", [
    ("ppo", 60, 2, 100, 5, dict(critic_l2=0.1, value_coef=2.0)),   # two tiles per step, last step 37 rows
    ("critic", 88, 2, 128, 5, dict()),                              # last step 50 rows
])
def test_update_multistep_fixed_weights_emas(kind, D, A, batch, K, extra):
    h = make_hp(beta1=0.5, beta2=0.5, **extra)
    n = (K - 1) * batch + (37 if kind == "ppo" else 50)
    flat, data, idx = make_case(kind, D, A, n, 31 * D + K, h)
    steps = [idx[k * batch:(k + 1) * batch] for k in range(K)]
    free = [reference(kind, D, A, flat, data, s, h) for s in steps]
    norms = sorted(r["norm"] for r in free)
    h["max_grad_norm"] = math.sqrt(norms[2] * norms[3])           # the two largest steps exceed it
    refs = [reference(kind, D, A, flat, data, s, h) for s in steps]
    clipped = sum(r["coef"] < 1.0 for r in refs)
    assert 0 < clipped < K
    st = make_state(flat, t=torch.tensor([3, 4, 5], dtype=torch.int32))
    t0 = st["t"].cpu().clone()
    res = launch(D, A, st, data, idx, batch, kind, h)
    assert res["steps"] == K
    m64, v64 = {}, {}
    for r in refs:
        for net, gs in r["grads"].items():
            for i, g in enumerate(gs):
                key = (net, i)
                m0, v0 = m64.get(key, torch.zeros_like(g)), v64.get(key, torch.zeros_like(g))
                m64[key] = m0 + 0.5 * (g - m0)
                v64[key] = 0.5 * v0 + 0.5 * g * g
    as_nets = lambda d: {net: [d[(net, i)] for i in range(len(_names(net)))] for net in ACTIVE[kind]}
    compare_grads((kind, D, A, batch, "m"), D, A, st["m"], as_nets(m64), key="ema_m")
    compare_grads((kind, D, A, batch, "v"), D, A, st["v"], as_nets(v64), key="ema_v")
    want = [sum(r["losses"][s] for r in refs) if refs[0]["losses"][s] is not None else None for s in range(3)]
    compare_losses((kind, D, A, batch), kind, res["loss_sum"], want, sum(r["scale_pi"] or 0.0 for r in refs))
    t = st["t"].cpu()
    for i, net in enumerate(NETS):
        assert int(t[i]) == int(t0[i]) + (K if net in ACTIVE[kind] else 0), (net, t.tolist())
    assert torch.equal(st["flat"].cpu(), flat)


# ---------------------------------------------------------------------------------------------------------------
# 4. several steps with moving weights
# ---------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("D,A,batch,tail", [(60, 2, 64, 13), (104, 3, 100, 100)])
def test_update_multistep_moving_weights_vs_float64_replay(D, A, batch, tail):
    """betas (0, 0) and adam_eps = 10: each step is p -= lr g / (|g| + 10), nearly SGD.  8 steps against a float64
    replay, per tensor relative to that tensor's total movement."""
    K, lr, eps = 8, 0.05, 10.0
    h = make_hp(lr=(lr, lr, lr), beta1=0.0, beta2=0.0, adam_eps=eps, value_coef=2.0)
    n = (K - 1) * batch + tail
    flat, data, idx = make_case("ppo", D, A, n, 17 * D + batch, h)
    st = make_state(flat)
    res = launch(D, A, st, data, idx, batch, "ppo", h)
    assert res["steps"] == K
    theta = flat.double().clone()
    for k in range(K):
        r = reference("ppo", D, A, theta, data, idx[k * batch:(k + 1) * batch], h)
        for net, name, sl, shp in tensor_slices(D, A):
            g = r["grads"][net][_names(net).index(name)].reshape(-1)
            theta[sl] -= lr * g / (g.abs() + eps)
    got = st["flat"].double().cpu()
    worst = 0.0
    for net, name, sl, _ in tensor_slices(D, A):
        move = float((theta[sl] - flat[sl].double()).abs().max())
        assert move > 0, (net, name)
        err = float((got[sl] - theta[sl]).abs().max()) / move
        worst = max(worst, err)
        assert err <= BAR["weights"], (D, A, net, name, err)
    _record("weights", worst)


# ---------------------------------------------------------------------------------------------------------------
# 5. state that must not move
# ---------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("kind,stop", [("ppo", 1), ("critic", 0), ("cup", 0)])
def test_update_leaves_inactive_state_untouched(kind, stop):
    D, A, B = 60, 2, 64
    h = make_hp(lr=(1e-3, 1e-3, 1e-3), beta1=0.9, beta2=0.999)
    flat, data, idx = make_case(kind, D, A, 3 * B, 5, h)
    g = torch.Generator().manual_seed(6)
    P = flat.numel()
    st = make_state(flat, m=0.01 * torch.randn(P, generator=g), v=1e-4 * torch.rand(P, generator=g),
                    t=torch.tensor([3, 4, 5], dtype=torch.int32))
    st0 = {k: v.cpu().clone() for k, v in st.items()}
    res = launch(D, A, st, data, idx, B, kind, h, stop=stop)
    if stop:
        assert res["steps"] == 0
        untouched(st, st0, D, A, NETS)
        return
    assert res["steps"] == 3
    untouched(st, st0, D, A, tuple(n for n in NETS if n not in ACTIVE[kind]))
    for net, name, sl, _ in tensor_slices(D, A, ACTIVE[kind]):
        assert not torch.equal(st["flat"][sl].cpu(), st0["flat"][sl]), (net, name)


# ---------------------------------------------------------------------------------------------------------------
# 6. the 16-CTA cluster
# ---------------------------------------------------------------------------------------------------------------

CLUSTER_CASES = [READOUT[5], READOUT[12]]     # PPO (65, 5, 100) and FOCOPS (27, 8, 48)


def dump_cluster_cases(path):
    out = {}
    for kind, D, A, B, extra in CLUSTER_CASES:
        st, _, res, _ = run_readout(kind, D, A, B, extra)
        out[f"{kind}-{D}-{A}-{B}"] = (st["m"].cpu(), st["v"].cpu(), torch.tensor(res["loss_sum"], dtype=torch.float64))
    torch.save(out, path)


@pytest.mark.gpu
def test_update_16_cta_cluster_matches_12(tmp_path):
    """launch_update tries a cluster of 12 CTAs first and falls back to 16 with four idle; the size is cached per
    process, so the 16-CTA run is a subprocess with SPO_CLUSTER=16.  The idle CTAs contribute nothing and the norm
    sums run in CTA order over the same twelve partials: moments and losses must be bit-identical."""
    here = os.path.dirname(os.path.abspath(__file__))
    root = os.path.dirname(here)
    path = str(tmp_path / "c16.pt")
    code = ("import sys; sys.path[:0] = {!r}; import test_update_gradients as T; T.dump_cluster_cases({!r})"
            .format([root, os.path.join(root, "safe-policy-optimization_b200"), here], path))
    env = dict(os.environ, SPO_CLUSTER="16")
    r = subprocess.run([sys.executable, "-c", code], env=env, cwd=root, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    got = torch.load(path)
    for kind, D, A, B, extra in CLUSTER_CASES:
        st, _, res, _ = run_readout(kind, D, A, B, extra)
        m16, v16, l16 = got[f"{kind}-{D}-{A}-{B}"]
        assert torch.equal(st["m"].cpu(), m16) and torch.equal(st["v"].cpu(), v16), kind
        assert l16.tolist() == res["loss_sum"], (kind, l16.tolist(), res["loss_sum"])


# ---------------------------------------------------------------------------------------------------------------
# 7. trust-region kernels
# ---------------------------------------------------------------------------------------------------------------

TR_SHAPES = [(1, 1), (17, 5), (60, 2), (64, 8), (65, 1), (116, 8), (117, 8), (120, 5), (121, 5), (124, 2), (125, 2), (128, 8)]
TR_CASES = [(D, A, "many") for D, A in TR_SHAPES] + [(D, A, S) for D, A in ((1, 1), (65, 1), (128, 8), (60, 2))
                                                   for S in (1, 63, 65)]


def _many_tiles():
    """Every CTA of the persistent grid (one per SM) loops over two tiles and the last tile holds 37 rows."""
    return 64 * 2 * torch.cuda.get_device_properties(0).multi_processor_count + 37


def trust_case(D, A, S, seed):
    torch.manual_seed(seed)
    pol = O.OraclePolicy(D, A)
    with torch.no_grad():
        pol.nets["actor"]["log_std"].copy_(torch.linspace(-0.5, 0.3, A) if A > 1 else torch.tensor([0.15]))
    flat = pack(pol)
    g = torch.Generator().manual_seed(seed + 1)
    obs = torch.randn(S, D, generator=g)
    p64 = unpack(flat.double(), D, A)
    with torch.no_grad():
        mean, std = O.actor_mean_std(p64, obs.double())
        act = (mean + std * torch.randn(S, A, generator=g, dtype=torch.float64)).float()
        logp = (O.normal_log_prob(act.double(), mean, std).sum(-1) + 0.1 * torch.randn(S, generator=g, dtype=torch.float64)).float()
        old_mean = (mean + 0.05 * torch.randn(S, A, generator=g, dtype=torch.float64)).float()
    old_ls = (p64.nets["actor"]["log_std"].detach() + 0.1 * torch.randn(A, generator=g, dtype=torch.float64)).float()
    adv_a, adv_b = torch.randn(S, generator=g), torch.randn(S, generator=g)
    P = tensor_slices(D, A, ("actor",))[-1][2].stop
    v = torch.randn(P, generator=g)
    return flat, dict(obs=obs, act=act, logp=logp, old_mean=old_mean, old_ls=old_ls, adv_a=adv_a, adv_b=adv_b, v=v), P


def compare_actor_vec(tag, D, A, got, want, key):
    got, want = got.double().cpu(), want.double()
    worst = 0.0
    for net, name, sl, _ in tensor_slices(D, A, ("actor",)):
        scale = float(want[sl].abs().max())
        err = float((got[sl] - want[sl]).abs().max()) / max(scale, 1e-30)
        worst = max(worst, err)
        assert err <= BAR[key], (tag, name, err, scale)
    _record(key, worst)
    return worst


@pytest.mark.gpu
@pytest.mark.parametrize("D,A,S", TR_CASES, ids=[f"{d}-{a}-{s}" for d, a, s in TR_CASES])
def test_trust_region_kernels_per_tensor_vs_float64(D, A, S):
    """spo_surrogate_grad, spo_fvp and spo_linesearch_eval per tensor against float64 autograd of cpo.py's
    surrogate, fvp() and line-search quantities (obs_dim 117..128 at act_dim 8 needed a smaller FVP layout)."""
    L = _L()
    dev = _dev()
    S = _many_tiles() if S == "many" else S
    flat, c, P = trust_case(D, A, S, 100 * D + A + S)
    d = L.dims(D, A)
    dv = {k: v.to(dev).contiguous() for k, v in c.items()}
    params = flat.to(dev)
    tag = (D, A, S)
    p64 = unpack(flat.double(), D, A)
    obs64, act64, logp64 = c["obs"].double(), c["act"].double(), c["logp"].double()

    # surrogate and its gradient
    loss = torch.zeros(1, device=dev)
    grad = torch.zeros(P, device=dev)
    L.check(L.lib().spo_surrogate_grad(C.byref(d), L.ptr(params), L.ptr(dv["obs"]), L.ptr(dv["act"]), L.ptr(dv["logp"]),
                                       L.ptr(dv["adv_a"]), S, L.ptr(loss), L.ptr(grad), L.stream()), "spo_surrogate_grad")
    surr = O.surrogate_loss(p64, obs64, act64, logp64, c["adv_a"].double())
    g64 = torch.cat([x.reshape(-1) for x in torch.autograd.grad(surr, p64.params("actor"))])
    with torch.no_grad():
        mean, std = O.actor_mean_std(p64, obs64)
        ratio = torch.exp(O.normal_log_prob(act64, mean, std).sum(-1) - logp64)
    scale = float((ratio * c["adv_a"].double()).abs().mean())
    err = abs(float(loss) - float(surr.detach())) / scale
    _record("tr_loss", err)
    assert err <= BAR["tr_loss"], (tag, float(loss), float(surr.detach()))
    compare_actor_vec(tag, D, A, grad, g64, "tr_grad")

    # Fisher-vector product
    out = torch.zeros(P, device=dev)
    L.check(L.lib().spo_fvp(C.byref(d), L.ptr(params), L.ptr(dv["obs"]), S, L.ptr(dv["v"]), 0.1, L.ptr(out), L.stream()),
            "spo_fvp")
    f64 = O.fvp_autograd(p64, obs64, c["v"].double()).detach()
    ls_closed = (2.0 / A + 0.1) * c["v"][:A].double()
    assert float((f64[:A] - ls_closed).abs().max()) <= 1e-12 * float(ls_closed.abs().max()) + 1e-300
    compare_actor_vec(tag, D, A, out, f64, "tr_fvp")

    # line-search quantities, with and without the second advantage
    with torch.no_grad():
        kl64 = O.normal_kl(c["old_mean"].double(), torch.exp(c["old_ls"].double()).expand(S, A), mean, std).mean()
        want = [float((ratio * c["adv_a"].double()).mean()), float((ratio * c["adv_b"].double()).mean()), float(kl64)]
    scale_b = float((ratio * c["adv_b"].double()).abs().mean())
    for adv_b in (None, dv["adv_b"]):
        out3 = torch.zeros(3, device=dev)
        L.check(L.lib().spo_linesearch_eval(C.byref(d), L.ptr(params), L.ptr(dv["obs"]), L.ptr(dv["act"]), L.ptr(dv["logp"]),
                                            L.ptr(dv["adv_a"]), L.ptr(adv_b), L.ptr(dv["old_mean"]), L.ptr(dv["old_ls"]), S,
                                            L.ptr(out3), L.stream()), "spo_linesearch_eval")
        o = out3.cpu().double().tolist()
        e0 = abs(o[0] - want[0]) / scale
        e1 = abs(o[1] - want[1]) / scale_b if adv_b is not None else abs(o[1])
        e2 = abs(o[2] - want[2]) / abs(want[2])
        _record("tr_loss", max(e0, e1))
        _record("tr_kl", e2)
        assert e0 <= BAR["tr_loss"] and e2 <= BAR["tr_kl"], (tag, o, want)
        assert (e1 <= BAR["tr_loss"]) if adv_b is not None else o[1] == 0.0, (tag, o, want)


@pytest.mark.gpu
def test_conjugate_gradient_equals_split_solver_bit_for_bit():
    """spo_conjugate_gradient against the split spo_cg_begin / spo_fvp / spo_cg_update sequence the data-parallel
    CPO path runs.  S = 127 gives two CTAs, whose two atomic adds into a zeroed vector commute exactly, so the FVP is
    deterministic and both solvers must agree bit for bit."""
    L = _L()
    dev = _dev()
    D, A, S, iters = 117, 8, 127, 10
    flat, c, P = trust_case(D, A, S, 9)
    d = L.dims(D, A)
    obs, params, b = c["obs"].to(dev), flat.to(dev), c["v"].to(dev)
    x1, w1 = torch.zeros(P, device=dev), torch.zeros(4 * P + 8, device=dev)
    L.check(L.lib().spo_conjugate_gradient(C.byref(d), L.ptr(params), L.ptr(obs), S, L.ptr(b), iters, 0.1, 1e-10, 1e-6,
                                           L.ptr(x1), L.ptr(w1), L.stream()), "spo_conjugate_gradient")
    x2, w2 = torch.zeros(P, device=dev), torch.zeros(4 * P + 8, device=dev)
    L.check(L.lib().spo_cg_begin(C.byref(d), L.ptr(b), L.ptr(x2), L.ptr(w2), L.stream()), "spo_cg_begin")
    for _ in range(iters):
        L.check(L.lib().spo_fvp(C.byref(d), L.ptr(params), L.ptr(obs), S, L.ptr(w2[P:2 * P]), 0.1, L.ptr(w2[2 * P:3 * P]),
                                L.stream()), "spo_fvp")
        L.check(L.lib().spo_cg_update(C.byref(d), L.ptr(x2), L.ptr(w2), 1e-10, 1e-6, L.stream()), "spo_cg_update")
    torch.cuda.synchronize()
    assert torch.equal(x1, x2)
    assert torch.equal(w1[:3 * P], w2[:3 * P]) and torch.equal(w1[4 * P:], w2[4 * P:])
    assert float(x1.abs().max()) > 0


@pytest.fixture(scope="module", autouse=True)
def _print_measured():
    yield
    if MEASURED:
        print("\nmeasured maxima (error / scale) vs bars:")
        for k in sorted(MEASURED):
            print(f"  {k:9s} {MEASURED[k]:.3e}   bar {BAR[k]:.1e}")
