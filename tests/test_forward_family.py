"""The single-agent forward family (csrc/spo_forward.cu, spo_ffma_forward.cuh, spo_tc_forward.cu) against float64, per kernel.

Five entry points -- spo_policy_step, spo_critic_values, spo_actor_forward, spo_actor_kl and the spo_actor_kl_accumulate +
spo_kl_finalize pair -- go through one dispatcher that runs one of three kernels: the TMA + wgmma kernel (3xTF32, SFU tanh,
128-row tiles), the FFMA tile kernel at action capacity 8, or at capacity 16.  Every GPU case below asserts which kernel it
ran (by kernel name) and sits on an edge of that choice: obs_dim 4 (one K-chunk), 64 / 65 / 68, n = 127 / 128,
S = 1023 / 1024, one row, and S_multi = 3 * 128 * SMs + 37 rows, which gives each CTA of either persistent grid at least three
tiles.  The inputs take five regimes: nominal, saturated tanh (weights x4, obs x10), the |x| < 0.04 Taylor branch of the SFU
tanh (zero obs rows, |b1| < 0.04), column scales from 1e-3 to 1e2 (where the lo term of the 3xTF32 split matters), and
log_std at -5, -1, 0 and 1.5; host eps always holds exact zeros and |e| up to 5.

The reference is float64 evaluation of the oracle's own functions (oracle.spo_oracle.actor_mean_std, critic_value,
normal_log_prob, normal_kl) on the same float32 inputs the kernel gets.  Each error is relative to its tensor's max |float64|,
must be exactly 0 where float64 is 0, and each bar is at most 4x the largest error measured over this file's matrix on one
H100 (MEASURED; run with -s to print it).  Two quantities take their own scale:
  logp  for a = mu + e sigma, (a - mu) / sigma cancels in fp32 (in the reference as well), so row i passes when
        |logp - logp64| <= bar * sum_j (e_j^2 / 2 + |log sigma_j| + 0.92) + sum_j |e_j| 2^-23 max(|a_j|, |mu_j|) / sigma_j
  KL    relative to the mean |per-row term| (divided by act_dim for the mean over rows x act_dim).

The in-kernel sampler is restated on the host: Philox4x32-10 (checked against Random123's known answers on the CPU) on the
counter (row, dimension pair, offset lo, offset hi) keyed by the seed, and the kernel's Box-Muller with its fp32 steps.  The
KL pass tests pin the control block: the stop decision of every launch, reuse across kernels with different grids, the
no-op once stop is set, and the data-parallel split into accumulate + finalize."""
import ctypes as C
import os
import re
import tempfile
import warnings

import numpy as np
import pytest
import torch

from oracle import spo_oracle as O

import test_update_gradients as TU

# Bars: error / scale, each at most 4x the largest error measured over this file's matrix on one H100 80GB HBM3 at its 700 W
# limit (in brackets).
BAR = dict(
    mean=1.1e-5,    # [3.0e-6] actor means (spo_actor_forward, deterministic step)
    value=3.5e-6,   # [9.2e-7] v_r, v_c
    act=1.1e-5,     # [3.0e-6] sampled action with host eps
    logp=3.5e-7,    # [9.0e-8] log-density, in the scale of the module docstring
    kl=1e-5,        # [2.7e-6] final_kl of a pass and the accumulated sum, relative to the mean |per-row term|
    cross=5e-6)     # [1.3e-6] wgmma against FFMA on the same rows, relative to max |float64|
MEASURED = {}
Z_ULPS = 8          # sampler: fp32 ulps of |z| allowed on top of the rounding of the action (logf, sincosf, rad * cos)

NETS = TU.NETS
SENTINEL = 0x7FC0BEEF          # a quiet NaN: buffers are filled with it, and what the kernels must not write keeps its bits
PAD = 131                      # rows past n in over-allocated outputs (more than a tile of either kernel)
LOG_STD_EXTREMES = (-5.0, -1.0, 0.0, 1.5)
REGIMES = ("nominal", "saturated", "taylor", "wide", "log_std")
PHILOX_SEED = 0x9E3779B97F4A7C15                       # high word set
PHILOX_OFFSETS = (1, 2 ** 32 - 1, 2 ** 32, 2 ** 32 + 1)


# ============================================================ host restatements ============================================================
M32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """Random123's philox4x32_R(10, ctr, key): ctr four uint32 arrays (broadcast), key two ints."""
    c0, c1, c2, c3 = (np.asarray(x, dtype=np.uint64) & M32 for x in ctr)
    k0, k1 = np.uint64(key[0] & 0xFFFFFFFF), np.uint64(key[1] & 0xFFFFFFFF)
    for _ in range(10):
        p0, p1 = c0 * np.uint64(0xD2511F53), c2 * np.uint64(0xCD9E8D57)     # < 2^64: exact in uint64
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & M32, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & M32
        k0, k1 = (k0 + np.uint64(0x9E3779B9)) & M32, (k1 + np.uint64(0xBB67AE85)) & M32
    return tuple(x.astype(np.uint32) for x in (c0, c1, c2, c3))


def box_muller(a, b):
    """The kernel's Box-Muller (spo_box_muller): u = (float(a) + 0.5f) * 2^-32 and the angle 6.2831855f * u2 in fp32,
    then log, sqrt, sin and cos in float64.  Returns (rad * cos, rad * sin)."""
    f = np.float32
    u1 = (a.astype(np.float32) + f(0.5)) * f(2.3283064365386963e-10)
    u2 = (b.astype(np.float32) + f(0.5)) * f(2.3283064365386963e-10)
    theta = (f(6.283185307179586) * u2).astype(np.float64)
    rad = np.sqrt(-2.0 * np.log(u1.astype(np.float64)))
    return rad * np.cos(theta), rad * np.sin(theta)


def host_draws(n, A, seed, offset):
    """[n, A] standard-normal draws of the rollout step: dimension j of row g is component j & 1 of the Box-Muller pair
    of Philox counter (g, j >> 1, offset lo, offset hi) under key (seed lo, seed hi)."""
    g = np.arange(n, dtype=np.uint64)[:, None]
    pair = np.arange((A + 1) // 2, dtype=np.uint64)[None, :]
    x, y, _, _ = philox4x32_10((g, pair, offset & 0xFFFFFFFF, offset >> 32), (seed & 0xFFFFFFFF, seed >> 32))
    zc, zs = box_muller(x, y)
    return np.stack([zc, zs], -1).reshape(n, -1)[:, :A]


# ============================================================ inputs ============================================================
def make_case(D, A, n, regime, seed):
    """Packed float32 parameters, obs [n, D] and host eps [n, A] in one of the input regimes."""
    torch.manual_seed(seed)
    g = torch.Generator().manual_seed(seed + 1)
    flat = TU.pack(O.OraclePolicy(D, A)).float().clone()
    where = {(net, name): sl for net, name, sl, _ in TU.tensor_slices(D, A)}
    log_std = torch.linspace(-0.5, 0.3, A) if A > 1 else torch.tensor([-0.2])
    obs = torch.randn(n, D, generator=g)
    if regime == "saturated":
        for (net, name), sl in where.items():
            if name != "log_std":
                flat[sl] *= 4
        obs *= 10
    elif regime == "taylor":
        for net in NETS:
            sl = where[(net, ("mean" if net == "actor" else "critic") + ".0.bias")]
            flat[sl] *= 0.035 / float(flat[sl].abs().max())
        obs[::3] = 0
    elif regime == "wide":
        obs *= torch.logspace(-3, 2, D)
    elif regime == "log_std":
        log_std = torch.tensor([LOG_STD_EXTREMES[(j + D) % 4] for j in range(A)])
    flat[where[("actor", "log_std")]] = log_std
    eps = torch.randn(n, A, generator=g).clamp(-5, 5)
    eps[::5] = 0.0
    flat_eps = eps.view(-1)
    flat_eps[3::11] = 5.0
    flat_eps[7::13] = -5.0
    return flat, obs.contiguous(), eps.contiguous()


def tanh_regime_counts(flat, D, A, obs):
    """Hidden pre-activations of the three nets in float64 (the oracle's _mlp cut after layer 1 and after layer 2), counted
    per branch of the SFU tanh: |x| < 0.04 (Taylor), mid, |x| > 9 (saturated)."""
    pol = TU.unpack(flat.double(), D, A)
    x = obs.double()
    pre = []
    with torch.no_grad():
        for net in NETS:
            prefix = "mean" if net == "actor" else "critic"
            d = pol.nets[net]
            for depth in (1, 2):
                sub = {f"{prefix}.{2 * i}.{w}": d[f"{prefix}.{2 * i}.{w}"] for i in range(depth) for w in ("weight", "bias")}
                pre.append(O._mlp(sub, prefix, x).reshape(-1))
    p = torch.cat(pre).abs()
    small, big = int((p < 0.04).sum()), int((p > 9).sum())
    return dict(taylor=small, mid=p.numel() - small - big, saturated=big)


def assert_regime(regime, counts, n):
    assert counts["mid"] > 0, counts
    if regime == "saturated":
        assert counts["saturated"] >= n, counts
    if regime == "taylor":
        assert counts["taylor"] >= 64 * len(NETS) * ((n + 2) // 3), counts     # every zero row's layer-1 pre-activations


def reference(flat, D, A, obs, eps=None):
    """float64: means, std, v_r, v_c and (with eps) act and logp, from the float32 inputs."""
    pol = TU.unpack(flat.double(), D, A)
    x = obs.double()
    with torch.no_grad():
        mean, std = O.actor_mean_std(pol, x)
        out = dict(mean=mean, std=std[0], v_r=O.critic_value(pol, "reward_critic", x), v_c=O.critic_value(pol, "cost_critic", x),
                   det_logp=O.normal_log_prob(mean, mean, std).sum(-1))
        if eps is not None:
            act = mean + eps.double() * std
            out.update(act=act, logp=O.normal_log_prob(act, mean, std).sum(-1))
    return out


# ============================================================ checks ============================================================
def _record(key, err):
    MEASURED[key] = max(MEASURED.get(key, 0.0), float(err))


def _check(key, got, want, scale=None):
    """max |got - want| / scale (default max |want|) against BAR[key]; exactly 0 where want is exactly 0."""
    got = torch.as_tensor(got).detach().double().cpu().reshape(-1)
    want = torch.as_tensor(want).detach().double().cpu().reshape(-1)
    assert got.shape == want.shape, (key, got.shape, want.shape)
    assert bool(torch.isfinite(got).all()), (key, "non-finite output")
    zero = want == 0
    assert bool((got[zero] == 0).all()), (key, "nonzero where float64 is exactly 0")
    scale = float(want.abs().max()) if scale is None else float(scale)
    err = float((got - want).abs().max()) / scale if scale > 0 else float((got - want).abs().max())
    _record(key, err)
    assert err <= BAR[key], (key, err, BAR[key])
    return err


def _check_logp(logp, want, e, act, mu, log_std):
    """The logp bar of the module docstring, row by row."""
    logp, want = logp.detach().double().cpu(), want.double()
    e, act, mu = e.double(), act.detach().double().cpu(), mu.detach().double().cpu()
    ls = log_std.double()
    sigma = torch.exp(ls)
    scale = (e * e / 2 + ls.abs() + 0.92).sum(-1)
    slack = (e.abs() * 2.0 ** -23 * torch.maximum(act.abs(), mu.abs()) / sigma).sum(-1)
    assert bool(torch.isfinite(logp).all()), "non-finite logp"
    err = float((((logp - want).abs() - slack).clamp(min=0) / scale).max())
    _record("logp", err)
    assert err <= BAR["logp"], ("logp", err, BAR["logp"])


def _check_kl(final_kl, kl_rows, reduce, A):
    """final_kl of a pass against the float64 mean of the per-row KL sums kl_rows, relative to their mean |value|."""
    want = float(kl_rows.mean()) / (A if reduce else 1)
    scale = float(kl_rows.abs().mean()) / (A if reduce else 1)
    err = abs(float(final_kl) - want) / scale
    _record("kl", err)
    assert err <= BAR["kl"], ("kl", err, BAR["kl"], float(final_kl), want)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if MEASURED:
        print("\nforward family: measured maxima (error / scale) and bars:\n" +
              "\n".join(f"  {k:6s} {v:.2e}  bar {BAR[k]:.1e}" for k, v in sorted(MEASURED.items())))


# ============================================================ CPU ============================================================
def test_philox_reproduces_random123_known_answers():
    """Random123's philox4x32_R(10) known-answer vectors (kat_vectors): the host restatement the sampler tests rely on."""
    kat = [((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
           ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
           ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
            (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1))]
    for ctr, key, want in kat:
        got = philox4x32_10(tuple(np.array([c], dtype=np.uint64) for c in ctr), key)
        assert tuple(int(x[0]) for x in got) == want, (ctr, key, [hex(int(x[0])) for x in got])


def test_host_box_muller_is_standard_normal():
    z = host_draws(20000, 4, PHILOX_SEED, 2 ** 32 + 1).reshape(-1)
    assert abs(z.mean()) < 0.02 and abs(z.std() - 1) < 0.02 and abs((z ** 4).mean() - 3) < 0.15
    assert not np.array_equal(host_draws(8, 2, PHILOX_SEED, 1), host_draws(8, 2, PHILOX_SEED, 2 ** 32))   # both offset words count


def test_input_regimes_reach_their_tanh_branches():
    """Every GPU case's inputs (S_multi stood in for by 4133 rows) take the tanh branches of its regime."""
    for _, D, A, n, regime in STEP_CASES + FULL_CASES:
        n = 4133 if n == "multi" else n
        flat, obs, eps = make_case(D, A, n, regime, 5)
        assert_regime(regime, tanh_regime_counts(flat, D, A, obs), n)
        assert bool((eps == 0).any()) and (n * A < 8 or float(eps.abs().max()) == 5.0)
        if regime == "log_std":
            assert set(flat[:A].tolist()) <= set(LOG_STD_EXTREMES)


def test_regimes_cover_the_log_std_extremes_on_every_kernel():
    for cases in (STEP_CASES, FULL_CASES):
        for kernel in ("wgmma", "ffma8", "ffma16"):
            seen = set()
            for k, D, A, _, regime in cases:
                if k == kernel and regime == "log_std":
                    seen |= {LOG_STD_EXTREMES[(j + D) % 4] for j in range(A)}
            assert seen == set(LOG_STD_EXTREMES), (kernel, seen)
            assert {r for k, _, _, _, r in cases if k == kernel} == set(REGIMES), kernel


# ============================================================ GPU helpers ============================================================
def _cuda():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    return torch.device("cuda:0")


def _lib():
    from safepo import _lib as L
    return L


def s_multi():
    """3 * 128 * SMs + 37 rows: at least three tiles per CTA of the wgmma grid (SMs CTAs x 128 rows) and of the FFMA grid
    (2 x SMs CTAs x 64 rows)."""
    return 3 * 128 * torch.cuda.get_device_properties(0).multi_processor_count + 37


def sentinel(*shape):
    return torch.full(shape, SENTINEL, dtype=torch.int32, device="cuda").view(torch.float32)


def untouched(t):
    return bool((t.view(torch.int32) == SENTINEL).all())


def ran_kernels(fn):
    """Run fn once and return the forward kernels it launched, as 'wgmma', 'ffma8' or 'ffma16'.  fn is captured into a CUDA
    graph whose kernel nodes name the kernels, then replayed: the same launches with the same arguments.  (torch.profiler
    drops kernel records once a process has opened many profiling sessions, and a test that sees none cannot tell which
    kernel ran.)"""
    g = torch.cuda.CUDAGraph(keep_graph=True)         # the captured graph stays for debug_dump; replay instantiates it
    g.enable_debug_mode()
    with torch.cuda.graph(g, capture_error_mode="relaxed"):
        fn()
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "graph.dot")
        with warnings.catch_warnings():
            warnings.filterwarnings("ignore", message="DEBUG: calling")    # torch announces every dump
            g.debug_dump(path)
        dot = open(path).read()
    g.replay()
    torch.cuda.synchronize()
    kinds = {"ffma" + ac for ac in re.findall(r"spo_ffma_forward_kernel(?:<|ILi)(\d+)", dot)}
    if "spo_tc_forward_kernel" in dot:
        kinds.add("wgmma")
    return kinds


def make_store(n, T, D, A):
    L = _lib()
    bufs = dict(obs=sentinel(n, T, D), act=sentinel(n, T, A), reward=sentinel(n, T), cost=sentinel(n, T),
                value_r=sentinel(n, T), value_c=sentinel(n, T), logp=sentinel(n, T), seg_end=sentinel(n, T),
                boot_r=sentinel(n, T), boot_c=sentinel(n, T))
    st = L.Rollout(*[bufs[k].data_ptr() for k in ("obs", "act", "reward", "cost", "value_r", "value_c", "logp", "seg_end",
                                                   "boot_r", "boot_c")], n, T)
    return st, bufs


def step(dims, flat, obs, n, eps=None, seed=0, offset=0, det=0, outs=(None,) * 4, store=None, t=0):
    L = _lib()
    L.check(L.lib().spo_policy_step(C.byref(dims), L.ptr(flat), obs.data_ptr(), L.ptr(eps), seed, offset, det, n,
                                    *[None if o is None else o.data_ptr() for o in outs],
                                    None if store is None else C.byref(store), t, L.stream()), "spo_policy_step")


def critic_values(dims, flat, obs, n, v_r, v_c):
    L = _lib()
    L.check(L.lib().spo_critic_values(C.byref(dims), L.ptr(flat), obs.data_ptr(), n, v_r.data_ptr(), v_c.data_ptr(), L.stream()),
            "spo_critic_values")


def actor_forward(dims, flat, obs, S, out):
    L = _lib()
    L.check(L.lib().spo_actor_forward(C.byref(dims), L.ptr(flat), obs.data_ptr(), S, out.data_ptr(), L.stream()), "spo_actor_forward")


def actor_kl(dims, flat, obs, S, old_mean, old_ls, ctrl, reduce=0, target=1e9):
    L = _lib()
    L.check(L.lib().spo_actor_kl(C.byref(dims), L.ptr(flat), obs.data_ptr(), L.ptr(old_mean), L.ptr(old_ls), S, reduce, target,
                                 L.ptr(ctrl), L.stream()), "spo_actor_kl")


def kl_accumulate(dims, flat, obs, S, old_mean, old_ls, ctrl):
    L = _lib()
    L.check(L.lib().spo_actor_kl_accumulate(C.byref(dims), L.ptr(flat), obs.data_ptr(), L.ptr(old_mean), L.ptr(old_ls), S,
                                            L.ptr(ctrl), L.stream()), "spo_actor_kl_accumulate")


def kl_finalize(ctrl, denom, target):
    L = _lib()
    L.check(L.lib().spo_kl_finalize(L.ptr(ctrl), denom, target, L.stream()), "spo_kl_finalize")


def read_ctrl(ctrl):
    torch.cuda.synchronize()
    return ctrl.cpu().numpy().view(_lib().CTRL_DTYPE)[0].copy()


def make_ctrl(**fields):
    arr = np.zeros(1, dtype=_lib().CTRL_DTYPE)
    for k, v in fields.items():
        arr[k] = v
    return torch.from_numpy(arr.view(np.uint8).copy()).to("cuda")


def old_distribution(mean64, log_std, seed):
    """A perturbed old distribution (float32) for the KL passes."""
    g = torch.Generator().manual_seed(seed)
    old_mean = (mean64 + 0.05 * torch.randn(mean64.shape, generator=g, dtype=torch.float64)).float().contiguous()
    old_ls = (log_std + 0.1 * torch.randn(log_std.shape, generator=g)).float().contiguous()
    return old_mean, old_ls


def kl_rows64(old_mean, old_ls, ref):
    return O.normal_kl(old_mean.double(), torch.exp(old_ls.double()).expand_as(ref["mean"]), ref["mean"], ref["std"].expand_as(ref["mean"])).sum(-1)


# ============================================================ GPU: rollout step and critic values ============================================================
def _step_cases():
    cases = []
    wg_n, wg_reg = (128, 129, 255, 1061), ("nominal", "taylor", "saturated", "wide", "nominal", "taylor", "wide", "saturated", "log_std")
    for i, (D, A) in enumerate((D, A) for D in (4, 28, 64) for A in (1, 3, 8)):
        cases.append(("wgmma", D, A, wg_n[i % 4] if i != 8 else 1061, wg_reg[i]))
    for i, n in enumerate((1, 63, 64, 65, 127)):
        cases.append(("ffma8", 4, (1, 8)[i % 2], n, REGIMES[i % 5]))
        cases.append(("ffma8", 64, (8, 1)[i % 2], n, REGIMES[(i + 2) % 5]))
    for i, (D, A) in enumerate((D, A) for D in (1, 3, 27, 65, 68, 128) for A in (1, 8)):
        cases.append(("ffma8", D, A, 129, ("log_std" if A == 8 and D in (27, 65) else REGIMES[i % 4])))
    for i, (D, A) in enumerate((D, A) for D in (4, 64, 128) for A in (9, 16)):
        cases.append(("ffma16", D, A, (1, 129)[i % 2], ("taylor", "log_std", "saturated", "wide", "nominal", "log_std")[i]))
    return cases


STEP_CASES = _step_cases()


@pytest.mark.gpu
@pytest.mark.parametrize("kernel,D,A,n,regime", STEP_CASES, ids=[f"{k}-D{d}-A{a}-n{n}-{r}" for k, d, a, n, r in STEP_CASES])
def test_step_and_critic_values_vs_float64(kernel, D, A, n, regime):
    """Sample with host eps, log-density, both critics, the deterministic step, spo_critic_values; the writes into slots 0
    and T-1 of a T = 3 store, the store-only call, and no write past n or into another slot."""
    dev = _cuda()
    L = _lib()
    T = 3
    flat, obs, eps = make_case(D, A, n, regime, 1000 * D + 10 * A + n)
    assert_regime(regime, tanh_regime_counts(flat, D, A, obs), n)
    ref = reference(flat, D, A, obs, eps)
    dims = L.dims(D, A)
    flat_d, obs_d, eps_d = flat.to(dev), obs.to(dev), eps.to(dev)
    outs = [sentinel(n + PAD, A), sentinel(n + PAD), sentinel(n + PAD), sentinel(n + PAD)]
    outs2 = [sentinel(n + PAD, A), sentinel(n + PAD), sentinel(n + PAD), sentinel(n + PAD)]
    det = [sentinel(n + PAD, A), sentinel(n + PAD), sentinel(n + PAD), sentinel(n + PAD)]
    vals = [sentinel(n + PAD), sentinel(n + PAD)]
    means = sentinel(n + PAD, A)
    same_means_kernel = kernel != "wgmma" or n >= 1024        # spo_actor_forward takes the wgmma kernel from 1024 rows
    st, sb = make_store(n, T, D, A)
    st2, sb2 = make_store(n, T, D, A)

    def run():
        step(dims, flat_d, obs_d, n, eps=eps_d, outs=outs, store=st, t=0)
        step(dims, flat_d, obs_d, n, eps=eps_d, store=st2, t=0)                       # store only: null output pointers
        step(dims, flat_d, obs_d, n, eps=eps_d, outs=outs2, store=st, t=T - 1)
        step(dims, flat_d, obs_d, n, det=1, outs=det)
        critic_values(dims, flat_d, obs_d, n, *vals)
        if same_means_kernel:
            actor_forward(dims, flat_d, obs_d, n, means)

    assert ran_kernels(run) == {kernel}
    for o in outs + outs2 + det + vals + [means]:
        assert untouched(o[n:]), "write past row n"
    act, logp, v_r, v_c = (o[:n] for o in outs)
    log_std = flat[:A]
    _check("act", act, ref["act"])
    _check_logp(logp, ref["logp"], eps, act, det[0][:n], log_std)
    _check("value", v_r, ref["v_r"])
    _check("value", v_c, ref["v_c"])
    _check("mean", det[0][:n], ref["mean"])
    _check_logp(det[1][:n], ref["det_logp"], torch.zeros(n, A), det[0][:n], det[0][:n], log_std)
    # bit-exact invariants
    for a, b in zip(outs, outs2):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), "two identical calls differ"
    assert torch.equal(vals[0][:n], v_r) and torch.equal(vals[1][:n], v_c), "spo_critic_values != the step's values"
    assert torch.equal(det[2][:n], v_r) and torch.equal(det[3][:n], v_c)
    if same_means_kernel:
        assert torch.equal(means[:n], det[0][:n]), "deterministic act != spo_actor_forward means"
    for t in (0, T - 1):
        assert torch.equal(sb["act"][:, t], act) and torch.equal(sb["logp"][:, t], logp), t
        assert torch.equal(sb["value_r"][:, t], v_r) and torch.equal(sb["value_c"][:, t], v_c), t
        assert torch.equal(sb["obs"][:, t].view(torch.int32), obs_d.view(torch.int32)), t
    for k in ("obs", "act", "value_r", "value_c", "logp"):
        assert torch.equal(sb2[k][:, 0].view(torch.int32), sb[k][:, 0].view(torch.int32)), k
        assert untouched(sb[k][:, 1]) and untouched(sb2[k][:, 1:]), k
    for k in ("reward", "cost", "seg_end", "boot_r", "boot_c"):
        assert untouched(sb[k]) and untouched(sb2[k]), k


# ============================================================ GPU: full-batch means and KL ============================================================
def _full_cases():
    cases = []
    wg_reg = ("wide", "nominal", "taylor", "saturated", "log_std", "wide", "taylor", "nominal", "log_std")
    for i, (D, A) in enumerate((D, A) for D in (4, 28, 64) for A in (1, 3, 8)):
        cases.append(("wgmma", D, A, (1024, 1025, "multi")[i % 3], wg_reg[i]))
    cases += [("ffma8", 64, 1, 1023, "saturated"), ("ffma8", 64, 8, 1023, "wide")]
    for i, (D, A) in enumerate((D, A) for D in (1, 3, 27, 65, 68, 128) for A in (1, 8)):
        cases.append(("ffma8", D, A, (1025, "multi")[i % 2], ("log_std" if A == 8 and D in (3, 68) else REGIMES[i % 4])))
    for i, (D, A) in enumerate((D, A) for D in (4, 64, 128) for A in (9, 16)):
        cases.append(("ffma16", D, A, (1025, "multi")[i % 2], ("log_std", "taylor", "saturated", "log_std", "wide", "nominal")[i]))
    return cases


FULL_CASES = _full_cases()


@pytest.mark.gpu
@pytest.mark.parametrize("kernel,D,A,S,regime", FULL_CASES, ids=[f"{k}-D{d}-A{a}-S{s}-{r}" for k, d, a, s, r in FULL_CASES])
def test_means_and_kl_vs_float64(kernel, D, A, S, regime):
    """spo_actor_forward and spo_actor_kl (reduce 0 and 1, each closing its pass on a fresh control block)."""
    dev = _cuda()
    L = _lib()
    S = s_multi() if S == "multi" else S
    flat, obs, _ = make_case(D, A, S, regime, 1000 * D + 10 * A + 7)
    assert_regime(regime, tanh_regime_counts(flat, D, A, obs), S)
    ref = reference(flat, D, A, obs)
    old_mean, old_ls = old_distribution(ref["mean"], flat[:A], D + A)
    kl64 = kl_rows64(old_mean, old_ls, ref)
    dims = L.dims(D, A)
    flat_d, obs_d, om_d, ols_d = flat.to(dev), obs.to(dev), old_mean.to(dev), old_ls.to(dev)
    means = sentinel(S + PAD, A)
    ctrls = [make_ctrl(), make_ctrl()]

    def run():
        actor_forward(dims, flat_d, obs_d, S, means)
        for reduce in (0, 1):
            actor_kl(dims, flat_d, obs_d, S, om_d, ols_d, ctrls[reduce], reduce=reduce)

    assert ran_kernels(run) == {kernel}
    assert untouched(means[S:]), "write past row S"
    _check("mean", means[:S], ref["mean"])
    for reduce in (0, 1):
        r = read_ctrl(ctrls[reduce])
        _check_kl(r["final_kl"], kl64, reduce, A)
        assert (int(r["passes"]), int(r["stop"]), int(r["ticket"]), float(r["kl_sum"])) == (1, 0, 0, 0.0), r


# ============================================================ GPU: wgmma against FFMA ============================================================
@pytest.mark.gpu
@pytest.mark.parametrize("D,A,regime", [(28, 3, "wide"), (64, 8, "saturated"), (4, 1, "nominal")])
def test_wgmma_and_ffma_agree_on_the_same_rows(D, A, regime):
    """1061 rows in one call (wgmma) against the same rows in chunks of 127 (FFMA): step outputs and means."""
    dev = _cuda()
    L = _lib()
    n, chunk = 1061, 127
    flat, obs, eps = make_case(D, A, n, regime, 31 * D + A)
    ref = reference(flat, D, A, obs, eps)
    dims = L.dims(D, A)
    flat_d, obs_d, eps_d = flat.to(dev), obs.to(dev), eps.to(dev)
    whole = [torch.empty(n, A, device=dev), torch.empty(n, device=dev), torch.empty(n, device=dev), torch.empty(n, device=dev)]
    parts = [torch.empty_like(o) for o in whole]
    m_whole, m_parts = torch.empty(n, A, device=dev), torch.empty(n, A, device=dev)
    k1 = ran_kernels(lambda: (step(dims, flat_d, obs_d, n, eps=eps_d, outs=whole), actor_forward(dims, flat_d, obs_d, n, m_whole)))

    def chunks():
        for i in range(0, n, chunk):
            m = min(chunk, n - i)
            step(dims, flat_d, obs_d[i:i + m], m, eps=eps_d[i:i + m], outs=[o[i:i + m] for o in parts])
            actor_forward(dims, flat_d, obs_d[i:i + m], m, m_parts[i:i + m])

    k2 = ran_kernels(chunks)
    assert (k1, k2) == ({"wgmma"}, {"ffma8"})
    for key, a, b, want in (("act", 0, 0, ref["act"]), ("v_r", 2, 2, ref["v_r"]), ("v_c", 3, 3, ref["v_c"])):
        _check("cross", whole[a], parts[b], scale=float(want.abs().max()))
    _check("cross", m_whole, m_parts, scale=float(ref["mean"].abs().max()))
    _check_logp(whole[1], parts[1].double().cpu(), eps, whole[0], m_whole, flat[:A])


# ============================================================ GPU: the in-kernel sampler ============================================================
SAMPLER_CASES = ([("wgmma", 28, A, n) for n in (129, 70000) for A in (1, 3, 8)] +
                 [("ffma8", 27, A, n) for n in (1, 129, 70000) for A in (1, 3, 8)] +
                 [("ffma16", 64, A, n) for n in (1, 129, 70000) for A in (9, 16)])


def _recover_z(act, mu, log_std):
    """z = (act - mean_det) / sigma in float64, and the bar: ulp(|act|) / sigma + Z_ULPS ulps of |z|."""
    act, mu = act.detach().cpu().numpy().astype(np.float64), mu.detach().cpu().numpy().astype(np.float64)
    sigma = torch.exp(log_std.float()).numpy().astype(np.float64)
    z = (act - mu) / sigma
    return z, np.spacing(np.abs(act).astype(np.float32)).astype(np.float64) / sigma


def _check_draws(z, act_ulp, want):
    tol = act_ulp + Z_ULPS * np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)
    bad = np.abs(z - want) > tol
    assert not bad.any(), (int(bad.sum()), np.argwhere(bad)[:4].tolist(), z[bad][:4], want[bad][:4])


@pytest.mark.gpu
@pytest.mark.parametrize("kernel,D,A,n", SAMPLER_CASES, ids=[f"{k}-D{d}-A{a}-n{n}" for k, d, a, n in SAMPLER_CASES])
def test_in_kernel_sampler_matches_host_philox_box_muller(kernel, D, A, n):
    """Element by element: draw (row, j) is component j & 1 of Philox counter (row, j >> 1, offset lo, offset hi) under the
    seed, at offsets either side of 2^32, rows past 2^16, odd act_dim and pair 7."""
    dev = _cuda()
    L = _lib()
    flat, obs, _ = make_case(D, A, n, "nominal", 77 + A)
    dims = L.dims(D, A)
    flat_d, obs_d = flat.to(dev), obs.to(dev)
    det = torch.empty(n, A, device=dev)
    acts = [torch.empty(n, A, device=dev) for _ in PHILOX_OFFSETS]

    def run():
        step(dims, flat_d, obs_d, n, det=1, outs=(det, None, None, None))
        for off, a in zip(PHILOX_OFFSETS, acts):
            step(dims, flat_d, obs_d, n, seed=PHILOX_SEED, offset=off, outs=(a, None, None, None))

    assert ran_kernels(run) == {kernel}
    for off, a in zip(PHILOX_OFFSETS, acts):
        z, act_ulp = _recover_z(a, det, flat[:A])
        _check_draws(z, act_ulp, host_draws(n, A, PHILOX_SEED, off))


@pytest.mark.gpu
@pytest.mark.parametrize("D,A", [(28, 3), (64, 8)])
def test_wgmma_and_ffma_draw_the_same_numbers(D, A):
    dev = _cuda()
    L = _lib()
    n, m = 1061, 127
    flat, obs, _ = make_case(D, A, n, "nominal", 3)
    dims = L.dims(D, A)
    flat_d, obs_d = flat.to(dev), obs.to(dev)
    det, a_wg = torch.empty(n, A, device=dev), torch.empty(n, A, device=dev)
    det_f, a_ff = torch.empty(m, A, device=dev), torch.empty(m, A, device=dev)
    k1 = ran_kernels(lambda: (step(dims, flat_d, obs_d, n, det=1, outs=(det, None, None, None)),
                              step(dims, flat_d, obs_d, n, seed=PHILOX_SEED, offset=2 ** 32 + 1, outs=(a_wg, None, None, None))))
    k2 = ran_kernels(lambda: (step(dims, flat_d, obs_d, m, det=1, outs=(det_f, None, None, None)),
                              step(dims, flat_d, obs_d, m, seed=PHILOX_SEED, offset=2 ** 32 + 1, outs=(a_ff, None, None, None))))
    assert (k1, k2) == ({"wgmma"}, {"ffma8"})
    z_wg, u_wg = _recover_z(a_wg[:m], det[:m], flat[:A])
    z_ff, u_ff = _recover_z(a_ff, det_f, flat[:A])
    tol = u_wg + u_ff + 2 * Z_ULPS * np.spacing(np.abs(z_wg).astype(np.float32)).astype(np.float64)
    assert bool((np.abs(z_wg - z_ff) <= tol).all()), float(np.abs(z_wg - z_ff).max())


@pytest.mark.gpu
def test_successive_steps_use_successive_offsets():
    """ActorVCritic.step draws with offset k, then k + 1, under its seed."""
    dev = _cuda()
    from safepo.common.model import ActorVCritic
    torch.manual_seed(4)
    D, A, n = 28, 3, 300
    pol = ActorVCritic(D, A).to(dev)
    with torch.no_grad():
        pol.actor.log_std.copy_(torch.tensor([-0.7, 0.0, 0.4]))
    obs = torch.randn(n, D, device=dev)
    mu = pol.step(obs, deterministic=True)[0]
    k = pol._philox_offset
    a1, a2 = pol.step(obs)[0], pol.step(obs)[0]
    assert pol._philox_offset == k + 2
    for a, off in ((a1, k + 1), (a2, k + 2)):
        z, act_ulp = _recover_z(a, mu, pol.actor.log_std.detach().cpu())
        _check_draws(z, act_ulp, host_draws(n, A, pol._philox_seed, off))


# ============================================================ GPU: the KL pass control block ============================================================
def _kl_setup(D, A, S, seed):
    flat, obs, _ = make_case(D, A, S, "nominal", seed)
    ref = reference(flat, D, A, obs)
    old_mean, old_ls = old_distribution(ref["mean"], flat[:A], seed)
    return flat, obs, old_mean, old_ls, kl_rows64(old_mean, old_ls, ref)


@pytest.mark.gpu
@pytest.mark.parametrize("S,kernel", [(1023, "ffma8"), (1025, "wgmma")])
def test_kl_stop_decision_matches_the_written_kl(S, kernel):
    """After every launch stop == (final_kl > target_kl) for the final_kl that launch wrote, with the target equal to a
    recorded final_kl and one fp32 ulp below it."""
    dev = _cuda()
    L = _lib()
    D, A = 28, 3
    flat, obs, old_mean, old_ls, kl64 = _kl_setup(D, A, S, 11)
    dims = L.dims(D, A)
    flat_d, obs_d, om_d, ols_d = flat.to(dev), obs.to(dev), old_mean.to(dev), old_ls.to(dev)
    ctrl = make_ctrl()
    assert ran_kernels(lambda: actor_kl(dims, flat_d, obs_d, S, om_d, ols_d, ctrl)) == {kernel}
    f0 = np.float32(read_ctrl(ctrl)["final_kl"])
    _check_kl(f0, kl64, 0, A)
    stops = []
    for target in (f0, np.nextafter(f0, np.float32(-np.inf))):
        for _ in range(3):
            ctrl = make_ctrl()
            actor_kl(dims, flat_d, obs_d, S, om_d, ols_d, ctrl, target=float(target))
            r = read_ctrl(ctrl)
            assert int(r["stop"]) == int(np.float32(r["final_kl"]) > np.float32(target)), (r, target)
            assert int(r["passes"]) == 1 and int(r["ticket"]) == 0 and float(r["kl_sum"]) == 0.0, r
            stops.append(int(r["stop"]))
    assert stops[:3].count(0) > 0 and stops[3:].count(1) > 0, stops     # the recorded value recurs in each run


@pytest.mark.gpu
def test_one_control_block_across_kernels_with_different_grids():
    """Passes on FFMA (S = 1023, 16 CTAs), wgmma (S = 1025, 9 CTAs), FFMA again, on one control block: each closes (ticket
    and kl_sum back to 0), passes counts 3."""
    dev = _cuda()
    L = _lib()
    D, A = 28, 3
    flat, obs, old_mean, old_ls, kl64 = _kl_setup(D, A, 1025, 12)
    dims = L.dims(D, A)
    flat_d, obs_d, om_d, ols_d = flat.to(dev), obs.to(dev), old_mean.to(dev), old_ls.to(dev)
    ctrl = make_ctrl()
    for i, (S, kernel) in enumerate(((1023, "ffma8"), (1025, "wgmma"), (1023, "ffma8"))):
        assert ran_kernels(lambda: actor_kl(dims, flat_d, obs_d, S, om_d, ols_d, ctrl)) == {kernel}
        r = read_ctrl(ctrl)
        assert (int(r["passes"]), int(r["ticket"]), float(r["kl_sum"]), int(r["stop"])) == (i + 1, 0, 0.0, 0), (i, r)
        _check_kl(r["final_kl"], kl64[:S], 0, A)


@pytest.mark.gpu
def test_kl_launches_after_stop_leave_the_control_block_alone():
    """With stop set, spo_actor_kl (both kernels) and spo_actor_kl_accumulate change nothing; spo_kl_finalize only zeroes
    kl_sum."""
    dev = _cuda()
    L = _lib()
    D, A = 28, 3
    flat, obs, old_mean, old_ls, _ = _kl_setup(D, A, 1025, 13)
    dims = L.dims(D, A)
    flat_d, obs_d, om_d, ols_d = flat.to(dev), obs.to(dev), old_mean.to(dev), old_ls.to(dev)
    fields = dict(loss_sum=[1.0, 2.0, 3.0], kl_sum=0.375, steps=7, stop=1, passes=2, final_kl=0.5, ticket=0, extra_sumsq=0.25)
    ctrl = make_ctrl(**fields)
    before = ctrl.clone()
    for S in (1023, 1025):
        actor_kl(dims, flat_d, obs_d, S, om_d, ols_d, ctrl, target=0.0)
        kl_accumulate(dims, flat_d, obs_d, S, om_d, ols_d, ctrl)
    torch.cuda.synchronize()
    assert torch.equal(ctrl, before), (read_ctrl(ctrl), read_ctrl(before))
    kl_finalize(ctrl, 1025.0, 0.0)
    want = make_ctrl(**dict(fields, kl_sum=0.0))
    assert torch.equal(ctrl, want), (read_ctrl(ctrl), read_ctrl(want))


@pytest.mark.gpu
def test_kl_split_over_three_shards_and_finalize():
    """spo_actor_kl_accumulate on shards of 1023 (FFMA), 1061 (wgmma) and 5 (FFMA) rows, then spo_kl_finalize(2089): the
    sum and the mean against float64, and the mean against the shards' own sums up to fp64 reassociation."""
    dev = _cuda()
    L = _lib()
    D, A = 28, 3
    S = 1023 + 1061 + 5
    flat, obs, old_mean, old_ls, kl64 = _kl_setup(D, A, S, 14)
    dims = L.dims(D, A)
    flat_d, obs_d, om_d, ols_d = flat.to(dev), obs.to(dev), old_mean.to(dev), old_ls.to(dev)
    shards = ((0, 1023, "ffma8"), (1023, 1061, "wgmma"), (2084, 5, "ffma8"))
    ctrl = make_ctrl()
    own = []
    for r0, m, kernel in shards:
        c1 = make_ctrl()
        assert ran_kernels(lambda: (kl_accumulate(dims, flat_d, obs_d[r0:r0 + m], m, om_d[r0:r0 + m], ols_d, ctrl),
                                    kl_accumulate(dims, flat_d, obs_d[r0:r0 + m], m, om_d[r0:r0 + m], ols_d, c1))) == {kernel}
        own.append(float(read_ctrl(c1)["kl_sum"]))
    r = read_ctrl(ctrl)
    assert (int(r["passes"]), int(r["stop"]), int(r["ticket"])) == (0, 0, 0), r
    scale = float(kl64.abs().mean())
    err = abs(float(r["kl_sum"]) - float(kl64.sum())) / (S * scale)
    _record("kl", err)
    assert err <= BAR["kl"], err
    assert abs(float(r["kl_sum"]) - sum(own)) <= 1e-12 * abs(sum(own)), (float(r["kl_sum"]), own)
    target = np.float32(float(kl64.mean()))
    kl_finalize(ctrl, float(S), float(target))
    f = read_ctrl(ctrl)
    _check_kl(f["final_kl"], kl64, 0, A)
    whole = np.float32(sum(own) / S)
    assert abs(float(f["final_kl"]) - float(whole)) <= float(np.spacing(whole)), (float(f["final_kl"]), float(whole))
    assert (int(f["passes"]), float(f["kl_sum"])) == (1, 0.0), f
    assert int(f["stop"]) == int(np.float32(f["final_kl"]) > target), (f, target)


# ============================================================ GPU: misaligned observations ============================================================
@pytest.mark.gpu
def test_misaligned_obs_runs_the_scalar_path():
    """obs_dim 27 read one float at a time: a view one float into its allocation runs, meets the float64 bars and equals
    the aligned copy bit for bit."""
    dev = _cuda()
    L = _lib()
    D, A, n = 27, 3, 1100
    flat, obs, eps = make_case(D, A, n, "nominal", 21)
    ref = reference(flat, D, A, obs, eps)
    old_mean, old_ls = old_distribution(ref["mean"], flat[:A], 21)
    kl64 = kl_rows64(old_mean, old_ls, ref)
    dims = L.dims(D, A)
    flat_d, eps_d, om_d, ols_d = flat.to(dev), eps.to(dev), old_mean.to(dev), old_ls.to(dev)
    backing = torch.empty(n * D + 1, device=dev)
    mis = backing[1:].view(n, D)
    mis.copy_(obs)
    assert mis.data_ptr() % 16 == 4
    aligned = obs.to(dev)
    res = []
    for o in (mis, aligned):
        outs = [torch.empty(n, A, device=dev), torch.empty(n, device=dev), torch.empty(n, device=dev), torch.empty(n, device=dev)]
        vals = [torch.empty(n, device=dev), torch.empty(n, device=dev)]
        means = torch.empty(n, A, device=dev)
        ctrl = make_ctrl()

        def run():
            step(dims, flat_d, o, n, eps=eps_d, outs=outs)
            critic_values(dims, flat_d, o, n, *vals)
            actor_forward(dims, flat_d, o, n, means)
            actor_kl(dims, flat_d, o, n, om_d, ols_d, ctrl)

        assert ran_kernels(run) == {"ffma8"}
        res.append(outs + vals + [means, ctrl])
    act, logp, v_r, v_c = res[0][:4]
    _check("act", act, ref["act"])
    _check_logp(logp, ref["logp"], eps, act, res[0][6], flat[:A])
    _check("value", v_r, ref["v_r"])
    _check("value", v_c, ref["v_c"])
    _check("mean", res[0][6], ref["mean"])
    _check_kl(read_ctrl(res[0][7])["final_kl"], kl64, 0, A)
    for a, b in zip(res[0][:7], res[1][:7]):
        assert torch.equal(a, b)


@pytest.mark.gpu
def test_actor_v_critic_accepts_a_misaligned_view():
    """At obs_dim 60 the kernels read float4 rows and refuse a misaligned array; ActorVCritic copies such a view first and
    gives what the aligned tensor gives."""
    dev = _cuda()
    from safepo.common.model import ActorVCritic
    torch.manual_seed(6)
    D, A, n = 60, 2, 1061
    pol = ActorVCritic(D, A).to(dev)
    backing = torch.randn(n * D + 1, device=dev)
    mis = backing[1:].view(n, D)
    aligned = mis.clone()
    assert mis.data_ptr() % 16 == 4 and aligned.data_ptr() % 16 == 0
    eps = torch.randn(n, A, device=dev)
    got = pol.step(mis, eps=eps) + pol.values(mis) + (pol.actor_mean(mis),)
    want = pol.step(aligned, eps=eps) + pol.values(aligned) + (pol.actor_mean(aligned),)
    for a, b in zip(got, want):
        assert torch.equal(a, b)
    from safepo import _lib as L
    with pytest.raises(L.SpoError, match="16-byte aligned"):
        L.check(L.lib().spo_actor_forward(C.byref(pol.dims), L.ptr(pol.flat), mis.data_ptr(), n, want[-1].data_ptr(), L.stream()),
                "spo_actor_forward")
