"""The single-agent data path between ``env.step`` and the update, and the conjugate-gradient vector kernels, per output
against float64 at their shape and branch edges.

* ``spo_store_transition`` (csrc/spo_rollout.cu): bit for bit against the segment / bootstrap rule of ppo_lag.py:198-234,
  every term / trunc / epoch_end combination, ``final_v`` given and NULL, slots of other steps untouched, N across CTAs.
* ``spo_gae_dual`` (csrc/spo_gae.cu): the sequential mode bit for bit against ``gae_dual_np``; the scan mode per element
  against the float64 recurrence, with path ends on and either side of every thread (4 steps), warp (128) and tile (512)
  edge counted from T - 1, discounts 0 / 0.94 / 1, a cancelling regime, large values with small rewards, zero bootstraps.
* ``spo_adv_stats`` / ``spo_adv_apply``: the statistics against float64 sums across the grid-stride edge; the apply step
  bit for bit against a host fp32 restatement on the device's own statistics, every flag combination, ``mixed`` NULL.
* ``spo_obs_normalize`` / ``spo_action_rescale`` (csrc/spo_envio.cu) against oracle/envio.py.
* ``spo_cg_begin`` / ``spo_cg_update`` (csrc/spo_trust.cu) driven with z = M p for a float64 SPD matrix: one step against a
  float64 restatement of cpo.py:92-105, the whole solve against ``conjugate_gradients``, the residual stop, pz = 0.

The argument refusals run without a GPU.  Run with ``-s`` to see the measured maxima."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import envio
from oracle import spo_oracle as O

# Bars: error / scale, each at most 4x the largest error measured over this file's matrix on one H100 80GB HBM3 (in
# brackets).  gae_scan_c is the c of |scan - ref| <= ulp32(ref) + c * L * 2^-53 * sum|terms on the path suffix| (L the
# suffix length): the scan and the sequential recurrence associate the float64 carry differently, so where an advantage
# is a near-cancellation of its suffix they differ by many fp32 ulps (256 in the 'cancel' regime, reported per regime and
# per discount as ulps[...] and c[...]).
BAR = dict(
    gae_scan_c=2.5,        # [6.9e-1]
    adv_stats=3e-15,       # [8.2e-16] each sum relative to the sum of |terms|
    obs_stats=8e-15,       # [2.2e-15] running mean and var, relative
    obs_out_ulp=1.0,       # [5.0e-1]  |out - float64| in fp32 ulps of the float64 result
    rescale=1e-6,          # [2.6e-7]  relative to max(|low|, |high|) of the dimension
    cg_step=6e-7,          # [1.7e-7]  x, r, p, rdotr of one step, relative to the size of the terms
    cg_solve=8e-7,         # [2.2e-7]  x after ten steps, relative to max |x|
    cg_eps=4e-7)           # [1.2e-7]  the pz = 0 step, relative
MEASURED = {}
NOTES = {}                 # measured quantities without a bar (reported at teardown)

U64 = 2.0 ** -53


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs CUDA")
    return torch.device("cuda:0")


def _lib():
    from safepo import _lib as L
    return L


def _call(name, *args):
    L = _lib()
    L.check(getattr(L.lib(), name)(*args), name)


def _ptr(t):
    return _lib().ptr(t)


def _stream():
    return _lib().stream()


def _record(key, err):
    MEASURED[key] = max(MEASURED.get(key, 0.0), float(err))
    assert err <= BAR[key], (key, err, BAR[key])


def _note(key, val):
    NOTES[key] = max(NOTES.get(key, 0.0), float(val))


def _check(key, got, want, scale):
    got = np.asarray(torch.as_tensor(got).detach().double().cpu()).reshape(-1)
    want = np.asarray(want, dtype=np.float64).reshape(-1)
    assert got.shape == want.shape, (key, got.shape, want.shape)
    assert np.isfinite(got).all(), key
    err = float(np.abs(got - want).max()) / scale if scale > 0 else float(np.abs(got - want).max())
    _record(key, err)
    return err


def _ulp32(x):
    """Spacing of fp32 at |x| (x float64): one unit in the last place of the fp32 nearest to x."""
    return np.spacing(np.abs(np.asarray(x, dtype=np.float64)).astype(np.float32)).astype(np.float64)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if MEASURED or NOTES:
        lines = [f"  {k:14s} {v:.2e}  bar {BAR[k]:.1e}" for k, v in sorted(MEASURED.items())]
        lines += [f"  {k:14s} {v:.2e}" for k, v in sorted(NOTES.items())]
        print("\nmeasured maxima (error / scale) and bars:\n" + "\n".join(lines))


# ============================================================ CPU ============================================================
def test_store_transition_and_adv_apply_refuse_bad_arguments():
    """Refused before any launch (the pointers are never dereferenced): a slot outside [0, steps), epoch_end without
    next_v, one of final_v_r / final_v_c without the other; spo_adv_apply with a null pointer or count <= 0."""
    L = _lib()
    lib = L.lib()
    X = 0x200000
    r = L.Rollout(obs=X, act=X, reward=X, cost=X, value_r=X, value_c=X, logp=X, seg_end=X, boot_r=X, boot_c=X, num_envs=4, steps=3)
    store = lambda t, ee, nv, fr, fc: lib.spo_store_transition(C.byref(r), t, X, X, X, X, ee, nv, nv, fr, fc, None)
    for t in (-1, 3, 1 << 20):
        assert store(t, 0, None, None, None) == -1 and b"slot t=" in lib.spo_last_error(), t
    assert store(2, 1, None, None, None) == -1 and b"epoch_end needs next_v" in lib.spo_last_error()
    for fr, fc in ((X, None), (None, X)):
        assert store(1, 0, None, fr, fc) == -1 and b"final_v_r/final_v_c" in lib.spo_last_error()
    for args in ((None, X, 8, X), (X, None, 8, X), (X, X, 8, None), (X, X, 0, X), (X, X, -5, X)):
        a, c, n, st = args
        assert lib.spo_adv_apply(a, c, n, st, 1, 1, 0.5, 1.5, None, None) == -1, args
        assert b"spo_adv_apply" in lib.spo_last_error()


def _edge_positions(T, steps=(4, 128, 512)):
    """Slots on, and one step either side of, every edge T-1-k*step (thread 4, warp 128, tile 512) of the scan."""
    pos = set()
    for step in steps:
        for e in range(T - 1, -1, -step):
            pos.update(t for t in (e - 1, e, e + 1) if 0 <= t < T)
    return sorted(pos)


def _gae_f64(rew, cost, v_r, v_c, seg_end, boot_r, boot_c, gamma, lam, lam_c):
    """``gae_dual_np`` with its float64 carry kept: for reward and cost, the float64 advantage, the float64 target
    (advantage + value), the discounted sum of |delta| over the path suffix and the suffix length."""
    seg = np.asarray(seg_end).astype(bool).copy()
    N, T = rew.shape
    seg[:, -1] = True
    g32 = np.float32(gamma)
    out = []
    for r, v, boot, l in ((rew, v_r, boot_r, lam), (cost, v_c, boot_c, lam_c)):
        disc = gamma * l
        acc, mag, ln = (np.zeros((N, T)) for _ in range(3))
        a, m, k = np.zeros(N), np.zeros(N), np.zeros(N)
        for t in range(T - 1, -1, -1):
            end = seg[:, t]
            vnext = np.where(end, boot[:, t], v[:, t + 1] if t + 1 < T else boot[:, t]).astype(np.float32)
            d = ((r[:, t] + g32 * vnext).astype(np.float32) - v[:, t]).astype(np.float32).astype(np.float64)
            a = np.where(end, d, d + disc * a)
            m = np.where(end, np.abs(d), np.abs(d) + disc * m)
            k = np.where(end, 1.0, k + 1.0)
            acc[:, t], mag[:, t], ln[:, t] = a, m, k
        out.append((acc, acc + v.astype(np.float64), mag, ln))
    return out


REGIMES = ("cancel", "offset", "terminal")
# (gamma, lam, lam_c): discounts gamma*lam for reward / cost of (0.94, 1), (1, 0), (0, 0.94)
DISCOUNTS = ((1.0, 0.94, 1.0), (1.0, 1.0, 0.0), (0.94, 0.0, 1.0))


def _gae_layout(rng, N, T):
    """Path ends per env.  N = 300: env 0 only the last step (its seg_end[T-1] left 0: the kernel closes it), env 1 every
    step, the rest share every slot of _edge_positions(T) between them in random order.  N = 3: only-last, every step,
    the warp and tile edges.  N = 1: the tile edges."""
    seg = np.zeros((N, T), np.uint8)
    if N == 1:
        rows = [_edge_positions(T, (512,))]
    elif N == 3:
        rows = [[], list(range(T)), _edge_positions(T, (128, 512))]
    else:
        rows = [[], list(range(T))] + [list(x) for x in np.array_split(rng.permutation(_edge_positions(T)), N - 2)]
    for i, p in enumerate(rows):
        seg[i, p] = 1
    if N > 2:
        seg[2:, T - 1] = rng.random(N - 2) < 0.5
    return seg


def _gae_inputs(rng, seg, regime):
    """One regime's inputs for the layout ``seg``: 'cancel' rewards and costs of size 1e3 and alternating sign on a
    random half of the steps and of size 1e-5 on the others, values around 1e-6 (the advantages are small differences of
    partial sums around 1e3, and the float64 carry rounds), 'offset' values around 1e3 with rewards around 1e-2,
    'terminal' every path end terminal (zero bootstrap).  Elsewhere half the ends are terminal.  Bootstraps at slots that
    are not path ends are 1e6: the kernels must not read them."""
    N, T = seg.shape
    randn = lambda: rng.standard_normal((N, T))
    if regime == "cancel":
        big = rng.random((N, T)) < 0.5
        sign = np.where(np.cumsum(big, axis=1) % 2 == 0, 1.0, -1.0)
        rew, cost = (np.where(big, s * 1e3 + 1e-2 * randn(), 1e-5 * randn()) for s in (sign, -sign))
        v_r, v_c, br, bc = 1e-6 * randn(), 1e-6 * randn(), 1e-6 * randn(), 1e-6 * randn()
    elif regime == "offset":
        rew, cost = 1e-2 * randn(), 1e-2 * rng.random((N, T))
        v_r, v_c, br, bc = 1e3 + randn(), 1e3 + randn(), 1e3 + randn(), 1e3 + randn()
    else:
        rew, cost = randn(), (rng.random((N, T)) < 0.05).astype(np.float64)
        v_r, v_c, br, bc = randn(), randn(), randn(), randn()
    end = seg.astype(bool).copy()
    end[:, -1] = True
    live = end & (rng.random((N, T)) < 0.5) if regime != "terminal" else np.zeros((N, T), bool)
    br, bc = (np.where(live, b, np.where(end, 0.0, 1e6)) for b in (br, bc))
    f = lambda x: np.ascontiguousarray(x, dtype=np.float32)
    return dict(rew=f(rew), cost=f(cost), v_r=f(v_r), v_c=f(v_c), seg_end=seg, boot_r=f(br), boot_c=f(bc))


def test_gae_f64_helper_rounds_to_gae_dual_np():
    """The float64 GAE used as the scan's reference is gae_dual_np's recurrence: rounded to fp32 it equals it bit for
    bit, for every discount pair and regime, with path ends on the scan's edges."""
    rng = np.random.default_rng(5)
    for T in (1, 5, 130, 515):
        for N in (1, 3, 7):
            seg = _gae_layout(rng, N, T) if N != 7 else (rng.random((N, T)) < 0.1).astype(np.uint8)
            for regime in REGIMES:
                c = _gae_inputs(rng, seg, regime)
                for gamma, lam, lam_c in DISCOUNTS:
                    want = O.gae_dual_np(c["rew"], c["cost"], c["v_r"], c["v_c"], c["seg_end"], c["boot_r"], c["boot_c"], gamma, lam, lam_c)
                    (ar, tr, _, _), (ac, tc, _, _) = _gae_f64(c["rew"], c["cost"], c["v_r"], c["v_c"], c["seg_end"], c["boot_r"],
                                                              c["boot_c"], gamma, lam, lam_c)
                    for got, w in zip((ar, ac, tr, tc), want):
                        assert np.array_equal(got.astype(np.float32), w.numpy()), (T, N, regime, gamma, lam, lam_c)


# ============================================================ GPU ============================================================
# ---- spo_store_transition ----
def _segment_rule(term, trunc, epoch_end, next_v, final_v):
    """ppo_lag.py:198-234 per env: a path closes on epoch_end, done or time_out; its bootstrap is 0 when done, else the
    value of the next observation at the epoch end, overridden by the value of the final observation on a time-out."""
    end = epoch_end or term or trunc
    boot = (0.0, 0.0)
    if end and not term:
        if epoch_end:
            boot = next_v
        if trunc and final_v is not None:
            boot = final_v
    return int(end), boot


@pytest.mark.gpu
@pytest.mark.parametrize("N", [1, 129, 300])
def test_store_transition_bit_exact(N):
    """Slots t = 0, mid, T - 1; term / trunc given as any nonzero byte; next_v passed but unused when the epoch goes on."""
    dev = _cuda()
    L = _lib()
    T = 6
    g = torch.Generator().manual_seed(40 + N)
    bufs = {k: torch.randn(N, T, generator=g) for k in ("reward", "cost", "boot_r", "boot_c")}
    bufs["seg_end"] = torch.full((N, T), 7, dtype=torch.uint8)
    want = {k: v.clone() for k, v in bufs.items()}
    dbuf = {k: v.to(dev) for k, v in bufs.items()}
    r = L.Rollout(reward=_ptr(dbuf["reward"]), cost=_ptr(dbuf["cost"]), seg_end=_ptr(dbuf["seg_end"]), boot_r=_ptr(dbuf["boot_r"]),
                  boot_c=_ptr(dbuf["boot_c"]), num_envs=N, steps=T)
    seen = set()
    for t in (0, T // 2, T - 1):
        for epoch_end, nv_given, fv_given in ((0, 0, 0), (0, 1, 0), (0, 0, 1), (0, 1, 1), (1, 1, 0), (1, 1, 1)):
            for shift in range(4):
                rew, cost = torch.randn(N, generator=g), torch.randn(N, generator=g)
                code = (torch.arange(N) + shift) % 4                   # env n: term = bit 0, trunc = bit 1
                term = ((code & 1) * torch.randint(1, 256, (N,), generator=g)).to(torch.uint8)     # any nonzero byte is set
                trunc = ((code >> 1) * torch.randint(1, 256, (N,), generator=g)).to(torch.uint8)
                nv = (torch.randn(N, generator=g), torch.randn(N, generator=g))
                fv = (torch.randn(N, generator=g), torch.randn(N, generator=g))
                dn = [x.to(dev) for x in nv] if nv_given else [None, None]
                dfv = [x.to(dev) for x in fv] if fv_given else [None, None]
                args = [x.to(dev) for x in (rew, cost, term, trunc)]
                _call("spo_store_transition", C.byref(r), t, *[_ptr(x) for x in args], epoch_end, _ptr(dn[0]), _ptr(dn[1]),
                      _ptr(dfv[0]), _ptr(dfv[1]), _stream())
                want["reward"][:, t], want["cost"][:, t] = rew, cost
                for n in range(N):
                    end, (br, bc) = _segment_rule(bool(term[n]), bool(trunc[n]), bool(epoch_end), (nv[0][n], nv[1][n]),
                                                  (fv[0][n], fv[1][n]) if fv_given else None)
                    want["seg_end"][n, t], want["boot_r"][n, t], want["boot_c"][n, t] = end, br, bc
                    seen.add((bool(term[n]), bool(trunc[n]), epoch_end, fv_given))
                torch.cuda.synchronize()
                for k in bufs:                                          # slot t as the rule says, every other slot as it was
                    assert torch.equal(dbuf[k].cpu(), want[k]), (k, t, epoch_end, nv_given, fv_given, shift)
    assert len(seen) == 16                                              # every term / trunc / epoch_end / final_v combination


# ---- spo_gae_dual ----
@pytest.mark.gpu
@pytest.mark.parametrize("T", [1, 4, 5, 127, 128, 129, 511, 512, 513, 1025, 5000])
def test_gae_scan_and_exact_at_tile_warp_thread_edges(T):
    """Both modes at N = 1, 3, 300 for every regime and discount pair.  Exact mode equals gae_dual_np bit for bit; the
    scan is within ulp32(ref) + c * L * 2^-53 * sum|terms| of the float64 recurrence, per element."""
    dev = _cuda()
    rng = np.random.default_rng(T)
    blocks = []
    for N in (1, 3, 300):
        seg = _gae_layout(rng, N, T)
        for regime in REGIMES:
            blocks.append((N, regime, _gae_inputs(rng, seg, regime)))
    cat = {k: np.concatenate([b[2][k] for b in blocks]) for k in blocks[0][2]}
    dcat = {k: torch.from_numpy(v).to(dev) for k, v in cat.items()}
    R = cat["rew"].shape[0]
    keys = ("rew", "cost", "v_r", "v_c", "seg_end", "boot_r", "boot_c")
    for gamma, lam, lam_c in DISCOUNTS:
        want = [w.numpy() for w in O.gae_dual_np(*[cat[k] for k in keys], gamma, lam, lam_c)]
        ref = _gae_f64(*[cat[k] for k in keys], gamma, lam, lam_c)
        outs = {mode: [torch.full((R, T), float("nan"), device=dev) for _ in range(4)] for mode in (0, 1)}
        row = 0
        for N, regime, _ in blocks:
            for mode in (0, 1):
                _call("spo_gae_dual", *[_ptr(dcat[k][row:row + N]) for k in keys], gamma, gamma * lam, gamma * lam_c,
                      *[_ptr(o[row:row + N]) for o in outs[mode]], N, T, mode, _stream())
            row += N
        torch.cuda.synchronize()
        exact = [o.cpu().numpy() for o in outs[1]]
        scan = [o.cpu().numpy().astype(np.float64) for o in outs[0]]
        for name, e, w in zip(("adv_r", "adv_c", "tgt_r", "tgt_c"), exact, want):
            assert np.array_equal(e, w), (name, T, gamma, lam, lam_c, np.argwhere(e != w)[:4])
        row = 0
        for N, regime, _ in blocks:
            sl = slice(row, row + N)
            for s, (acc, tgt, mag, ln), disc in ((0, ref[0], gamma * lam), (1, ref[1], gamma * lam_c)):
                for got, r64 in ((scan[s][sl], acc[sl]), (scan[s + 2][sl], tgt[sl])):
                    err = np.abs(got - r64)
                    slack = np.maximum(err - _ulp32(r64), 0.0)
                    room = ln[sl] * U64 * mag[sl]
                    assert bool((slack[room == 0] == 0).all()), (T, N, regime, disc)
                    c = float((slack[room > 0] / room[room > 0]).max(initial=0.0))
                    for tag in (regime, f"disc={disc:.2f}"):
                        _note(f"c[{tag}]", c)
                        _note(f"ulps[{tag}]", float((err / _ulp32(r64)).max()))
                    _record("gae_scan_c", c)
            row += N


# ---- spo_adv_stats / spo_adv_apply ----
def _adv_apply_host(a, c, stats, std_r, std_c, lam, lam_p1):
    """spo_adv_apply in numpy: the float64 mean / unbiased variance of the statistics, then correctly rounded fp32
    operations in the kernel's order (numpy never fuses)."""
    s0, s1, s2, n = (np.float64(x) for x in stats)
    with np.errstate(all="ignore"):
        mean_d = s0 / n
        var_d = (s1 - s0 * s0 / n) / (n - np.float64(1.0))
        var_d = np.float64(0.0) if var_d < 0.0 else var_d
        mean = np.float32(mean_d)
        denom = np.float32(np.float32(np.sqrt(var_d)) + np.float32(1e-8))
        cmean = np.float32(s2 / n)
        a = (a - mean) / denom if std_r else a.copy()
        c = c - cmean if std_c else c.copy()
        mixed = (a - np.float32(lam) * c) / np.float32(lam_p1)
    return a, c, mixed


@pytest.mark.gpu
@pytest.mark.parametrize("count", [1, 2, 2047, 2048, 2049, "grid+37", (1 << 22) + 5])
def test_adv_stats_and_apply(count):
    """Advantages 1e3 + N(0, 1) and a constant cost advantage.  The four statistics against float64 sums (above
    8 * SMs * 2048 samples the grid-stride loop takes a second lap); then spo_adv_apply on the device's statistics bit for
    bit against the host restatement for every standardise-flag pair, lambda in {0, 0.37, 1.9} and ``mixed`` NULL.
    One sample gives NaN advantages, as torch's std() of one element does."""
    dev = _cuda()
    if count == "grid+37":
        count = 8 * torch.cuda.get_device_properties(dev).multi_processor_count * 2048 + 37
    rng = np.random.default_rng(count)
    a = (1e3 + rng.standard_normal(count)).astype(np.float32)
    c = np.full(count, 0.37, dtype=np.float32)
    da, dc = torch.from_numpy(a).to(dev), torch.from_numpy(c).to(dev)
    stats = torch.full((4,), float("nan"), dtype=torch.float64, device=dev)
    _call("spo_adv_stats", _ptr(da), _ptr(dc), count, _ptr(stats), _stream())
    st = stats.cpu().numpy()
    a64, c64 = a.astype(np.float64), c.astype(np.float64)
    for i, (got, terms) in enumerate(((st[0], a64), (st[1], a64 * a64), (st[2], c64))):
        _record("adv_stats", abs(got - terms.sum()) / np.abs(terms).sum())
    assert st[3] == count
    assert st[2] == np.float64(np.float32(0.37)) * count                  # multiples of one fp32 value: exact in float64
    wr, wc, wm = torch.empty_like(da), torch.empty_like(dc), torch.empty_like(da)
    for std_r in (0, 1):
        for std_c in (0, 1):
            for lam, mixed in ((0.0, None), (0.0, wm), (0.37, wm), (1.9, wm)):
                wr.copy_(da); wc.copy_(dc); wm.fill_(float("nan"))
                _call("spo_adv_apply", _ptr(wr), _ptr(wc), count, _ptr(stats), std_r, std_c, lam, lam + 1, _ptr(mixed), _stream())
                hr, hc, hm = _adv_apply_host(a, c, st, std_r, std_c, lam, lam + 1)
                got = [t.cpu().numpy() for t in (wr, wc, wm)]
                what = (count, std_r, std_c, lam, mixed is None)
                assert np.array_equal(got[0], hr, equal_nan=True), what
                assert np.array_equal(got[1], hc, equal_nan=True), what
                if mixed is None:
                    assert np.isnan(got[2]).all(), what                              # NULL: nothing written
                else:
                    assert np.array_equal(got[2], hm, equal_nan=True), what
                if std_c:
                    assert not got[1].any(), what                                     # a constant cost advantage centres to 0
                if std_r:
                    assert np.isnan(got[0]).all() if count == 1 else np.isfinite(got[0]).all(), what
    if count == 1:
        assert torch.tensor(a).std().isnan()


# ---- spo_obs_normalize / spo_action_rescale ----
@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 8, 9, 1024])
@pytest.mark.parametrize("D", [1, 31, 32, 33, 64, 128])
def test_obs_normalize_against_running_mean_std(D, n):
    """24 calls of which 21 update: columns drifting around 2 with spread 3, columns at 1e4 with spread 1e-2 (a one-pass
    variance cancels there), and a column constant across envs and steps; in-place calls, count_out NULL, out NULL.
    Statistics against oracle/envio.py, outputs within one fp32 ulp of the float64 result."""
    dev = _cuda()
    L = _lib()
    rng = np.random.default_rng(D * 1000 + n)
    kind = (np.arange(D) + D) % 3                                   # 0 drifting, 1 large offset, 2 constant
    ref = envio.NormalizeObservation(D)
    mean = torch.zeros(D, dtype=torch.float64, device=dev)
    var = torch.ones(D, dtype=torch.float64, device=dev)
    count = ref.obs_rms.count
    cnt = torch.zeros(1, dtype=torch.float64, device=dev)
    for k in range(24):
        update = k not in (6, 13, 20)
        obs = np.where(kind == 0, 2.0 + 0.1 * k + 3.0 * rng.standard_normal((n, D)),
                       np.where(kind == 1, 1e4 + 1e-2 * rng.standard_normal((n, D)), 3.25)).astype(np.float32)
        dobs = torch.from_numpy(obs).to(dev)
        inplace, no_out, no_count = k % 2 == 1, k == 4, k % 3 == 2
        out = dobs if inplace else (None if no_out else torch.empty_like(dobs))
        cnt.fill_(-1.0)
        _call("spo_obs_normalize", _ptr(dobs), n, D, _ptr(mean), _ptr(var), count, None if no_count else _ptr(cnt), int(update),
              1e-8, _ptr(out), _stream())
        want = ref.normalize(obs.astype(np.float64), update=update)
        if update:
            count = count + n
        torch.cuda.synchronize()
        assert ref.obs_rms.count == count
        assert float(cnt) == (-1.0 if (no_count or not update) else count), (k, float(cnt))
        for got, w in ((mean, ref.obs_rms.mean), (var, ref.obs_rms.var)):
            _record("obs_stats", float((np.abs(got.cpu().numpy() - w) / np.abs(w)).max()))
        if out is None:
            assert torch.equal(dobs.cpu(), torch.from_numpy(obs))
            continue
        got = out.cpu().numpy().astype(np.float64)
        _record("obs_out_ulp", float((np.abs(got - want) / _ulp32(want)).max()))


@pytest.mark.gpu
@pytest.mark.parametrize("A", list(range(1, 17)))
def test_action_rescale_against_float64(A):
    """Inputs exactly at, inside and beyond [min, max], the default and a non-default range, n * A not a multiple of the
    256-thread block, one dimension with low == high.  Against oracle/envio.py in float64; results inside [low, high]."""
    dev = _cuda()
    rng = np.random.default_rng(A)
    low = (rng.standard_normal(A) * 2 - 1).astype(np.float32)
    high = (low + rng.random(A) * 3 + 0.1).astype(np.float32)
    high[A // 2] = low[A // 2]
    dlow, dhigh = torch.from_numpy(low).to(dev), torch.from_numpy(high).to(dev)
    scale = np.maximum(np.abs(low), np.abs(high)).astype(np.float64)
    for n in (1, 37, 1000):
        assert (n * A) % 256 != 0
        for lo_a, hi_a in ((-1.0, 1.0), (-2.0, 0.5)):
            pick = rng.integers(0, 5, (n, A))
            inside = lo_a + (hi_a - lo_a) * rng.random((n, A))
            act = np.choose(pick, [np.full((n, A), lo_a), np.full((n, A), hi_a), inside, lo_a - 1 - 5 * rng.random((n, A)),
                                   hi_a + 1 + 5 * rng.random((n, A))]).astype(np.float32)
            dact = torch.from_numpy(act).to(dev)
            out = torch.empty_like(dact)
            _call("spo_action_rescale", _ptr(dact), n, A, _ptr(dlow), _ptr(dhigh), lo_a, hi_a, _ptr(out), _stream())
            got = out.cpu().numpy()
            want = envio.rescale_action(act.astype(np.float64), low.astype(np.float64), high.astype(np.float64), lo_a, hi_a)
            assert ((got >= low) & (got <= high)).all(), (A, n, lo_a)
            assert (got[:, A // 2] == low[A // 2]).all()
            assert (got[pick == 0] == np.broadcast_to(low, (n, A))[pick == 0]).all()       # exactly at min -> low
            _record("rescale", float((np.abs(got - want) / scale).max()))


# ---- spo_cg_begin / spo_cg_update ----
class _SPD:
    """M = Q diag(lam) Q^T, Q a product of two Householder reflections, eigenvalues geometric in [1, cond]: a float64
    symmetric positive-definite operator applied in O(P)."""

    def __init__(self, rng, P, cond):
        self.lam = np.geomspace(1.0, cond, P)[rng.permutation(P)]
        self.u = [v / np.linalg.norm(v) for v in rng.standard_normal((2, P))]

    def _h(self, u, v):
        return v - 2.0 * u * (u @ v)

    def __call__(self, v):
        y = self._h(self.u[0], self._h(self.u[1], v))
        return self._h(self.u[1], self._h(self.u[0], self.lam * y))


def _cg_step64(x, r, p, z, rdotr, eps):
    """cpo.py:92-105, one iteration in float64 from the given vectors: (alpha, x, r, new rdotr, p, mu)."""
    alpha = rdotr / (p @ z + eps)
    x1, r1 = x + alpha * p, r - alpha * z
    nrr = r1 @ r1
    mu = nrr / (rdotr + eps)
    return alpha, x1, r1, nrr, r1 + mu * p, mu


class _CG:
    """The device solver's state: x and work = r | p | z | - | rdotr, done."""

    def __init__(self, dev, d, P, b):
        self.d, self.P = d, P
        self.x = torch.full((P,), float("nan"), device=dev)
        self.work = torch.full((4 * P + 4,), 3.0, device=dev)
        _call("spo_cg_begin", C.byref(d), _ptr(b), _ptr(self.x), _ptr(self.work), _stream())

    def read(self):
        w = self.work.cpu().numpy().astype(np.float64)
        P = self.P
        return self.x.cpu().numpy().astype(np.float64), w[:P], w[P:2 * P], w[2 * P:3 * P], w[4 * P], w[4 * P + 1]

    def set_z(self, z):
        self.work[2 * self.P:3 * self.P].copy_(torch.from_numpy(np.asarray(z, dtype=np.float32)))

    def step(self, tol, eps):
        _call("spo_cg_update", C.byref(self.d), _ptr(self.x), _ptr(self.work), tol, eps, _stream())
        torch.cuda.synchronize()


def _check_step(state_in, state_out, eps, stopped=False):
    x, r, p, z, rdotr, _ = state_in
    x1, r1, p1, _, rdotr1, done = state_out
    alpha, wx, wr, nrr, wp, mu = _cg_step64(x, r, p, z, rdotr, eps)
    _check("cg_step", x1, wx, float(np.abs(x).max() + np.abs(alpha * p).max()))
    _check("cg_step", r1, wr, float(np.abs(r).max() + np.abs(alpha * z).max()))
    if stopped:
        assert done == 1.0
        assert np.array_equal(p1, p) and rdotr1 == rdotr                    # cpo.py:101: break before p and rdotr move
    else:
        assert done == 0.0
        _check("cg_step", [rdotr1], [nrr], float(((np.abs(r) + np.abs(alpha * z)) ** 2).sum()))
        _check("cg_step", p1, wp, float(np.abs(wr).max() + np.abs(mu * p).max()))
    return alpha


@pytest.mark.gpu
@pytest.mark.parametrize("dims", [(1, 1), (60, 2), (128, 16)])
def test_cg_vector_kernels_against_float64(dims):
    """spo_cg_begin / spo_cg_update with z = fp32(M p) written by the test: every step against the float64 step from the
    same fp32 state, ten steps against conjugate_gradients in float64; a residual tolerance equal to the fp32 residual
    norm does not stop; a tolerance between the float64 norms of steps k - 1 and k stops at step k with x and r moved and
    p not, and later calls leave x and the work vector bit-identical; z = 0 (alpha = rdotr / eps) against float64."""
    dev = _cuda()
    L = _lib()
    d = L.dims(*dims)
    P = L.param_count(d)[0]
    rng = np.random.default_rng(P)
    M = _SPD(rng, P, 100.0)
    eps = 1e-6
    b32 = rng.standard_normal(P).astype(np.float32)
    b64 = b32.astype(np.float64)
    db = torch.from_numpy(b32).to(dev)

    def fp32_z(cg):
        z = M(cg.read()[2]).astype(np.float32)
        cg.set_z(z)
        return cg.read()

    # ---- ten steps, each against float64 from its own inputs; step 3 replayed with tol = its fp32 residual norm ----
    cg = _CG(dev, d, P, db)
    x, r, p, _, rdotr, done = cg.read()
    assert (x == 0).all() and np.array_equal(r, b64) and np.array_equal(p, b64) and done == 0.0
    _check("cg_step", [rdotr], [b64 @ b64], float(b64 @ b64))
    for it in range(10):
        s_in = fp32_z(cg)
        if it == 3:
            snap = (cg.x.clone(), cg.work.clone())
            cg.step(1e-30, eps)
            after = (cg.x.clone(), cg.work.clone())
            tol = float(np.sqrt(np.float32(cg.read()[4])))                   # sqrtf(nrr) exactly: '<' does not stop
            cg.x.copy_(snap[0]); cg.work.copy_(snap[1])
            cg.step(tol, eps)
            assert torch.equal(cg.x, after[0]) and torch.equal(cg.work, after[1])
        else:
            cg.step(1e-30, eps)
        alpha = _check_step(s_in, cg.read(), eps)
        if it == 0:
            _check("cg_step", [alpha], [s_in[4] / (s_in[2] @ s_in[3] + eps)], abs(alpha))
    x64 = O.conjugate_gradients(lambda v: torch.from_numpy(M(v.numpy())), torch.from_numpy(b64), num_steps=10,
                                residual_tol=1e-10, eps=eps).numpy()
    _check("cg_solve", cg.read()[0], x64, float(np.abs(x64).max()))

    # ---- the residual stop at step k ----
    k = 4
    rho = [np.linalg.norm(b64 - M(O.conjugate_gradients(lambda v: torch.from_numpy(M(v.numpy())), torch.from_numpy(b64), num_steps=j,
                                                        residual_tol=1e-10, eps=eps).numpy())) for j in range(1, k + 1)]
    above = min(rho[:-1])                                                    # residual norms need not decrease monotonically
    assert above > 1.1 * rho[-1], rho
    tol = float(np.sqrt(above * rho[-1]))
    cg = _CG(dev, d, P, db)
    for it in range(1, k + 1):
        s_in = fp32_z(cg)
        cg.step(tol, eps)
        _check_step(s_in, cg.read(), eps, stopped=it == k)
    for _ in range(3):
        cg.set_z(7.0 * rng.standard_normal(P))
        snap = (cg.x.clone(), cg.work.clone())
        cg.step(tol, eps)
        assert torch.equal(cg.x, snap[0]) and torch.equal(cg.work, snap[1])

    # ---- z = 0: p.z + eps = eps, rdotr comparable to eps ----
    small = (b64 * np.sqrt(1e-6 / (b64 @ b64))).astype(np.float32)
    cg = _CG(dev, d, P, torch.from_numpy(small).to(dev))
    cg.set_z(np.zeros(P))
    s_in = cg.read()
    cg.step(1e-30, eps)
    s_out = cg.read()
    assert all(np.isfinite(v).all() for v in s_out[:3])
    x, r, p, z, rdotr, _ = s_in
    alpha, wx, wr, nrr, wp, mu = _cg_step64(x, r, p, z, rdotr, eps)
    assert 0.3 < alpha < 3.0 and 0.3 < mu < 0.7, (alpha, mu)                 # both + eps terms change the result by O(1)
    _check("cg_eps", s_out[0], wx, float(np.abs(wx).max()))
    _check("cg_eps", s_out[2], wp, float(np.abs(wp).max()))
    _check("cg_eps", [s_out[4]], [nrr], nrr)


@pytest.mark.gpu
def test_conjugate_gradient_zero_iterations():
    """spo_conjugate_gradient with iters = 0: x = 0, r = p = b, rdotr = b.b (no Fisher-vector product is run)."""
    dev = _cuda()
    L = _lib()
    d = L.dims(60, 2)
    P, _, total = L.param_count(d)
    b = torch.randn(P, generator=torch.Generator().manual_seed(3)).to(dev)
    params, obs = torch.zeros(total, device=dev), torch.zeros(16, 60, device=dev)
    x = torch.full((P,), float("nan"), device=dev)
    work = torch.full((4 * P + 4,), 3.0, device=dev)
    _call("spo_conjugate_gradient", C.byref(d), _ptr(params), _ptr(obs), 16, _ptr(b), 0, 0.1, 1e-10, 1e-6, _ptr(x), _ptr(work), _stream())
    torch.cuda.synchronize()
    assert bool((x == 0).all())
    assert torch.equal(work[:P], b) and torch.equal(work[P:2 * P], b)
    b64 = b.cpu().double()
    _check("cg_step", work[4 * P:4 * P + 1], (b64 @ b64).reshape(1), float(b64 @ b64))
    assert float(work[4 * P + 1]) == 0.0
