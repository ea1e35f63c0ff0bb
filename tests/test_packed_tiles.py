"""The packed minibatch tiles of the update pass.

spo_pg_update first writes the pass's rows out in step order (spo_pack_tiles): one record per 64-row tile, laid out like a
tile slot of the update kernel, [64][ldx] observations then [64][3 AC + 4] side data.  The update kernel copies each record
into shared memory with one bulk copy, through a ring of two slots, or of one at obs > 64 with act > 8 (where two do not fit).
These tests pin the records bit for bit against a torch gather, both slot counts against the oracle, and that a pass after
a KL early stop changes nothing."""
import ctypes as C

import pytest
import torch

import test_update_schedule as US

pytestmark = pytest.mark.gpu


def _cuda():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    return torch.device("cuda:0")


def _want_tiles(D, A, batch, perm, perm_len, kind, src):
    """The records spo_pack_tiles must write, from a torch gather of the same rows."""
    from safepo import _lib as L
    nt1, ac = (1 if D <= 64 else 2), (8 if A <= 8 else 16)
    ldx, auxw = 64 * nt1 + 8, 3 * ac + 4
    logp, adv, tgt, omean, ostd = ac, ac + 1, ac + 2, ac + 4, 2 * ac + 4
    tps, n_steps = -(-batch // 64), -(-perm_len // batch)
    x = torch.zeros(n_steps, tps * 64, ldx)
    aux = torch.zeros(n_steps, tps * 64, auxw)
    for s in range(n_steps):
        idx = perm[s * batch:min((s + 1) * batch, perm_len)].cpu()
        n = idx.numel()
        x[s, :n, :D] = src["obs"][idx]
        aux[s, :n, tgt] = src["target_r"][idx]
        aux[s, :n, tgt + 1] = src["target_c"][idx]
        if kind != L.LOSS_CRITIC_ONLY:
            aux[s, :n, :A] = src["act"][idx]
            aux[s, :n, logp] = src["logp"][idx]
            aux[s, :n, adv] = src["adv"][idx]
        if kind == L.LOSS_FOCOPS:
            aux[s, :n, omean:omean + A] = src["old_mean"][idx]
            aux[s, :n, ostd:ostd + A] = src["old_std"][idx]
    x = x.reshape(n_steps * tps, 64 * ldx)
    aux = aux.reshape(n_steps * tps, 64 * auxw)
    return torch.cat([x, aux], dim=1).reshape(-1)


@pytest.mark.parametrize("D,A", [(27, 2), (60, 8), (88, 12), (104, 16), (128, 2), (60, 12)])
@pytest.mark.parametrize("batch", [64, 128])
@pytest.mark.parametrize("kind", ["ppo", "focops", "critic"])
def test_pack_matches_gather(D, A, batch, kind):
    from safepo import _lib as L
    from safepo.single_agent._engine import make_ctrl
    if kind == "focops" and batch > 64:
        pytest.skip("FOCOPS runs batch <= 64")
    dev = _cuda()
    k = {"ppo": L.LOSS_PPO_CLIP, "focops": L.LOSS_FOCOPS, "critic": L.LOSS_CRITIC_ONLY}[kind]
    g = torch.Generator().manual_seed(D * 1000 + A * 10 + batch)
    S = 1000
    perm_len = 3 * batch + 37          # below S, not a multiple of batch: the last step is partial
    src = {"obs": torch.randn(S, D, generator=g), "act": torch.randn(S, A, generator=g), "logp": torch.randn(S, generator=g),
           "target_r": torch.randn(S, generator=g), "target_c": torch.randn(S, generator=g), "adv": torch.randn(S, generator=g),
           "old_mean": torch.randn(S, A, generator=g), "old_std": torch.rand(S, A, generator=g) + 0.5}
    # ppo: old_mean / old_std are passed but have no column for the clipped surrogate, so they must come out as zeros
    if kind == "critic":                # the actor's sources are absent (NULL) for the critic regression
        for n in ("act", "logp", "adv", "old_mean", "old_std"):
            src[n] = None
    d ={n: (None if v is None else v.to(dev).contiguous()) for n, v in src.items()}
    perm = torch.randperm(S, generator=g)[:perm_len + 5].to(dev)
    batch_s = L.Batch(*(L.ptr(d[n]) for n in ("obs", "act", "logp", "target_r", "target_c", "adv", "old_mean", "old_std")), S)
    want = _want_tiles(D, A, batch, perm, perm_len, k, src)
    out = torch.full((want.numel(),), float("nan"), device=dev)
    dims = L.Dims(D, A, 64)
    ctrl = make_ctrl(dev)
    lib = L.lib()
    fn = lib.spo_debug_pack_tiles
    fn.argtypes = [C.POINTER(L.Dims), C.POINTER(L.Batch), C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    L.check(fn(C.byref(dims), C.byref(batch_s), L.ptr(perm), perm_len, batch, k, L.ptr(ctrl), L.ptr(out), L.stream()),
            "spo_debug_pack_tiles")
    got = out.cpu()
    assert torch.equal(got.view(torch.int32), want.view(torch.int32)), int((got.view(torch.int32) != want.view(torch.int32)).sum())


@pytest.mark.parametrize("D,A,batch,n_steps,last_rows,seed", [
    (104, 12, 128, 6, 100, 21),    # one slot, two tiles per step, a partial last step
    (128, 16, 128, 5, 40, 22),     # one slot, the last step's second tile all padding
])
def test_one_slot(D, A, batch, n_steps, last_rows, seed):
    US._check(D=D, A=A, batch=batch, n_steps=n_steps, last_rows=last_rows, max_norm=20.0, hot={1, 2}, seed=seed)


@pytest.mark.parametrize("D,A,batch,n_steps,last_rows,seed", [
    (60, 12, 128, 5, 70, 23),      # two slots at AC = 16, two tiles per step
    (88, 8, 64, 9, 17, 24),        # two slots at NT1 = 2
])
def test_two_slots(D, A, batch, n_steps, last_rows, seed):
    US._check(D=D, A=A, batch=batch, n_steps=n_steps, last_rows=last_rows, max_norm=20.0, hot={0, 3}, seed=seed)


def test_pass_after_stop_changes_nothing():
    from safepo import _lib as L
    from safepo.common.model import ActorVCritic
    from safepo.single_agent._engine import PolicyGradientUpdate
    dev = _cuda()
    torch.manual_seed(5)
    D, A, S = 60, 2, 640
    pol = ActorVCritic(D, A).to(dev)
    cfg = dict(hidden_sizes=[64, 64], gamma=0.99, target_kl=1e9, batch_size=64, learning_iters=1, max_grad_norm=40.0)
    upd = PolicyGradientUpdate(pol, cfg, L.LOSS_PPO_CLIP, epochs=10, host_rng=False, device=dev)
    data = {"obs": torch.randn(S, D, device=dev), "act": torch.randn(S, A, device=dev), "log_prob": torch.full((S,), -2.5, device=dev),
            "target_value_r": torch.randn(S, device=dev), "target_value_c": torch.randn(S, device=dev), "adv": torch.randn(S, device=dev)}
    batch = L.Batch(L.ptr(data["obs"]), L.ptr(data["act"]), L.ptr(data["log_prob"]), L.ptr(data["target_value_r"]),
                    L.ptr(data["target_value_c"]), L.ptr(data["adv"]), None, None, S)
    upd.ctrl.zero_()
    upd.ctrl.view(torch.int32)[10] = 1          # spo_update_ctrl.stop (byte offset 40)
    before = [t.clone() for t in (pol.flat, upd.adam.m, upd.adam.v, upd.adam.t, upd.ctrl)]
    perm = torch.randperm(S, device=dev)
    L.check(L.lib().spo_pg_update(C.byref(pol.dims), L.ptr(pol.flat), L.ptr(upd.adam.m), L.ptr(upd.adam.v), L.ptr(upd.adam.t),
                                  C.byref(batch), L.ptr(perm), S, 64, L.LOSS_PPO_CLIP, C.byref(upd.hp), L.ptr(upd.ctrl), L.stream()),
            "spo_pg_update")
    torch.cuda.synchronize()
    after = (pol.flat, upd.adam.m, upd.adam.v, upd.adam.t, upd.ctrl)
    for b, a in zip(before, after):
        assert torch.equal(b, a)
