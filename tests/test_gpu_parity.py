"""GPU parity tests: every libspo kernel (called through the C-ABI via the python host
classes) against the oracle and the golden fixtures generated from the reference.

Tolerances: bit-exact for buffer indexing / segment logic and for the sequential GAE
variant; 1e-5 relative (BASELINE.json north_star) for floating-point advantages, values
and losses -- with the absolute floor stated at each assert."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import spo_oracle as O
from oracle import trainers as TR

pytestmark = pytest.mark.gpu

RTOL = 1e-5


def _cuda():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    return torch.device("cuda:0")


class Sp:
    def __init__(self, d):
        self.shape = (d,)


def make_policy(state, D, A):
    from safepo.common.model import ActorVCritic
    pol = ActorVCritic(D, A, [64, 64]).to(_cuda())
    pol.actor.load_state_dict(state["actor"])
    pol.reward_critic.load_state_dict(state["reward_critic"])
    pol.cost_critic.load_state_dict(state["cost_critic"])
    return pol


def policy_state(pol):
    return {n: {k: v.detach().cpu().clone() for k, v in getattr(pol, n).state_dict().items()}
            for n in ("actor", "reward_critic", "cost_critic")}


def oracle_policy(state, D, A):
    p = O.OraclePolicy(D, A, [64, 64])
    p.load(state)
    return p


def close(got, want, rtol=RTOL, atol=1e-6):
    got, want = torch.as_tensor(got).double().cpu(), torch.as_tensor(want).double().cpu()
    err = (got - want).abs()
    ok = bool((err <= atol + rtol * want.abs()).all())
    return ok, float(err.max()), float((err / (want.abs() + 1e-12)).max())


# ---------------------------------------------------------------------------------------
# F1 / F2
# ---------------------------------------------------------------------------------------

def test_packed_layout_is_reference_flat_order(golden):
    c = golden("trust")["trust"]
    pol = make_policy(c["state"], c["D"], c["A"])
    assert [n for n, _ in pol.actor.named_parameters()] == c["names"]
    assert torch.equal(pol.actor_flat().cpu(), c["theta"])           # get_flat_params_from(policy.actor)
    assert set(pol.actor.state_dict().keys()) == set(c["state"]["actor"].keys())


def test_policy_step_vs_reference(golden):
    dev = _cuda()
    for c in golden("forward")["forward"]:
        pol = make_policy(c["state"], c["D"], c["A"])
        act, logp, vr, vc = pol.step(c["obs"].to(dev), eps=c["eps"].to(dev))
        for name, got, want in (("act", act, c["act"]), ("logp", logp, c["logp"]), ("v_r", vr, c["v_r"]), ("v_c", vc, c["v_c"])):
            ok, ea, er = close(got, want)
            assert ok, (name, c["D"], ea, er)
        dact, dlogp, _, _ = pol.step(c["obs"].to(dev), deterministic=True)
        assert close(dact, c["det_act"])[0] and close(dlogp, c["det_logp"])[0]
        a1, l1, r1, c1 = pol.step(c["obs"][0].to(dev), eps=c["eps"][0].to(dev))     # single-row form
        assert [tuple(a1.shape), tuple(l1.shape), tuple(r1.shape)] == [tuple(s) for s in c["row_shapes"]]
        assert close(a1, c["act"][0])[0]
        vr2, vc2 = pol.values(c["obs"].to(dev))
        assert close(vr2, c["v_r"])[0] and close(vc2, c["v_c"])[0]
        mean = pol.actor(c["obs"].to(dev)).mean
        assert close(mean, c["det_act"])[0]


def test_policy_step_large_batch_and_philox():
    dev = _cuda()
    from safepo.common.model import ActorVCritic
    torch.manual_seed(0)
    pol = ActorVCritic(60, 2).to(dev)
    opol = oracle_policy(policy_state(pol), 60, 2)
    obs = torch.randn(1024 + 37, 60)
    eps = torch.randn(1024 + 37, 2)
    act, logp, vr, vc = pol.step(obs.to(dev), eps=eps.to(dev))
    with torch.no_grad():
        oa, ol, orr, oc = O.policy_step(opol, obs, eps=eps)
    for name, got, want in (("act", act, oa), ("logp", logp, ol), ("v_r", vr, orr), ("v_c", vc, oc)):
        ok, ea, er = close(got, want, atol=2e-6)      # 1061 rows, obs 60: the TMA + wgmma step kernel (3xTF32, SFU tanh)
        assert ok, (name, ea, er)
    # in-kernel Philox: standard normal draws, deterministic in (seed, offset), fresh each call
    a1, _, _, _ = pol.step(obs.to(dev))
    a2, _, _, _ = pol.step(obs.to(dev))
    mean = pol.actor(obs.to(dev)).mean
    z1 = ((a1 - mean) / torch.exp(pol.actor.log_std.detach())).cpu()
    z2 = ((a2 - mean) / torch.exp(pol.actor.log_std.detach())).cpu()
    assert not torch.equal(z1, z2)
    assert abs(float(z1.mean())) < 0.1 and abs(float(z1.std()) - 1.0) < 0.1
    assert abs(float(torch.cat([z1, z2]).pow(4).mean()) - 3.0) < 0.5           # kurtosis of N(0,1)


def test_fused_store_and_segment_rule_bit_exact():
    """policy.step(store=...) + store_transition == the reference's buffer.store /
    finish_path bookkeeping (ppo_lag.py:187-234), element for element."""
    dev = _cuda()
    from safepo.common.buffer import VectorizedOnPolicyBuffer
    from safepo.common.model import ActorVCritic
    torch.manual_seed(1)
    N, T, D, A = 70, 9, 27, 8
    pol = ActorVCritic(D, A).to(dev)
    buf = VectorizedOnPolicyBuffer(Sp(D), Sp(A), size=T, device=dev, num_envs=N)
    g = torch.Generator().manual_seed(5)
    want = {k: torch.zeros(N, T) for k in ("reward", "cost", "boot_r", "boot_c")}
    want_seg = torch.zeros(N, T, dtype=torch.uint8)
    obs_log, act_log, lp_log, vr_log = [], [], [], []
    for t in range(T):
        obs = torch.randn(N, D, generator=g)
        eps = torch.randn(N, A, generator=g)
        act, logp, vr, vc = pol.step(obs.to(dev), eps=eps.to(dev), store=(buf.struct, t))
        obs_log.append(obs); act_log.append(act.cpu()); lp_log.append(logp.cpu()); vr_log.append(vr.cpu())
        rew, cost = torch.randn(N, generator=g), torch.rand(N, generator=g)
        term = torch.rand(N, generator=g) < 0.2
        trunc = (torch.rand(N, generator=g) < 0.2) & ~term
        nv = (torch.randn(N, generator=g), torch.randn(N, generator=g))
        fv = (torch.randn(N, generator=g), torch.randn(N, generator=g))
        epoch_end = t == T - 1
        buf.store_transition(t, rew.to(dev), cost.to(dev), term.to(torch.uint8).to(dev), trunc.to(torch.uint8).to(dev),
                             epoch_end, tuple(x.to(dev) for x in nv) if epoch_end else None,
                             tuple(x.to(dev) for x in fv) if trunc.any() else None)
        want["reward"][:, t], want["cost"][:, t] = rew, cost
        for n in range(N):
            end = epoch_end or bool(term[n]) or bool(trunc[n])
            br = bc = 0.0
            if end and not term[n]:
                if epoch_end:
                    br, bc = nv[0][n], nv[1][n]
                if trunc[n]:
                    br, bc = fv[0][n], fv[1][n]
            want_seg[n, t] = int(end)
            want["boot_r"][n, t], want["boot_c"][n, t] = br, bc
    torch.cuda.synchronize()
    assert torch.equal(buf.data["obs"].cpu(), torch.stack(obs_log, 1))          # env-major [N,T,D]
    assert torch.equal(buf.data["act"].cpu(), torch.stack(act_log, 1))
    assert torch.equal(buf.data["log_prob"].cpu(), torch.stack(lp_log, 1))
    assert torch.equal(buf.data["value_r"].cpu(), torch.stack(vr_log, 1))
    assert torch.equal(buf.data["reward"].cpu(), want["reward"]) and torch.equal(buf.data["cost"].cpu(), want["cost"])
    assert torch.equal(buf.seg_end.cpu(), want_seg)
    assert torch.equal(buf.boot_r.cpu(), want["boot_r"]) and torch.equal(buf.boot_c.cpu(), want["boot_c"])
    from safepo import _lib as L
    with pytest.raises(L.SpoError):                                               # "Buffer overflow" (buffer.py:92)
        pol.step(torch.zeros(N, D, device=dev), store=(buf.struct, T))


@pytest.mark.parametrize("N,D,A", [(1024, 60, 2), (300, 60, 2), (128, 28, 8), (129, 64, 1)])
def test_tensor_core_rollout_step_and_store(N, D, A):
    """The rollout step of batches >= 128 rows with obs_dim % 4 == 0 runs on the TMA + wgmma kernel (csrc/spo_tc_forward.cu,
    step mode: grid (row tiles, nets), sample / log-prob / slot write in the epilogue): outputs against the oracle at 1e-5,
    the slot written by the kernel bit-identical to what it returned, observation rows copied bit-exactly,
    bootstrap values (critics only) equal to the step's values."""
    dev = _cuda()
    from safepo.common.buffer import VectorizedOnPolicyBuffer
    from safepo.common.model import ActorVCritic
    torch.manual_seed(N + D)
    T = 3
    pol = ActorVCritic(D, A).to(dev)
    with torch.no_grad():
        pol.actor.log_std.copy_(torch.linspace(-0.5, 0.3, A))
    opol = oracle_policy(policy_state(pol), D, A)
    buf = VectorizedOnPolicyBuffer(Sp(D), Sp(A), size=T, device=dev, num_envs=N)
    g = torch.Generator().manual_seed(9)
    for t in range(T):
        obs, eps = torch.randn(N, D, generator=g), torch.randn(N, A, generator=g)
        act, logp, vr, vc = pol.step(obs.to(dev), eps=eps.to(dev), store=(buf.struct, t))
        with torch.no_grad():
            oa, ol, orr, oc = O.policy_step(opol, obs, eps=eps)
        for name, got, want in (("act", act, oa), ("logp", logp, ol), ("v_r", vr, orr), ("v_c", vc, oc)):
            ok, ea, er = close(got, want, atol=2e-6)
            assert ok, (name, N, D, A, t, ea, er)
        torch.cuda.synchronize()
        assert torch.equal(buf.data["obs"][:, t].cpu(), obs)
        assert torch.equal(buf.data["act"][:, t], act) and torch.equal(buf.data["log_prob"][:, t], logp)
        assert torch.equal(buf.data["value_r"][:, t], vr) and torch.equal(buf.data["value_c"][:, t], vc)
        vr2, vc2 = pol.values(obs.to(dev))
        assert torch.equal(vr2, vr) and torch.equal(vc2, vc)
        dact, dlogp, _, _ = pol.step(obs.to(dev), deterministic=True)
        with torch.no_grad():
            da, dl, _, _ = O.policy_step(opol, obs, deterministic=True)
        assert close(dact, da, atol=2e-6)[0] and close(dlogp, dl, atol=2e-6)[0]


def test_buffer_two_epochs_store_finish_get_vs_oracle():
    """ADVICE r1: with the reference-compatible store() / finish_path() / get() loop, path boundaries and bootstrap values of
    one epoch must not leak into the next (get() clears them).  Two epochs with different cut points against the oracle's
    PathBuffer (itself pinned to the reference's VectorizedOnPolicyBuffer), sequential-GAE mode: targets bit-exact."""
    dev = _cuda()
    from safepo.common.buffer import VectorizedOnPolicyBuffer
    N, T, D, A = 3, 12, 4, 2
    buf = VectorizedOnPolicyBuffer(Sp(D), Sp(A), size=T, device=dev, num_envs=N, gae_mode="exact")
    obuf = TR.PathBuffer(N, T, D, A, 0.99)
    g = torch.Generator().manual_seed(3)
    for epoch, cuts in enumerate(({0: [4, 11], 1: [11], 2: [2, 7, 11]}, {0: [11], 1: [5, 11], 2: [9, 11]})):
        for t in range(T):
            obs, act = torch.randn(N, D, generator=g), torch.randn(N, A, generator=g)
            rew, cost = torch.randn(N, generator=g), torch.rand(N, generator=g)
            vr, vc, lp = torch.randn(N, generator=g), torch.randn(N, generator=g), torch.randn(N, generator=g)
            buf.store(obs=obs, act=act, reward=rew, cost=cost, value_r=vr, value_c=vc, log_prob=lp)
            obuf.store(t, obs, act, rew, cost, vr, vc, lp)
            for idx in range(N):
                if t in cuts[idx]:
                    lr_, lc_ = torch.randn(1, generator=g), torch.randn(1, generator=g)
                    buf.finish_path(lr_, lc_, idx=idx)
                    obuf.finish_path(lr_, lc_, idx)
        data, want = buf.get(), obuf.get()
        for k in ("target_value_r", "target_value_c"):
            assert torch.equal(data[k].cpu(), want[k]), (epoch, k, float((data[k].cpu() - want[k]).abs().max()))
        for k in ("adv_r", "adv_c"):
            ok, ea, er = close(data[k], want[k], rtol=RTOL, atol=2e-6)
            assert ok, (epoch, k, ea, er)
        assert int(buf.seg_end.sum()) == 0 and float(buf.boot_r.abs().sum()) == 0.0


# ---------------------------------------------------------------------------------------
# G1 / G3
# ---------------------------------------------------------------------------------------

def _run_gae(case, mode):
    dev = _cuda()
    from safepo import _lib as L
    N, T = case["rew"].shape
    outs = [torch.empty(N, T, device=dev) for _ in range(4)]
    ins = [case[k].to(dev).contiguous() for k in ("rew", "cost", "v_r", "v_c", "seg_end", "boot_r", "boot_c")]
    L.check(L.lib().spo_gae_dual(*[L.ptr(x) for x in ins], float(case["gamma"]), float(case["gamma"] * case["lam"]),
                                 float(case["gamma"] * case["lam_c"]), *[L.ptr(o) for o in outs], N, T, mode, L.stream()),
            "spo_gae_dual")
    torch.cuda.synchronize()
    return [o.cpu() for o in outs]


def test_gae_exact_mode_bit_exact_vs_reference_buffer(golden):
    for c in golden("gae")["gae_cases"]:
        outs = _run_gae(c, 1)
        for got, key in zip(outs, ("adv_r", "adv_c", "target_value_r", "target_value_c")):
            assert torch.equal(got, c["raw"][key]), key


def test_gae_scan_mode_within_one_ulp(golden):
    for c in golden("gae")["gae_cases"]:
        outs = _run_gae(c, 0)
        for got, key in zip(outs, ("adv_r", "adv_c", "target_value_r", "target_value_c")):
            want = c["raw"][key]
            ulp = (got.view(torch.int32) - want.view(torch.int32)).abs()
            assert int(ulp.max()) <= 1, (key, int(ulp.max()))
            assert close(got, want, rtol=1e-6, atol=1e-7)[0]


@pytest.mark.parametrize("N,T", [(1024, 1000), (4, 5000), (1024, 19), (7, 513), (3, 1), (300, 512)])
def test_gae_full_size_vs_oracle(N, T):
    g = torch.Generator().manual_seed(N * 7919 + T)
    seg = (torch.rand(N, T, generator=g) < 0.004)
    seg[:, -1] = True
    term = (torch.rand(N, T, generator=g) < 0.3) & seg
    case = dict(rew=0.01 * torch.randn(N, T, generator=g), cost=(torch.rand(N, T, generator=g) < 0.05).float(),
                v_r=torch.randn(N, T, generator=g), v_c=torch.randn(N, T, generator=g).abs(), seg_end=seg.to(torch.uint8),
                boot_r=torch.randn(N, T, generator=g) * seg * ~term, boot_c=torch.randn(N, T, generator=g) * seg * ~term,
                gamma=0.99, lam=0.95, lam_c=0.95)
    want = O.gae_dual_np(case["rew"], case["cost"], case["v_r"], case["v_c"], case["seg_end"], case["boot_r"], case["boot_c"])
    exact = _run_gae(case, 1)
    scan = _run_gae(case, 0)
    hist = {}
    for e, s, w in zip(exact, scan, want):
        assert torch.equal(e, w)                                                   # sequential kernel: bit-exact
        ulp = (s.view(torch.int32) - w.view(torch.int32)).abs()
        assert int(ulp.max()) <= 1
        hist[int(ulp.max())] = hist.get(int(ulp.max()), 0) + int((ulp > 0).sum())
        assert close(s, w, rtol=1e-6, atol=1e-7)[0]
    # size-independent property: zeroing rewards and values gives identically zero outputs
    zero = dict(case, rew=torch.zeros(N, T), cost=torch.zeros(N, T), v_r=torch.zeros(N, T), v_c=torch.zeros(N, T),
                boot_r=torch.zeros(N, T), boot_c=torch.zeros(N, T))
    assert all(float(o.abs().max()) == 0.0 for o in _run_gae(zero, 0))


def test_buffer_get_matches_reference_known_answer(golden):
    """SURVEY Appendix B.2 through the drop-in buffer API (store / finish_path / get)."""
    dev = _cuda()
    from safepo.common.buffer import VectorizedOnPolicyBuffer
    kat = golden("gae")["buffer_kat"]
    buf = VectorizedOnPolicyBuffer(Sp(1), Sp(1), size=4, device=dev, num_envs=2, gae_mode="exact")
    for t in range(4):
        z = torch.tensor([float(t), 10.0 + t])      # inputs formed on the CPU like the fixture (CUDA divides via reciprocal)
        buf.store(obs=torch.tensor([[t + 0.0], [t + 100.0]]), act=torch.zeros(2, 1), reward=z,
                  cost=z / 2, value_r=z / 10, value_c=z / 5, log_prob=torch.zeros(2))
        if t == 1:
            buf.finish_path(idx=0)
        if t == 3:
            buf.finish_path(torch.tensor([0.7]), torch.tensor([0.3]), idx=0)
            buf.finish_path(torch.tensor([1.1]), torch.tensor([0.9]), idx=1)
    data = buf.get()
    assert data["obs"][:, 0].cpu().tolist() == [0, 1, 2, 3, 100, 101, 102, 103]       # flat index = env*T + t
    assert torch.equal(data["target_value_r"].cpu(), kat["target_value_r"])
    assert torch.equal(data["target_value_c"].cpu(), kat["target_value_c"])
    for k in ("adv_r", "adv_c"):
        ok, ea, er = close(data[k], kat[k], rtol=RTOL, atol=2e-6)
        assert ok, (k, ea, er)
    assert buf.ptr_list == [0, 0] and buf.path_start_idx_list == [0, 0]


def test_adv_finalize_vs_oracle():
    dev = _cuda()
    from safepo.common.buffer import VectorizedOnPolicyBuffer
    for (N, T, lam) in ((1024, 1000, 0.37), (4, 50, 0.0), (3, 7, 1.9)):
        g = torch.Generator().manual_seed(N + T)
        buf = VectorizedOnPolicyBuffer(Sp(1), Sp(1), size=T, device=dev, num_envs=N)
        adv_r, adv_c = torch.randn(N, T, generator=g) * 3 + 0.5, torch.randn(N, T, generator=g).abs()
        buf.data["adv_r"].copy_(adv_r); buf.data["adv_c"].copy_(adv_c)
        mixed = buf.finalize(lam).cpu()
        a, c, m = O.adv_finalize(adv_r.reshape(-1), adv_c.reshape(-1), lam)
        for got, want in ((buf.data["adv_r"].reshape(-1), a), (buf.data["adv_c"].reshape(-1), c), (mixed, m)):
            ok, ea, er = close(got, want, rtol=RTOL, atol=2e-6)
            assert ok, (N, T, ea, er)


# ---------------------------------------------------------------------------------------
# U1 / U2 / U3
# ---------------------------------------------------------------------------------------

def _upd_setup(c, kind):
    dev = _cuda()
    from safepo import _lib as L
    from safepo.single_agent._engine import PolicyGradientUpdate
    pol = make_policy(c["init"], c["D"], c["A"])
    cfg = dict(hidden_sizes=[64, 64], gamma=0.99, target_kl=0.02, batch_size=c["batch"], learning_iters=1, max_grad_norm=40.0)
    upd = PolicyGradientUpdate(pol, cfg, L.LOSS_PPO_CLIP if kind == "ppo" else L.LOSS_FOCOPS, epochs=10**9, host_rng=False,
                               device=dev)
    data = {k: v.to(dev).contiguous() for k, v in c["data"].items()}
    lam = c["lam"]
    data["adv"] = ((c["data"]["adv_r"] - lam * c["data"]["adv_c"]) / (lam + 1)).to(dev)
    return pol, upd, data


@pytest.mark.parametrize("kind", ["ppo", "focops"])
def test_update_single_steps_vs_reference(golden, kind):
    """The first minibatch steps one launch each: per-step losses of the reference."""
    c = golden("update")["update_chain"][kind]
    pol, upd, data = _upd_setup(c, kind)
    B = c["batch"]
    perm = c["perms"][0]
    n_steps = (perm.numel() + B - 1) // B
    for s in range(n_steps):
        idx = perm[s * B:(s + 1) * B]
        upd.cfg["target_kl"] = 1e9 if kind == "ppo" else 0.02
        upd.hp.focops_kl = 0.02
        res = upd.run(data, perms=[idx], refresh_old=(s == 0))
        want = c["losses"][s]
        for name, got, w in (("loss_r", res["loss_r"], want[0]), ("loss_c", res["loss_c"], want[1]), ("loss_pi", res["loss_pi"], want[2])):
            ok, ea, er = close(got, w, rtol=2e-5, atol=2e-6)
            assert ok, (kind, s, name, got, float(w), ea, er)
        assert res["steps"] == 1


@pytest.mark.parametrize("kind", ["ppo", "focops"])
def test_update_chain_vs_reference(golden, kind):
    """8 passes x 16 minibatches (128 consecutive Adam steps incl. the short last batch):
    pass-mean losses, the full-batch KL after every pass and the final weights."""
    c = golden("update")["update_chain"][kind]
    pol, upd, data = _upd_setup(c, kind)
    B = c["batch"]
    steps_per_pass = (c["perms"][0].numel() + B - 1) // B
    for p, perm in enumerate(c["perms"]):
        upd.cfg["target_kl"] = 1e9      # never stop: the fixture ran all 8 passes
        upd.hp.focops_kl = 0.02
        res = upd.run(data, perms=[perm], refresh_old=(p == 0))
        want = c["losses"][p * steps_per_pass:(p + 1) * steps_per_pass].double().mean(0)
        for name, got, w in (("loss_r", res["loss_r"], want[0]), ("loss_c", res["loss_c"], want[1]), ("loss_pi", res["loss_pi"], want[2])):
            ok, ea, er = close(got, w, rtol=1e-4, atol=1e-5)
            assert ok, (kind, p, name, got, float(w), ea, er)
        assert res["steps"] == steps_per_pass and res["stop_iter"] == 1
    final = policy_state(pol)
    worst = 0.0
    for net in O.NET_ORDER:
        for k, v in c["final"][net].items():
            err = float((final[net][k] - v).abs().max())
            worst = max(worst, err)
            assert err < 2e-4, (net, k, err)       # 128 chained Adam steps (lr 3e-4): sign-level drift on tiny grads
    print("max |dtheta| after 128 steps:", worst)


def test_full_batch_kl_vs_reference(golden):
    dev = _cuda()
    from safepo import _lib as L
    from safepo.single_agent._engine import make_ctrl, read_ctrl
    c = golden("update")["update_chain"]["ppo"]
    pol_old = oracle_policy(c["init"], c["D"], c["A"])
    with torch.no_grad():
        old_mean, _ = O.actor_mean_std(pol_old, c["data"]["obs"])
    pol = make_policy(c["final"], c["D"], c["A"])
    ctrl = make_ctrl(dev)
    obs = c["data"]["obs"].to(dev)
    old_ls = c["init"]["actor"]["log_std"].to(dev)
    old_mean_d = old_mean.contiguous().to(dev)      # keep device operands alive across the asynchronous launch
    for reduce, scale in ((0, 1.0), (1, 1.0 / c["A"])):
        ctrl.zero_()
        L.check(L.lib().spo_actor_kl(C.byref(pol.dims), L.ptr(pol.flat), L.ptr(obs), L.ptr(old_mean_d),
                                     L.ptr(old_ls), obs.shape[0], reduce, 0.02, L.ptr(ctrl), L.stream()), "spo_actor_kl")
        r = read_ctrl(ctrl)
        want = float(c["kls"][-1]) * scale
        assert abs(float(r["final_kl"]) - want) <= 1e-5 * abs(want) + 1e-7, (float(r["final_kl"]), want)
        assert int(r["passes"]) == 1 and int(r["stop"]) == int(want > 0.02)
    # a set stop flag turns the next update launch into a no-op
    from safepo.single_agent._engine import PolicyGradientUpdate


@pytest.mark.parametrize("kind,D,A,batch", [
    ("ppo", 17, 6, 64),       # obs_dim % 4 != 0: scalar stage-in path; 6 action dims
    ("focops", 27, 8, 64),    # widest action space: 26 side-data columns per row
    ("ppo", 104, 3, 64),      # obs_dim > 64: two W1 column blocks (moments of the second in shared memory)
    ("ppo", 60, 2, 128),      # two 64-row tiles per minibatch step
    ("ppo", 60, 2, 100),      # ragged second tile in every step
    ("focops", 60, 2, 48),    # minibatch smaller than the tile
    ("ppo", 1, 1, 64),        # smallest supported shapes
    ("pg", 60, 2, 64),        # SPO_LOSS_PG: the surrogate without the clip (pg.py:309)
    ("pg", 17, 6, 100),
])
def test_update_other_shapes_vs_oracle(kind, D, A, batch):
    """One pass of minibatch steps at shapes the golden fixtures do not cover, against the oracle's
    loop (oracle/spo_oracle.py minibatch_step, pinned to the reference by tests/test_oracle_golden.py):
    pass-mean losses and the weights after the pass.  The last step of the pass is short (13 rows)."""
    from safepo import _lib as L
    from safepo.common.model import ActorVCritic
    from safepo.single_agent._engine import PolicyGradientUpdate
    dev = _cuda()
    torch.manual_seed(1000 * D + 10 * A + batch)
    pol = ActorVCritic(D, A, [64, 64]).to(dev)
    state = policy_state(pol)
    opol = oracle_policy(state, D, A)
    S = 5 * batch + 13
    g = torch.Generator().manual_seed(S)
    obs = torch.randn(S, D, generator=g)
    with torch.no_grad():
        mean, std = O.actor_mean_std(opol, obs)
        act = mean + std * torch.randn(S, A, generator=g)
        logp = O.normal_log_prob(act, mean, std).sum(-1) + 0.05 * torch.randn(S, generator=g)
        old_mean, old_std = mean.clone(), std.expand_as(mean).clone()
    data_cpu = {"obs": obs, "act": act, "log_prob": logp, "target_value_r": torch.randn(S, generator=g),
                "target_value_c": torch.randn(S, generator=g).abs(), "adv": torch.randn(S, generator=g)}
    perm = torch.randperm(S, generator=g)
    cfg = dict(hidden_sizes=[64, 64], gamma=0.99, target_kl=1e9, batch_size=batch, learning_iters=1, max_grad_norm=40.0)
    upd = PolicyGradientUpdate(pol, cfg, {"ppo": L.LOSS_PPO_CLIP, "pg": L.LOSS_PG, "focops": L.LOSS_FOCOPS}[kind], epochs=10**9,
                               host_rng=False, device=dev)
    upd.hp.focops_kl = 0.02
    data = {k: v.to(dev).contiguous() for k, v in data_cpu.items()}
    res = upd.run(data, perms=[perm], refresh_old=True)
    opt = O.OracleOptim(opol)
    losses = []
    for s0 in range(0, S, batch):
        idx = perm[s0:s0 + batch]
        b = {k: v[idx] for k, v in data_cpu.items()}
        b["old_mean"], b["old_std"] = old_mean[idx], old_std[idx]
        losses.append(O.minibatch_step(opol, opt, b, kind))
    want = torch.tensor(losses, dtype=torch.float64).mean(0)
    n_steps = (S + batch - 1) // batch
    assert res["steps"] == n_steps
    for name, got, w in (("loss_r", res["loss_r"], want[0]), ("loss_c", res["loss_c"], want[1]), ("loss_pi", res["loss_pi"], want[2])):
        ok, ea, er = close(got, w, rtol=5e-5, atol=5e-6)
        assert ok, (kind, D, A, batch, name, got, float(w), ea, er)
    final, ofinal = policy_state(pol), opol.state()
    for net in O.NET_ORDER:
        for k, v in ofinal[net].items():
            err = float((final[net][k] - v).abs().max())
            assert err < 5e-5, (kind, D, A, batch, net, k, err)    # 6 Adam steps of lr 3e-4


@pytest.mark.gpu
@pytest.mark.parametrize("kind,D,batch,max_norm", [
    ("ppo", 60, 64, 0.05),     # every step clipped: every speculative Adam step is undone and redone
    ("ppo", 60, 64, 2.5),      # around the typical joint norm (2.0 .. 2.8 here): clipped and unclipped steps alternate
    ("focops", 27, 64, 2.9),   # the same for FOCOPS (2.6 .. 3.3)
    ("ppo", 104, 100, 0.5),    # two W1 blocks, two tiles per step, ragged tile, clipped
])
def test_update_with_active_gradient_clip_vs_oracle(kind, D, batch, max_norm):
    """clip_grad_norm_ (ppo_lag.py:325) with a limit the joint norm exceeds.  The kernel runs Adam before the
    cluster-wide norm is known and repeats the step with the clip coefficient when it turns out < 1: weights after
    12 steps and the pass-mean losses against the oracle; the number of clipped steps is counted on the oracle side."""
    from safepo import _lib as L
    from safepo.common.model import ActorVCritic
    from safepo.single_agent._engine import PolicyGradientUpdate
    dev = _cuda()
    A = 2 if D != 27 else 8
    torch.manual_seed(77 + D)
    pol = ActorVCritic(D, A, [64, 64]).to(dev)
    state = policy_state(pol)
    opol = oracle_policy(state, D, A)
    S = 11 * batch + 29
    g = torch.Generator().manual_seed(S + D)
    obs = torch.randn(S, D, generator=g)
    with torch.no_grad():
        mean, std = O.actor_mean_std(opol, obs)
        act = mean + std * torch.randn(S, A, generator=g)
        logp = O.normal_log_prob(act, mean, std).sum(-1) + 0.05 * torch.randn(S, generator=g)
        old_mean, old_std = mean.clone(), std.expand_as(mean).clone()
    data_cpu = {"obs": obs, "act": act, "log_prob": logp, "target_value_r": torch.randn(S, generator=g),
                "target_value_c": torch.randn(S, generator=g).abs(), "adv": torch.randn(S, generator=g)}
    perm = torch.randperm(S, generator=g)
    cfg = dict(hidden_sizes=[64, 64], gamma=0.99, target_kl=1e9, batch_size=batch, learning_iters=1, max_grad_norm=max_norm)
    upd = PolicyGradientUpdate(pol, cfg, {"ppo": L.LOSS_PPO_CLIP, "focops": L.LOSS_FOCOPS}[kind], epochs=10**9, host_rng=False, device=dev)
    upd.hp.focops_kl = 0.02
    data = {k: v.to(dev).contiguous() for k, v in data_cpu.items()}
    res = upd.run(data, perms=[perm], refresh_old=True)
    opt = O.OracleOptim(opol)
    losses, clipped = [], 0
    for s0 in range(0, S, batch):
        idx = perm[s0:s0 + batch]
        b = {k: v[idx] for k, v in data_cpu.items()}
        b["old_mean"], b["old_std"] = old_mean[idx], old_std[idx]
        losses.append(O.minibatch_step(opol, opt, b, kind, max_grad_norm=max_norm))
        norm = torch.sqrt(sum((p.grad ** 2).sum() for p in opol.all_params() if p.grad is not None))
        clipped += int(float(norm) >= max_norm * 0.999)     # grads are the clipped ones here: norm == max_norm when clipped
    n_steps = (S + batch - 1) // batch
    assert res["steps"] == n_steps
    if max_norm <= 0.05:
        assert clipped == n_steps
    else:
        assert 0 < clipped, (clipped, n_steps)
    want = torch.tensor(losses, dtype=torch.float64).mean(0)
    for name, got, w in (("loss_r", res["loss_r"], want[0]), ("loss_c", res["loss_c"], want[1]), ("loss_pi", res["loss_pi"], want[2])):
        ok, ea, er = close(got, w, rtol=5e-5, atol=5e-6)
        assert ok, (kind, D, batch, max_norm, name, got, float(w), ea, er)
    final, ofinal = policy_state(pol), opol.state()
    for net in O.NET_ORDER:
        for k, v in ofinal[net].items():
            err = float((final[net][k] - v).abs().max())
            assert err < 1e-4, (kind, D, batch, max_norm, net, k, err, clipped, n_steps)    # 12 Adam steps of lr 3e-4


# ---------------------------------------------------------------------------------------
# env I/O transforms (SURVEY 8f rank 1; oracle/envio.py restates third-party gymnasium: parity unpinned)
# ---------------------------------------------------------------------------------------

@pytest.mark.parametrize("N,D", [(1024, 60), (7, 33), (1, 1), (300, 128)])
def test_obs_normalize_vs_oracle(N, D):
    """Running statistics (fp64) to 1e-12 relative over 6 env steps, normalised observations to 1 fp32 ulp
    (the oracle's float64 output rounded to fp32, as torch.as_tensor(..., dtype=float32) does)."""
    from oracle import envio
    from safepo.common.normalizer import SafeNormalizeObservation
    dev = _cuda()
    rng = np.random.default_rng(N * 1000 + D)
    norm = SafeNormalizeObservation(D, dev)
    onorm = envio.NormalizeObservation(D)
    for step in range(6):
        x = (rng.normal(1.5, 4.0, size=(N, D)) * (1 + np.arange(D)) * 0.1).astype(np.float32)
        got = norm.normalize(torch.from_numpy(x).to(dev))
        want = onorm.normalize(x.astype(np.float64))
        np.testing.assert_allclose(norm.obs_rms.mean.cpu().numpy(), onorm.obs_rms.mean, rtol=1e-12, atol=1e-300)
        np.testing.assert_allclose(norm.obs_rms.var.cpu().numpy(), onorm.obs_rms.var, rtol=1e-12, atol=1e-300)
        assert abs(norm.obs_rms.count - onorm.obs_rms.count) < 1e-9
        w32 = want.astype(np.float32)
        err = np.abs(got.cpu().numpy() - w32)
        assert (err <= np.spacing(np.abs(w32)) + 1e-30).all(), (N, D, step, float(err.max()))
    x = rng.normal(size=(N, D)).astype(np.float32)
    got = norm.normalize(torch.from_numpy(x).to(dev), update=False)           # evaluation mode: statistics frozen
    want = onorm.normalize(x.astype(np.float64), update=False).astype(np.float32)
    assert (np.abs(got.cpu().numpy() - want) <= np.spacing(np.abs(want)) + 1e-30).all()
    assert abs(norm.obs_rms.count - onorm.obs_rms.count) < 1e-9


def test_action_rescale_vs_oracle():
    from oracle import envio
    from safepo.common.normalizer import SafeRescaleAction
    dev = _cuda()
    rng = np.random.default_rng(5)
    low, high = np.array([-2.0, 0.0, -0.3], np.float32), np.array([2.0, 10.0, 0.4], np.float32)
    act = (rng.normal(size=(1024, 3)) * 1.2).astype(np.float32)
    got = SafeRescaleAction(low, high, dev).action(torch.from_numpy(act).to(dev)).cpu().numpy()
    want = envio.rescale_action(act.astype(np.float64), low.astype(np.float64), high.astype(np.float64))
    np.testing.assert_allclose(got, want, rtol=1e-6, atol=1e-6)
    assert (got >= low).all() and (got <= high).all()


def test_trainer_with_device_obs_normalisation(tmp_path):
    """--normalize-obs end to end: the rollout normalises every observation batch on the device (reset
    included); after one epoch the running statistics equal the oracle's over the same raw stream, and the
    buffer holds the oracle's normalised observations."""
    from oracle import envio
    from safepo.common import synthetic_env as senv
    from safepo.common.buffer import VectorizedOnPolicyBuffer
    from safepo.common.logger import EpochLogger
    from safepo.common.model import ActorVCritic
    from safepo.single_agent._engine import Rollout
    from safepo.utils.config import single_agent_args
    dev = _cuda()
    N, T = 5, 37
    args, _ = single_agent_args(["--num-envs", str(N), "--normalize-obs", "--rng", "host", "--log-dir", str(tmp_path)])
    D, A = senv.TASK_DIMS[args.task]
    env = senv.SyntheticVecEnv(N, D, A, episode_len=20, seed=9, stagger=True)
    torch.manual_seed(0)
    pol = ActorVCritic(D, A).to(dev)
    buf = VectorizedOnPolicyBuffer(Sp(D), Sp(A), size=T, device=dev, num_envs=N)
    logger = EpochLogger(log_dir=str(tmp_path / "run"), seed="0")
    ro = Rollout(env, pol, buf, logger, args, dev)
    ro.run(T)
    # replay the raw observation stream through the oracle: same env, same actions (stored in the buffer)
    env2 = senv.SyntheticVecEnv(N, D, A, episode_len=20, seed=9, stagger=True)
    onorm = envio.NormalizeObservation(D)
    obs, _ = env2.reset()
    cur = onorm.normalize(np.asarray(obs, dtype=np.float32).astype(np.float64))
    acts = buf.data["act"].cpu().numpy().reshape(N, T, A)
    stored = buf.data["obs"].cpu().numpy().reshape(N, T, D)
    for t in range(T):
        w32 = cur.astype(np.float32)
        assert (np.abs(stored[:, t] - w32) <= np.spacing(np.abs(w32)) + 1e-30).all(), t
        nxt = env2.step(acts[:, t])[0]
        cur = onorm.normalize(np.asarray(nxt, dtype=np.float32).astype(np.float64))
    np.testing.assert_allclose(ro.obs_norm.obs_rms.mean.cpu().numpy(), onorm.obs_rms.mean, rtol=1e-12, atol=1e-300)
    np.testing.assert_allclose(ro.obs_norm.obs_rms.var.cpu().numpy(), onorm.obs_rms.var, rtol=1e-12, atol=1e-300)
    assert abs(ro.obs_norm.obs_rms.count - onorm.obs_rms.count) < 1e-9


# ---------------------------------------------------------------------------------------
# end to end
# ---------------------------------------------------------------------------------------

@pytest.mark.parametrize("algo", ["ppo_lag", "focops", "ppo", "pg", "cppo_pid", "cup"])
def test_trainer_tracks_oracle_trainer(tmp_path, algo):
    """The drop-in CLI entry (main) on the synthetic env in host-RNG (parity) mode follows
    oracle.trainers.train -- i.e. the reference's main() -- through two epochs."""
    import importlib
    from safepo.common import synthetic_env as senv
    from safepo.utils.config import single_agent_args
    mod = importlib.import_module(f"safepo.single_agent.{algo}")
    N, T, L_ep = 6, 120, 40
    extra = ["--cost-limit", "5.0"] if algo == "cppo_pid" else (["--cost-limit", "0.2"] if algo == "cup" else [])   # limits the synthetic costs exceed
    argv = ["--seed", "3", "--num-envs", str(N), "--steps-per-epoch", str(N * T), "--total-steps", str(2 * N * T),
            "--rng", "host", "--gae", "exact", "--log-dir", str(tmp_path)] + extra
    args, _ = single_agent_args(argv)
    args.log_dir = str(tmp_path / "exp" / args.task / algo / "run")
    D, A = senv.TASK_DIMS[args.task]
    env = senv.SyntheticVecEnv(N, D, A, episode_len=L_ep, seed=3, stagger=True, p_terminate=0.01)
    pol, logger, timings, _ = mod.main(args, env=env, quiet=True)
    oargs = TR.default_args(seed=3, num_envs=N, steps_per_epoch=N * T, total_steps=2 * N * T, cost_limit=args.cost_limit)
    oenv = senv.SyntheticVecEnv(N, D, A, episode_len=L_ep, seed=3, stagger=True, p_terminate=0.01)
    opol, olog, _ = TR.train(algo, oargs, oenv)
    import csv
    rows = list(csv.DictReader(open(tmp_path / "exp" / args.task / algo / "run" / "progress.csv")))
    assert len(rows) == len(olog.rows) == 2
    for got, want in zip(rows, olog.rows):
        for k in ("Metrics/EpRet", "Metrics/EpCost", "Metrics/EpLen", "Train/Epoch", "Train/TotalSteps", "Train/LR"):
            assert float(got[k]) == pytest.approx(float(want[k]), rel=1e-6, abs=1e-9), k
        assert ("Train/LagragianMultiplier" in got) == ("Train/LagragianMultiplier" in want) == (algo not in ("ppo", "pg"))
        if "Train/LagragianMultiplier" in want:
            assert float(got["Train/LagragianMultiplier"]) == pytest.approx(float(want["Train/LagragianMultiplier"]), rel=1e-5, abs=1e-8)
        assert int(float(got["Train/StopIter"])) == int(want["Train/StopIter"])
        if algo == "cup":
            assert int(float(got["Train/SeconStageStopIter"])) == int(want["Train/SeconStageStopIter"])
        for k in ("Loss/Loss_reward_critic", "Loss/Loss_cost_critic", "Loss/Loss_actor", "Train/KL"):
            assert float(got[k]) == pytest.approx(float(want[k]), rel=2e-3, abs=2e-5), (k, got[k], want[k])
    # first-epoch rollout (before any update) must agree to fp32 rounding: compare actor weights loosely after 2 epochs
    for k, v in opol.nets["actor"].items():
        assert float((pol.actor.state_dict()[k].cpu() - v.detach()).abs().max()) < 5e-3, k


# ---------------------------------------------------------------------------------------
# C1-C5: trust-region pieces
# ---------------------------------------------------------------------------------------

def _trust_setup(golden):
    dev = _cuda()
    from safepo.single_agent._engine import TrustRegionUpdate
    c = golden("trust")["trust"]
    pol = make_policy(c["state"], c["D"], c["A"])
    cfg = dict(hidden_sizes=[64, 64], gamma=0.99, target_kl=0.01, batch_size=128, learning_iters=10, max_grad_norm=40.0)
    tr = TrustRegionUpdate(pol, cfg, dev)
    data = {k: v.to(dev).contiguous() for k, v in c["data"].items()}
    return c, pol, tr, data, dev


def test_surrogate_grad_vs_reference(golden):
    c, pol, tr, data, dev = _trust_setup(golden)
    loss = tr._grad(data, data["adv_r"], tr.g)
    assert close(loss, c["surr"], rtol=RTOL, atol=1e-7)[0], (float(loss), float(c["surr"]))
    err = (tr.g.cpu() - c["surr_grad"]).norm() / c["surr_grad"].norm()
    assert float(err) < 1e-5, float(err)
    ok, ea, er = close(tr.g, c["surr_grad"], rtol=1e-4, atol=1e-7)
    assert ok, (ea, er)


def test_fvp_closed_form_vs_reference_double_backprop(golden):
    c, pol, tr, data, dev = _trust_setup(golden)
    tr._fvp(data, c["v"].to(dev), tr.Fx)
    err = (tr.Fx.cpu() - c["Fv"]).norm() / c["Fv"].norm()
    assert float(err) < 1e-5, float(err)          # SURVEY fact 7: the closed form equals cpo.fvp
    # linearity (size-independent property): F(2v) == 2 F(v) up to the damping-consistent scaling
    out2 = torch.zeros_like(tr.Fx)
    tr._fvp(data, (2 * c["v"]).to(dev), out2)
    assert float((out2 - 2 * tr.Fx).abs().max()) < 1e-5 * float(tr.Fx.abs().max()) + 1e-7


def test_conjugate_gradient_on_device_vs_reference(golden):
    c, pol, tr, data, dev = _trust_setup(golden)
    tr._cg(data, c["rhs"].to(dev), tr.x)
    x = tr.x.cpu()
    err = (x - c["cg_x"]).norm() / c["cg_x"].norm()
    assert float(err) < 2e-3, float(err)          # 15 fp32 CG iterations amplify 1e-7-level FVP differences
    # the solve itself: residual of (H + 0.1 I) x = b measured with the reference's autograd FVP on the oracle
    opol = oracle_policy(c["state"], c["D"], c["A"])
    r_mine = O.fvp_autograd(opol, c["data"]["obs"], x) - c["rhs"]
    r_ref = O.fvp_autograd(opol, c["data"]["obs"], c["cg_x"]) - c["rhs"]
    assert float(r_mine.norm()) <= 1.5 * float(r_ref.norm()) + 1e-6


def test_linesearch_eval_vs_oracle(golden):
    c, pol, tr, data, dev = _trust_setup(golden)
    tr._old_dist(data)
    opol = oracle_policy(c["state"], c["D"], c["A"])
    with torch.no_grad():
        om, os_ = O.actor_mean_std(opol, c["data"]["obs"])
        om, os_ = om.clone(), os_.clone()
    g = torch.Generator().manual_seed(2)
    step = 0.02 * torch.randn(c["P"], generator=g)
    pol.actor_flat().add_(step.to(dev))
    O.set_flat_params(opol, O.flat_params(opol) + step)
    out = tr._eval(data, data["adv_r"], data["adv_c"])
    d = c["data"]
    with torch.no_grad():
        want0 = O.surrogate_loss(opol, d["obs"], d["act"], d["log_prob"], d["adv_r"])
        want1 = O.surrogate_loss(opol, d["obs"], d["act"], d["log_prob"], d["adv_c"])
        m, s = O.actor_mean_std(opol, d["obs"])
        want2 = O.normal_kl(om, os_, m, s).mean()
    for got, want in zip(out, (want0, want1, want2)):
        assert close(got, want, rtol=2e-5, atol=1e-7)[0], (float(got), float(want))


@pytest.mark.parametrize("algo", ["cpo", "trpo_lag", "trpo", "natural_pg", "rcpo", "pcpo"])
def test_trust_region_trainer_tracks_oracle(tmp_path, algo):
    import csv
    import importlib
    from safepo.common import synthetic_env as senv
    from safepo.utils.config import single_agent_args
    mod = importlib.import_module(f"safepo.single_agent.{algo}")
    N, T, L_ep = 5, 160, 40
    task = "SafetyCarButton1-v0" if algo in ("cpo", "pcpo") else "SafetyPointGoal1-v0"
    argv = ["--seed", "5", "--num-envs", str(N), "--steps-per-epoch", str(N * T), "--total-steps", str(2 * N * T), "--task", task,
            "--rng", "host", "--gae", "exact", "--log-dir", str(tmp_path)]
    args, _ = single_agent_args(argv)
    args.log_dir = str(tmp_path / "exp" / task / algo / "run")
    D, A = senv.TASK_DIMS[task]
    env = senv.SyntheticVecEnv(N, D, A, episode_len=L_ep, seed=5, stagger=True, p_terminate=0.01)
    pol, logger, timings, _ = mod.main(args, env=env, quiet=True)
    oargs = TR.default_args(seed=5, num_envs=N, steps_per_epoch=N * T, total_steps=2 * N * T, task=task)
    oenv = senv.SyntheticVecEnv(N, D, A, episode_len=L_ep, seed=5, stagger=True, p_terminate=0.01)
    opol, olog, _ = TR.train(algo, oargs, oenv)
    rows = list(csv.DictReader(open(tmp_path / "exp" / task / algo / "run" / "progress.csv")))
    assert len(rows) == len(olog.rows) == 2
    for got, want in zip(rows, olog.rows):
        for k in ("Metrics/EpRet", "Metrics/EpCost", "Metrics/EpLen", "Train/Epoch", "Train/TotalSteps"):
            assert float(got[k]) == pytest.approx(float(want[k]), rel=1e-6, abs=1e-9), k
        assert ("Misc/AcceptanceStep" in got) == ("Misc/AcceptanceStep" in want) == (algo not in ("natural_pg", "rcpo"))
        if "Misc/AcceptanceStep" in want:
            assert int(float(got["Misc/AcceptanceStep"])) == int(want["Misc/AcceptanceStep"])
        assert ("Train/LagragianMultiplier" in got) == ("Train/LagragianMultiplier" in want) == (algo in ("trpo_lag", "rcpo"))
        for k in ("Misc/Alpha", "Misc/xHx", "Misc/gradient_norm", "Misc/H_inv_g", "Misc/FinalStepNorm", "Loss/Loss_actor", "Train/KL",
                  "Loss/Loss_reward_critic", "Loss/Loss_cost_critic"):
            assert float(got[k]) == pytest.approx(float(want[k]), rel=5e-3, abs=5e-5), (k, got[k], want[k])


# ---------------------------------------------------------------------------------------
# full-batch forward (large S) against the oracle and small-batch calls: wgmma / TMA where obs_dim % 4 == 0 and
# obs_dim <= 64, the FFMA tile kernel over many CTAs for obs_dim 88 and 27
# ---------------------------------------------------------------------------------------

@pytest.mark.parametrize("D,A,S", [(60, 2, 4096 + 37), (60, 2, 128 * 1024), (28, 8, 2048 + 5), (64, 2, 1500),
                                   (88, 2, 4096 + 37), (27, 8, 2048 + 5)])
def test_tensor_core_forward_and_kl_large_batch(D, A, S):
    dev = _cuda()
    from safepo import _lib as L
    from safepo.common.model import ActorVCritic
    from safepo.single_agent._engine import make_ctrl, read_ctrl
    torch.manual_seed(D + A)
    pol = ActorVCritic(D, A).to(dev)
    with torch.no_grad():
        pol.actor.log_std.copy_(torch.linspace(-0.4, 0.2, A))
    opol = oracle_policy(policy_state(pol), D, A)
    obs = torch.randn(S, D)
    with torch.no_grad():
        want, _ = O.actor_mean_std(opol, obs)
    obs_d = obs.to(dev)
    got = pol.actor_mean(obs_d)                                   # S >= 1024, D % 4 == 0 and D <= 64 -> wgmma path
    ok, ea, er = close(got, want, rtol=RTOL, atol=2e-6)
    assert ok, (D, A, S, ea, er)
    chunks = torch.cat([pol.actor_mean(obs_d[i:i + 512]) for i in range(0, S, 512)])   # small batches -> FFMA tile kernel
    assert float((chunks - got).abs().max()) < 5e-6
    # KL against a perturbed "old" distribution
    old_mean = (want + 0.05 * torch.randn(S, A)).contiguous()
    old_ls = torch.linspace(-0.3, 0.1, A)
    ctrl = make_ctrl(dev)
    old_mean_d, old_ls_d = old_mean.to(dev), old_ls.to(dev)      # keep alive across the asynchronous launch
    L.check(L.lib().spo_actor_kl(C.byref(pol.dims), L.ptr(pol.flat), L.ptr(obs_d), L.ptr(old_mean_d), L.ptr(old_ls_d), S, 0,
                                 1e9, L.ptr(ctrl), L.stream()), "spo_actor_kl")
    r = read_ctrl(ctrl)
    with torch.no_grad():
        m, s = O.actor_mean_std(opol, obs)
        want_kl = O.normal_kl(old_mean, torch.exp(old_ls), m, s).sum(-1, keepdim=True).mean().item()
    assert abs(float(r["final_kl"]) - want_kl) <= 2e-5 * abs(want_kl) + 1e-7, (float(r["final_kl"]), want_kl)
    assert int(r["passes"]) == 1


# ---- row G2: masked GAE of the multi-agent buffer (first hardware run: round-1 driver box, 4 XPASS; strict since round 2)
@pytest.mark.gpu
@pytest.mark.parametrize("T,N", [(8, 5), (64, 3), (1, 4), (33, 1024), (8, 8192)])
def test_masked_gae_bit_exact_vs_oracle(T, N):
    """spo_gae_masked (SURVEY 8 row G2) against oracle/ma_oracle.masked_gae -- itself pinned bit for bit to the reference's
    SeparatedReplayBuffer.compute_returns -- for reward and cost returns: bit-exact (sequential fp32 recurrence)."""
    from safepo.common.buffer import masked_gae_returns
    from oracle import ma_oracle as MA
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(T * 1000 + N)
    pop = MA.OraclePopArt(1)
    for _ in range(3):
        pop.normalize(torch.randn(40, 1, generator=g) * 3 + 1.5)
    mean, var = pop.running_mean_var()
    sqrt_var = torch.sqrt(var)
    vp = torch.randn(T + 1, N, 1, generator=g)
    rew = torch.randn(T, N, 1, generator=g)
    masks = (torch.rand(T + 1, N, 1, generator=g) > 0.15).float()
    want = MA.masked_gae(rew, vp, masks, pop, 0.96, 0.95)
    got = masked_gae_returns(rew.to(dev), vp.to(dev), masks.to(dev), float(mean), float(sqrt_var), 0.96, 0.95).cpu()
    assert torch.equal(got, want), float((got - want).abs().max())


def _ma_state(g, din, H, A, head):
    """A MultiAgentActor / MultiAgentCritic state dict (reference names, model.py:172-363) with non-trivial LayerNorm
    parameters and biases."""
    st = {"base.feature_norm.weight": 1 + 0.1 * torch.randn(din, generator=g), "base.feature_norm.bias": 0.1 * torch.randn(din, generator=g)}
    dims = [din, H, H, H]
    for li, name in enumerate(("fc1", "fc2.0", "fc2.1")):
        st[f"base.mlp.{name}.0.weight"] = torch.randn(H, dims[li], generator=g) * (1.4 / dims[li] ** 0.5)
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


# ---- SURVEY 8f rank 3, first slice: multi-agent nets, forward (MAPPO_L_Policy.get_actions) against the pinned oracle
@pytest.mark.gpu
@pytest.mark.parametrize("N,D,DS,A,H", [(24, 10, 14, 3, 128), (8192, 398, 398, 20, 512), (77, 66, 130, 5, 256)])
def test_ma_get_actions_vs_oracle(N, D, DS, A, H):
    """spo_ma_mlp_layer / spo_ma_head through safepo.common.ma_model.MultiAgentNets against oracle/ma_oracle.py (pinned bit for
    bit to the reference's MAPPO_L_Policy, tests/golden/ma_update.pt); the middle case is config 5's shape
    (ShadowHandOver: obs 398, act 20, hidden 512, 8192 envs).  1e-5 relative on values / actions / per-dimension log-probs."""
    from oracle import ma_oracle as MA
    from safepo.common.ma_model import MultiAgentNets
    dev = _cuda()
    g = torch.Generator().manual_seed(N + D)

    def make(din, head):
        return _ma_state(g, din, H, A, head)

    sa, sc, sk = make(D, "actor"), make(DS, "critic"), make(DS, "critic")
    obs, cent = torch.randn(N, D, generator=g) * 2 + 0.3, torch.randn(N, DS, generator=g) * 3
    eps = torch.randn(N, A, generator=g)
    nets = MultiAgentNets(sa, sc, sk, dev)
    oa, oc, ok_ = MA.OracleMANet(sa), MA.OracleMANet(sc), MA.OracleMANet(sk)
    with torch.no_grad():
        dist = MA.ma_actor_dist(oa, obs)
        want_act = dist.mean + dist.stddev * eps
        want = (MA.ma_critic_value(oc, cent), want_act, dist.log_prob(want_act), MA.ma_critic_value(ok_, cent))
        want_det = (dist.mean, dist.log_prob(dist.mean))
    got = nets.get_actions(cent.to(dev), obs.to(dev), eps=eps.to(dev))
    # three 398/512-wide fp32 layers, each followed by a LayerNorm: the reordering noise of two fp32 implementations is ~1e-6
    # per element and a few 1e-6 at the maximum over N x 512 activations (printed)
    worst = {}
    for name, a_, b_ in zip(("values", "actions", "logp", "cost"), got, want):
        ok, ea, er = close(a_, b_, rtol=2e-5, atol=1e-5)
        worst[name] = (ea, float((a_.cpu() - b_).abs().mean()))
        assert ok, (name, N, D, H, ea, er)
    print(f"\nMA get_actions N={N} D={D} H={H}: max / mean |err| " + ", ".join(f"{k} {v[0]:.2e} / {v[1]:.2e}" for k, v in worst.items()))
    gd = nets.get_actions(cent.to(dev), obs.to(dev), deterministic=True)
    assert close(gd[1], want_det[0], rtol=2e-5, atol=1e-5)[0] and close(gd[2], want_det[1], rtol=2e-5, atol=1e-5)[0]
    assert gd[2].shape == (N, A)          # log-probs stay per action dimension (distributions.py:8-9)


# ---- SURVEY 8f rank 3, second slice: the update of the multi-agent nets (MAPPO_L_Trainer.ppo_update)
@pytest.mark.gpu
@pytest.mark.parametrize("M,N,Kd", [(100, 14, 128), (777, 130, 256), (64, 64, 16), (1000, 398, 512), (333, 512, 20), (50, 128, 1)])
def test_ma_tile_products_vs_float64(M, N, Kd):
    """spo_ma_gemm_nn (C = A B) and spo_ma_gemm_tn + spo_ma_partial_reduce (C = A^T B over row slices) against float64
    products of the same fp32 inputs: edges that are not multiples of the 128 x 64 x 32 tile, one-column and one-row operands."""
    from safepo import _lib as L
    dev = _cuda()
    g = torch.Generator().manual_seed(M * 7 + N)
    A_, B_ = torch.randn(M, Kd, generator=g), torch.randn(Kd, N, generator=g)
    C = torch.empty(M, N, device=dev)
    Ad, Bd = A_.to(dev), B_.to(dev)          # named: a temporary would be freed (and its memory reused) before the launch
    L.check(L.lib().spo_ma_gemm_nn(L.ptr(Ad), L.ptr(Bd), L.ptr(C), M, N, Kd, L.stream()), "spo_ma_gemm_nn")
    want = (A_.double() @ B_.double())
    assert float((C.cpu().double() - want).abs().max()) < 1e-5 * (Kd ** 0.5) * 4
    # transposed-A product, reduction over the M rows here: [Kd][N] = A^T [Kd][M] ... use A as [R=M][Kd], B2 as [R=M][N]
    B2 = torch.randn(M, N, generator=g)
    B2d = B2.to(dev)
    for slices in (1, 3):
        if slices > 1 and M < 200:     # three slices of whole 32-row chunks need more rows than that
            continue
        part = torch.empty(slices * Kd * N, device=dev)
        out = torch.empty(Kd, N, device=dev)
        L.check(L.lib().spo_ma_gemm_tn(L.ptr(Ad), L.ptr(B2d), L.ptr(part), M, Kd, N, slices, L.stream()), "spo_ma_gemm_tn")
        L.check(L.lib().spo_ma_partial_reduce(L.ptr(part), slices, Kd * N, 1, Kd * N, L.ptr(out), None, None, 1.0, L.stream()), "spo_ma_partial_reduce")
        want2 = A_.double().t() @ B2.double()
        assert float((out.cpu().double() - want2).abs().max()) < 1e-5 * (M ** 0.5) * 4, (slices, M, N, Kd)


@pytest.mark.gpu
@pytest.mark.parametrize("N,D,DS,A,H", [(100, 10, 14, 3, 128), (777, 66, 130, 5, 256), (2048, 398, 398, 20, 512)])
def test_ma_ppo_update_vs_oracle(golden, N, D, DS, A, H):
    """Two consecutive MAPPO_L_Trainer.ppo_update calls (mappolag.py:135-199) through safepo.common.ma_model.MultiAgentTrainer
    against oracle/ma_oracle.py OracleMATrainer (pinned to the reference's trainer by tests/golden/ma_update.pt): the gradients of
    every parameter tensor before the clip, the eight returned quantities, lamda_lagr, the PopArt statistics and all weights
    after each update.  The last case is config 5's layer shape (obs 398, act 20, hidden 512) on a quarter of its rows."""
    from oracle import ma_oracle as MA
    from safepo.common.ma_model import MultiAgentNets, MultiAgentTrainer
    dev = _cuda()
    cfg = dict(golden("ma_update")["ma_update"]["cfg"])      # the yaml's values (actor_lr 9e-5, critic_lr 5e-3, max_grad_norm 10, ...)
    cfg["entropy_coef"] = 0.01                               # the yaml has 0.0: exercise the entropy gradient of log_std too
    g = torch.Generator().manual_seed(3 * N + D)
    sa, sc, sk = _ma_state(g, D, H, A, "actor"), _ma_state(g, DS, H, A, "critic"), _ma_state(g, DS, H, A, "critic")
    oa, oc, ok_ = MA.OracleMANet(sa), MA.OracleMANet(sc), MA.OracleMANet(sk)
    obs, share = torch.randn(N, D, generator=g) * 2 + 0.5, torch.randn(N, DS, generator=g) * 3
    with torch.no_grad():
        dist = MA.ma_actor_dist(oa, obs)
        actions = dist.mean + dist.stddev * torch.randn(N, A, generator=g)
        logp = dist.log_prob(actions)
        v0, k0 = MA.ma_critic_value(oc, share), MA.ma_critic_value(ok_, share)
    sample = dict(share_obs=share, obs=obs, actions=actions, value_preds=v0 + 0.1 * torch.randn(N, 1, generator=g),
                  returns=torch.randn(N, 1, generator=g) * 4 + 1, old_action_log_probs=logp + 0.05 * torch.randn(N, A, generator=g),
                  adv_targ=torch.randn(N, 1, generator=g), factor=torch.rand(N, 1, generator=g) + 0.5,
                  cost_preds=k0 + 0.1 * torch.randn(N, 1, generator=g), cost_returns=torch.randn(N, 1, generator=g).abs() * 30,
                  cost_adv_targ=torch.randn(N, 1, generator=g), aver_episode_costs=torch.rand(N, 1, generator=g) * 60)
    otr = MA.OracleMATrainer(oa, oc, ok_, cfg)
    nets = MultiAgentNets(sa, sc, sk, dev, layer_N=cfg["layer_N"], std_x_coef=cfg["std_x_coef"], std_y_coef=cfg["std_y_coef"])
    tr = MultiAgentTrainer(nets, cfg)
    names = ("value_loss", "critic_grad_norm", "policy_loss", "dist_entropy", "actor_grad_norm", "imp_weights", "cost_loss", "cost_grad_norm")
    worst = {}
    for it in range(2):
        want = otr.ppo_update(sample)
        got = dict(zip(names, tr.ppo_update(sample)))
        torch.cuda.synchronize()
        # the second update starts from weights that already differ by fp32 reordering noise; the product of 20 per-dimension
        # ratios amplifies that (measured 1.7e-4 relative on an importance weight of ~7 at the config-5 shape)
        slack = 1.0 if it == 0 else 10.0
        for k in names:
            ok, ea, er = close(got[k].reshape(-1), want[k].reshape(-1), rtol=1e-4 * slack, atol=2e-6 * slack)
            assert ok, (it, k, ea, er)
        # gradients before the clip: the oracle's .grad are the clipped ones
        for net, onet, nk in ((nets.actor, oa, "actor_grad_norm"), (nets.critic, oc, "critic_grad_norm"), (nets.cost_critic, ok_, "cost_grad_norm")):
            coef = min(1.0, float(cfg["max_grad_norm"]) / (float(want[nk]) + 1e-6))
            for k, pt in onet.p.items():
                wg = pt.grad / coef
                err = float((net.g[k].cpu() - wg).abs().max())
                scale = float(wg.abs().max())
                worst[k] = max(worst.get(k, 0.0), err / (scale + 1e-12))
                assert err <= (5e-5 * scale + 1e-7) * slack, (it, k, err, scale)
        assert abs(float(tr.lamda_lagr) - float(otr.lamda_lagr)) <= 1e-5 * max(1.0, abs(float(otr.lamda_lagr))), (float(tr.lamda_lagr), float(otr.lamda_lagr))
        pst = tr.popart_state.cpu()
        for got_s, want_s in zip(pst, (otr.popart.running_mean, otr.popart.running_mean_sq, otr.popart.debiasing_term)):
            assert abs(float(got_s) - float(want_s)) <= 1e-5 * abs(float(want_s)) + 1e-12
        # weights: an Adam step moves an element by lr * g / (|g| + eps)-ish, so a gradient error of 1e-7 on an element whose gradient is
        # below opti_eps = 1e-5 shows up as 1 % of lr; a wrong sign would be 2 lr
        for net, onet, lr in ((nets.actor, oa, cfg["actor_lr"]), (nets.critic, oc, cfg["critic_lr"]), (nets.cost_critic, ok_, cfg["critic_lr"])):
            for k, pt in onet.p.items():
                err = float((net.p[k].cpu() - pt.detach()).abs().max())
                assert err < 0.05 * lr + 1e-6, (it, k, err, lr)
    print(f"\nMA ppo_update N={N} D={D} H={H}: worst relative gradient error per tensor {max(worst.values()):.2e}")



@pytest.mark.gpu
def test_ma_runner_iteration_vs_oracle(golden):
    """safepo/multi_agent/mappolag.py Runner on the device -- collect / insert / compute / train of two agents with
    SeparatedReplayBuffer, spo_gae_masked, MultiAgentTrainer.train and the cross-agent factor -- against the oracle's runner
    (pinned bit for bit to the reference's Runner by tests/golden/ma_epoch.pt) on a synthetic environment stream with the same
    injected draws: two iterations.  (The same host code runs against an emulated C-ABI in the CPU suite:
    tests/test_cpu_host.py::test_multi_agent_runner_iteration_vs_oracle.)"""
    from oracle import ma_oracle as MA
    from safepo.common.ma_model import MultiAgentNets
    from safepo.multi_agent.mappolag import Runner
    dev = _cuda()
    cfg = dict(golden("ma_epoch")["ma_epoch"]["cfg"])
    T, N, D, DS, A, H, NA = 4, 24, 10, 14, 3, 128, 2
    cfg.update(episode_length=T, n_rollout_threads=N)
    g = torch.Generator().manual_seed(31)
    states = [dict(actor=_ma_state(g, D, H, A, "actor"), critic=_ma_state(g, DS, H, A, "critic"), cost_critic=_ma_state(g, DS, H, A, "critic"))
              for _ in range(NA)]
    onets = [tuple(MA.OracleMANet(st[n], layer_N=cfg["layer_N"]) for n in ("actor", "critic", "cost_critic")) for st in states]
    orun = MA.OracleMARunner(onets, cfg, T, N, D, DS, A)
    nets = [MultiAgentNets(st["actor"], st["critic"], st["cost_critic"], dev, layer_N=cfg["layer_N"], std_x_coef=cfg["std_x_coef"],
                           std_y_coef=cfg["std_y_coef"]) for st in states]
    run = Runner(nets, cfg, D, DS, A)
    obs0, share0 = torch.randn(N, NA, D, generator=g) * 2 + 0.5, torch.randn(N, NA, DS, generator=g) * 3
    orun.warmup(obs0, share0)
    run.warmup(obs0, share0)

    def near(a, b, tol):
        a, b = a.detach().cpu(), b.detach().cpu()
        return float((a - b).abs().max()) <= tol * (1.0 + float(b.abs().max()))
    for it in range(2):
        for step in range(T):
            eps = [torch.randn(N, A, generator=g) for _ in range(NA)]
            ov, oact, olp, ocp = orun.collect(step, eps=eps)
            v, act, lp, cp = run.collect(step, eps=eps)
            assert near(v, ov, 5e-5) and near(cp, ocp, 5e-5) and all(near(act[a], oact[a], 5e-5) and near(lp[a], olp[a], 5e-5) for a in range(NA)), (it, step)
            obs, share = torch.randn(N, NA, D, generator=g) * 2 + 0.5, torch.randn(N, NA, DS, generator=g) * 3
            rewards, costs = torch.randn(N, NA, 1, generator=g), (torch.rand(N, NA, 1, generator=g) < 0.3).float()
            dones = (torch.rand(N, generator=g) < 0.2)[:, None].expand(N, NA).clone()
            # both sides store the ORACLE's actions / predictions, so that the buffers only differ by what is under test
            orun.insert(obs, share, rewards, costs, dones, ov, oact, olp, ocp)
            run.insert(obs, share, rewards, costs, dones, ov.to(dev), [x.to(dev) for x in oact], [x.to(dev) for x in olp], ocp.to(dev))
        orun.compute()
        run.compute()
        for a in range(NA):
            for k in ("returns", "cost_returns", "value_preds", "cost_preds", "masks", "active_masks"):
                assert near(getattr(run.buffer[a], k), getattr(orun.buffer[a], k), 1e-4), (it, a, k)
        order = torch.randperm(NA, generator=g)
        perms = [[torch.randperm(T * N, generator=g) for _ in range(cfg["learning_iters"])] for _ in range(NA)]
        orun.train(agent_order=order, perms=perms)
        assert run.train(agent_order=order, perms=perms) == [int(a) for a in order]
        torch.cuda.synchronize()
        for a in range(NA):
            assert near(run.buffer[a].factor, orun.buffer[a].factor, 5e-4), (it, a)
            assert abs(float(run.trainer[a].lamda_lagr) - float(orun.trainer[a].lamda_lagr)) < 1e-5
            pop = orun.trainer[a].popart
            for got_s, want_s in zip(run.trainer[a].popart_state.cpu(), (pop.running_mean, pop.running_mean_sq, pop.debiasing_term)):
                assert abs(float(got_s) - float(want_s)) <= 1e-4 * abs(float(want_s)) + 1e-12
            for net, onet, lr in zip((nets[a].actor, nets[a].critic, nets[a].cost_critic), onets[a], (cfg["actor_lr"], cfg["critic_lr"], cfg["critic_lr"])):
                for k, pt in onet.p.items():
                    err = float((net.p[k].cpu() - pt.detach()).abs().max())
                    assert err < 0.2 * lr + 2e-6, (it, a, k, err)       # a wrong gradient sign would be 2 lr per update
    assert any(bool((run.buffer[a].factor != 1).any()) for a in range(NA))


@pytest.mark.gpu
def test_ma_run_loop_on_device(tmp_path):
    """Runner.run on the synthetic multi-agent environment on the device (the loop's logic is checked against expectations in the
    CPU suite through the emulated C-ABI): three iterations with episodes finishing inside them -- finite losses, weights that
    move, the finished episodes' mean cost handed to the buffers, identical log rows for identical seeds."""
    from safepo.common.ma_model import MultiAgentNets
    from safepo.common.synthetic_env import SyntheticMultiAgentEnv
    from safepo.multi_agent import mappolag as M
    dev = _cuda()
    cfg = dict(M.DEFAULT_CONFIG, episode_length=4, n_rollout_threads=48, hidden_size=128, learning_iters=2, entropy_coef=0.01)
    T, N, D, DS, A, NA = 4, 48, 22, 30, 5, 2

    def build(seed):
        gg = torch.Generator().manual_seed(seed)
        nets = [MultiAgentNets(M.init_state(D, 128, 2, "actor", A, generator=gg), M.init_state(DS, 128, 2, "critic", generator=gg),
                               M.init_state(DS, 128, 2, "critic", generator=gg), dev) for _ in range(NA)]
        return M.Runner(nets, cfg, D, DS, A), SyntheticMultiAgentEnv(N, NA, D, DS, A, episode_len=3, seed=seed, device=dev)
    run, envs = build(2)
    w0 = run.nets[1].critic.flat.clone()
    torch.manual_seed(7)
    torch.cuda.manual_seed(7)
    rows = run.run(envs, 3)
    assert [r["Train/TotalSteps"] for r in rows] == [T * N, 2 * T * N, 3 * T * N]
    for r in rows:
        assert all(np.isfinite(v) for v in r.values()), r
        assert "Metrics/EpCost" in r and 0.0 <= r["Metrics/EpCost"] <= 3.0
    assert float((run.nets[1].critic.flat - w0).abs().max()) > 0
    assert run.buffer[0].aver_episode_costs.numel() == 1 and abs(float(run.buffer[0].aver_episode_costs) - rows[-1]["Metrics/EpCost"]) < 1e-6
    run2, envs2 = build(2)
    torch.manual_seed(7)
    torch.cuda.manual_seed(7)
    rows2 = run2.run(envs2, 3)
    for r, r2 in zip(rows, rows2):       # every kernel sums in a fixed order: the same seeds give the same numbers
        for k, v in r.items():
            if k not in ("Time/Total", "Time/FPS"):
                assert abs(v - r2[k]) <= 1e-6 * (1.0 + abs(v)), (k, v, r2[k])
