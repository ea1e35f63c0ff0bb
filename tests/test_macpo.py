"""MACPO (safepo/multi_agent/macpo.py, safepo/common/ma_model.py: MACPOTrainer, csrc/spo_ma_trust.cu) against the CPU restatement
of the reference's MACPO_Trainer (tests/macpo_oracle.py).  CPU tests run the host orchestration through the emulated C-ABI
(tests/macpo_emulator.py); GPU tests run the kernels."""
import math
import os
import subprocess
import sys

import pytest
import torch

from oracle import ma_oracle as MA

SHAPES = [(100, 10, 3, 128), (777, 66, 5, 256), (2048, 398, 20, 512)]


def _state(g, din, H, A, head):
    """A MultiAgentActor / MultiAgentCritic state dict with non-trivial LayerNorm parameters and biases."""
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


class Setup:
    """Actor / critics on both sides and a sample generator whose constraint value and cost advantages pick the MACPO case."""

    def __init__(self, N, D, DS, A, H, device, seed=5):
        from safepo.common.ma_model import MACPOTrainer, MultiAgentNets
        from safepo.multi_agent.macpo import DEFAULT_CONFIG
        import macpo_oracle as MO
        self.cfg = dict(DEFAULT_CONFIG, hidden_size=H)
        g = self.g = torch.Generator().manual_seed(seed)
        sa, sc, sk = _state(g, D, H, A, "actor"), _state(g, DS, H, A, "critic"), _state(g, DS, H, A, "critic")
        self.oa, self.oc, self.ok = MA.OracleMANet(sa), MA.OracleMANet(sc), MA.OracleMANet(sk)
        self.otr = MO.OracleMACPOTrainer(self.oa, self.oc, self.ok, dict(self.cfg))
        self.nets = MultiAgentNets(sa, sc, sk, device, layer_N=2)
        self.tr = MACPOTrainer(self.nets, dict(self.cfg))
        self.N, self.A = N, A
        self.obs, self.share = torch.randn(N, D, generator=g) * 2 + 0.5, torch.randn(N, DS, generator=g) * 3
        with torch.no_grad():
            dist = MA.ma_actor_dist(self.oa, self.obs)
            self.actions = dist.mean + dist.stddev * torch.randn(N, A, generator=g)
            self.logp = dist.log_prob(self.actions)

    def sample(self, aver, cadv_scale=1.0):
        N, g = self.N, self.g
        if cadv_scale == "shrink":
            # zero cost advantages and reward advantages -sum_j (z_j^2 - 1), z = (action - mean) / std: the step shrinks every std,
            # and the reference's KL (its log terms enter with the sign opposite to a true KL's) grows LINEARLY with the step
            s = self.sample(aver, 0.0)
            with torch.no_grad():
                dist = MA.ma_actor_dist(self.oa, self.obs)
                z = (self.actions - dist.mean) / dist.stddev
            s["adv_targ"] = -(z ** 2 - 1).sum(-1, keepdim=True)
            return s
        return dict(share_obs=self.share, obs=self.obs, actions=self.actions, value_preds=0.1 * torch.randn(N, 1, generator=g),
                    returns=torch.randn(N, 1, generator=g) * 4 + 1,
                    old_action_log_probs=self.logp + 0.05 * torch.randn(N, self.A, generator=g) / self.A ** 0.5,
                    adv_targ=torch.randn(N, 1, generator=g), factor=torch.rand(N, 1, generator=g) + 0.5,
                    cost_preds=0.1 * torch.randn(N, 1, generator=g), cost_returns=torch.randn(N, 1, generator=g).abs() * 30,
                    cost_adv_targ=cadv_scale * torch.randn(N, 1, generator=g), aver_episode_costs=torch.full((N, 1), float(aver)))

    def set_search(self, target_kl, searching_steps):
        for c in (self.tr.cfg, self.otr.cfg):
            c["target_kl"], c["searching_steps"] = target_kl, searching_steps


# (aver_episode_costs, cost advantages, target_kl, searching_steps, expected case, expected accepted trial).  "shrink": case 4 with a
# KL that grows linearly with the step (its size at trial 0 is ~0.01 sqrt(target_kl)), so that target_kl 1e-5 rejects trial 0 and
# accepts a later one ("later": >= 1), and target_kl 1e-6 with one trial rejects it: the old actor comes back (-1).
SCENARIOS = [(30.0, 1.0, 0.016, 10, 1, 0), (20.0, 1.0, 0.016, 10, 2, 0), (0.0, 1.0, 0.016, 10, 3, 0), (20.0, 0.0, 0.016, 10, 4, 0),
             (100.0, 1.0, 0.016, 10, 0, 0), (20.0, "shrink", 1e-5, 10, 4, "later"), (20.0, "shrink", 1e-6, 1, 4, -1)]


def _packed(net, flat_state_order):
    """Oracle-layout (state_dict order, no padding) vector -> the net's packed layout."""
    out = torch.zeros_like(net.flat, device="cpu")
    i = 0
    base = net.flat.data_ptr()
    for k, t in net.p.items():
        off = (t.data_ptr() - base) // 4
        out[off:off + t.numel()] = flat_state_order[i:i + t.numel()]
        i += t.numel()
    return out


def _unpacked(net, v):
    v, base = v.cpu(), net.flat.data_ptr()
    return torch.cat([v[(t.data_ptr() - base) // 4:(t.data_ptr() - base) // 4 + t.numel()] for t in net.p.values()])


def _padding_mask(net):
    m = torch.ones(net.flat.numel(), dtype=torch.bool)
    base = net.flat.data_ptr()
    for t in net.p.values():
        off = (t.data_ptr() - base) // 4
        m[off:off + t.numel()] = False
    return m


# ------------------------------------------------------------------ CPU ------------------------------------------------------------------
def test_logstd_curvature_matches_double_backprop():
    """The closed-form log_std block of F equals float64 double backprop of the reference's kl_divergence (macpo.py:153-166)."""
    import macpo_emulator
    for x_coef, y_coef in ((1.0, 0.5), (2.0, 0.3)):
        ls = torch.linspace(-6, 6, 25, dtype=torch.float64)
        want = []
        for l0 in ls:
            lp = l0.clone().requires_grad_(True)
            std = torch.sigmoid(lp / x_coef) * y_coef
            std_old = (torch.sigmoid(l0 / x_coef) * y_coef).detach()
            kl = torch.log(std_old) - torch.log(std) + (std_old ** 2 + 0.0) / (1e-8 + 2.0 * std ** 2) - 0.5
            (d1,) = torch.autograd.grad(kl, lp, create_graph=True)
            (d2,) = torch.autograd.grad(d1, lp)
            want.append(d2)
        got = macpo_emulator.logstd_curvature(ls, x_coef, y_coef)
        assert torch.allclose(got, torch.stack(want), rtol=1e-12, atol=0), (got, want)


@pytest.mark.parametrize("scenario", range(len(SCENARIOS)))
def test_trpo_update_host_path_vs_oracle(monkeypatch, scenario):
    """MACPOTrainer's host orchestration (emulated C-ABI) takes the oracle's case and accepted trial and ends at its weights."""
    import macpo_emulator
    macpo_emulator.install(monkeypatch)
    threads = torch.get_num_threads()
    torch.set_num_threads(1)
    try:
        su = Setup(48, 10, 14, 3, 128, "cpu")
        aver, cs, tkl, steps, case, acc = SCENARIOS[scenario]
        su.set_search(tkl, steps)
        before = su.nets.actor.flat.clone()
        s = su.sample(aver, cs)
        want, got = su.otr.trpo_update(s), su.tr.trpo_update(s)
    finally:
        torch.set_num_threads(threads)
    assert (got["optim_case"], got["accepted"]) == (want["optim_case"], want["accepted"]) and want["optim_case"] == case
    assert (want["accepted"] >= 1) if acc == "later" else want["accepted"] == acc
    for k in ("q", "r", "s", "lam", "nu"):
        assert float(got[k]) == pytest.approx(float(want[k]), rel=1e-4, abs=1e-7), k
    if want["accepted"] < 0:
        assert torch.equal(su.nets.actor.flat, before)
    # critics: 5 % of an Adam step (the rule of test_ma_ppo_update_vs_oracle: gradients below opti_eps amplify reordering noise)
    for net, onet, tol in ((su.nets.actor, su.oa, 1e-6), (su.nets.critic, su.oc, 0.05 * su.cfg["critic_lr"]), (su.nets.cost_critic, su.ok, 0.05 * su.cfg["critic_lr"])):
        for k, p in onet.p.items():
            assert float((net.p[k] - p.detach()).abs().max()) < tol, k


def test_oracle_reproduces_reference_macpo_bit_for_bit(golden):
    """tests/macpo_oracle.py against tests/golden/macpo.pt -- seven consecutive trpo_update calls of the reference's own
    MACPO_Trainer (tests/golden/make_macpo_golden.py): cases 1, 2, 3, 4 and 0, an acceptance at trial 4 and a reverted search.
    Every recorded intermediate, the case, the accepted trial, the returned scalars, PopArt and all weights: bit for bit."""
    import macpo_oracle as MO
    c = golden("macpo")["macpo"]
    threads = torch.get_num_threads()
    torch.set_num_threads(1)            # as the generator: LayerNorm's backward reductions depend on the thread count
    try:
        nets = [MA.OracleMANet(c["init"][n], layer_N=c["cfg"]["layer_N"]) for n in ("actor", "critic", "cost_critic")]
        cfg = dict(c["cfg"])
        otr = MO.OracleMACPOTrainer(*nets, cfg)
        seen = []
        for i, call in enumerate(c["calls"]):
            cfg["target_kl"], cfg["searching_steps"] = call["target_kl"], call["searching_steps"]
            w = otr.trpo_update(call["sample"])
            seen.append((w["optim_case"], w["accepted"]))
            assert (w["optim_case"], w["accepted"]) == (call["optim_case"], call["accepted"]), (i, seen[-1])
            for k, wk in (("g", "g"), ("b", "b"), ("xg", "xg"), ("xb", "xb"), ("q", "q"), ("x", "x_final"), ("lam", "lam"), ("nu", "nu")):
                assert torch.equal(torch.as_tensor(w[wk]).float(), torch.as_tensor(call[k]).float()), (i, k)
            if call["optim_case"] != 4:
                for k in ("r", "s"):
                    assert torch.equal(w[k], call[k]), (i, k)
            for k, v in call["out"].items():
                assert torch.equal(torch.as_tensor(w[k]), torch.as_tensor(v)), (i, k, w[k], v)
            for got_s, want_s in zip((otr.popart.running_mean, otr.popart.running_mean_sq, otr.popart.debiasing_term), call["popart"]):
                assert torch.equal(got_s, want_s), i
            for net, n in zip(nets, ("actor", "critic", "cost_critic")):
                for k, v in call["state"][n].items():
                    assert torch.equal(net.p[k].detach(), v), (i, n, k)
    finally:
        torch.set_num_threads(threads)
    assert {x[0] for x in seen} == {0, 1, 2, 3, 4} and -1 in {x[1] for x in seen} and max(x[1] for x in seen) >= 1


def test_macpo_fixture_regenerates_identically(tmp_path):
    """make_macpo_golden.py writes the committed macpo.pt byte for byte (only where the reference is checked out)."""
    gen = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "make_macpo_golden.py")
    sys.path.insert(0, os.path.dirname(gen))
    import make_golden
    if not os.path.isdir(make_golden.REF):
        pytest.skip("the reference checkout is not present")
    out = tmp_path / "macpo.pt"
    r = subprocess.run([sys.executable, gen, str(out)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    with open(out, "rb") as f1, open(os.path.join(os.path.dirname(gen), "macpo.pt"), "rb") as f2:
        assert f1.read() == f2.read()


def test_macpo_runner_reuses_mappolag_runner():
    from safepo.common.ma_model import MACPOTrainer, MultiAgentTrainer
    from safepo.multi_agent import macpo, mappolag
    assert mappolag.Runner.trainer_class is MultiAgentTrainer and macpo.Runner.trainer_class is MACPOTrainer
    assert macpo.DEFAULT_CONFIG["target_kl"] == 0.016 and macpo.DEFAULT_CONFIG["searching_steps"] == 10


# ------------------------------------------------------------------ GPU ------------------------------------------------------------------
def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs CUDA")
    return torch.device("cuda:0")


@pytest.mark.gpu
@pytest.mark.parametrize("N,D,A,H", SHAPES)
def test_fvp_gradients_cg_and_linesearch_eval_vs_oracle(N, D, A, H):
    """Layer tangents vs torch.func.jvp in float64; FVP vs the oracle's double backprop; g / b vs autograd; the CG residual; the
    line-search scalars."""
    from safepo import _lib as L
    from safepo.common.ma_model import _tangent_views
    dev = _cuda()
    su = Setup(N, D, D, A, H, dev, seed=N + D)
    tr, net, otr = su.tr, su.nets.actor, su.otr
    obs_d = su.obs.to(dev).contiguous()
    mean_old = tr.actor_forward(obs_d)
    ws = tr._fws
    g = torch.Generator().manual_seed(7)
    mask = _padding_mask(net)
    v = torch.randn(net.flat.numel(), generator=g) * 0.1
    v[mask] = 0
    vd = v.to(dev)

    # ---- layer tangents (float64 torch.func.jvp of the oracle's block) ----
    st = {k: p.detach().double() for k, p in su.oa.p.items()}
    tv = {k: t.double().cpu() for k, t in _tangent_views(net, v.clone()).items()}
    x64 = su.obs.double()
    import torch.nn.functional as F

    def block(i, x, p):
        if i == 0:
            x = F.layer_norm(x, (x.shape[-1],), p["base.feature_norm.weight"], p["base.feature_norm.bias"])
        w, b, lw, lb = net.blocks[i]
        return F.layer_norm(F.elu(F.linear(x, p[w], p[b])), (p[w].shape[0],), p[lw], p[lb])
    names0 = ["base.feature_norm.weight", "base.feature_norm.bias"]
    din = None
    worst_layer = 0.0
    for i in range(3):
        keys = list(net.blocks[i]) + (names0 if i == 0 else [])
        xin = x64 if i == 0 else ws["out"][i - 1].double().cpu()

        def fn(xx, *ps):
            p = dict(st, **dict(zip(keys, ps)))
            return block(i, xx, p)
        tin = torch.zeros_like(x64) if i == 0 else din
        _, want = torch.func.jvp(fn, (xin, *[st[k] for k in keys]), (tin, *[tv[k] for k in keys]))
        a, _b = tr._tangent_bufs(N, H)
        tvd = _tangent_views(net, vd)
        p = net.p
        w, bb, lw, lb = net.blocks[i]
        if i == 0:
            args = (L.ptr(obs_d), None, N, D)
            lin = (L.ptr(p[names0[0]]), L.ptr(p[names0[1]]), L.ptr(tvd[names0[0]]), L.ptr(tvd[names0[1]]))
        else:
            din_d = din.float().to(dev).contiguous()
            args = (L.ptr(ws["out"][i - 1]), L.ptr(din_d), N, H)
            lin = (None, None, None, None)
        L.check(L.lib().spo_ma_mlp_layer_jvp(*args, L.ptr(p[w]), L.ptr(tvd[w]), L.ptr(tvd[bb]), L.ptr(ws["pre"][i]), L.ptr(p[lw]),
                                              L.ptr(tvd[lw]), L.ptr(tvd[lb]), H, *lin, L.ptr(a), L.stream()), "spo_ma_mlp_layer_jvp")
        got = a.double().cpu()
        err = float((got - want).abs().max() / want.abs().max())
        worst_layer = max(worst_layer, err)
        assert err < 1e-4, (i, err)
        din = want

    # ---- FVP ----
    out = torch.empty_like(vd)
    tr.fvp(vd, out)
    out2 = torch.empty_like(vd)
    tr.fvp(2 * vd, out2)
    torch.cuda.synchronize()
    want = otr.fisher_vector_product(su.obs, su.actions, _unpacked(net, v))
    got = _unpacked(net, out)
    fvp_err = float((got - want).norm() / want.norm())
    assert fvp_err <= 1e-4, fvp_err
    # the A log_std entries (the closed-form block of spo_ma_fvp_finalize) are too few to register in the norm above: on their own
    ls_off = tr._ls_off
    ls_got = out[ls_off:ls_off + A].cpu()
    ls_want = _packed(net, want)[ls_off:ls_off + A]
    ls_err = float((ls_got - ls_want).abs().max() / ls_want.abs().max())
    assert ls_err <= 1e-4, (ls_got, ls_want)
    assert float((out2 - 2 * out).norm() / (2 * out).norm()) < 1e-6
    assert torch.count_nonzero(out.cpu()[mask]) == 0 and torch.count_nonzero(out2.cpu()[mask]) == 0

    # ---- g and b ----
    s = su.sample(30.0)
    dd = {k: torch.as_tensor(t, dtype=torch.float32).to(dev).contiguous() for k, t in s.items()}
    lp = MA.ma_actor_dist(su.oa, su.obs).log_prob(su.actions)
    ratio = torch.prod(torch.exp(lp - s["old_action_log_probs"]), dim=-1, keepdim=True)
    loss_r = -torch.sum(ratio * s["factor"] * s["adv_targ"], dim=-1, keepdim=True).mean()
    loss_c = torch.sum(ratio * s["factor"] * s["cost_adv_targ"], dim=-1, keepdim=True).mean()
    gw = torch.autograd.grad(loss_r, su.oa.params(), retain_graph=True)
    bw = torch.autograd.grad(loss_c, su.oa.params())
    lbuf = torch.zeros(32, device=dev)
    worst_g = 0.0
    for sign, adv, wantg, wl in ((-1.0, dd["adv_targ"].reshape(-1), gw, loss_r), (1.0, dd["cost_adv_targ"].reshape(-1), bw, loss_c)):
        gv = torch.zeros_like(net.flat)
        tr.surrogate_grad(mean_old, dd["actions"], dd["old_action_log_probs"], adv, dd["factor"].reshape(-1), sign, lbuf, gv)
        torch.cuda.synchronize()
        views = _tangent_views(net, gv.cpu())
        for (k, _), wg in zip(su.oa.p.items(), wantg):
            scale = float(wg.abs().max())
            e = float((views[k] - wg).abs().max())
            worst_g = max(worst_g, e / (scale + 1e-12))
            assert e <= 5e-5 * scale + 1e-9, (sign, k, e, scale)
        assert abs(float(lbuf[0]) - float(wl)) <= 2e-5 * float((ratio * s["factor"]).abs().mean()) + 1e-9
        assert torch.count_nonzero(gv.cpu()[mask]) == 0

    # ---- CG on b ----
    bvec = gv.clone()
    x = torch.zeros_like(bvec)
    tr.conjugate_gradient(bvec, x)
    torch.cuda.synchronize()
    b_o = _unpacked(net, bvec)
    xo, _ = otr.conjugate_gradient(su.obs, su.actions, b_o, tr.cfg["conjugate_gradient_iters"])
    res_dev = float((otr.fisher_vector_product(su.obs, su.actions, _unpacked(net, x)) - b_o).norm())
    res_or = float((otr.fisher_vector_product(su.obs, su.actions, xo) - b_o).norm())
    assert res_dev <= 1.5 * res_or + 1e-6, (res_dev, res_or)
    assert torch.count_nonzero(x.cpu()[mask]) == 0

    # ---- line-search evaluation at perturbed weights ----
    old_flat = net.flat.clone()
    tr.old_flat.copy_(old_flat)
    step = torch.randn(net.flat.numel(), generator=g) * 1e-3
    step[mask] = 0
    net.flat.add_(step.to(dev))
    res = torch.zeros(8, device=dev)
    tr.linesearch_eval(obs_d, mean_old, dd["actions"], dd["old_action_log_probs"], dd["adv_targ"].reshape(-1), dd["cost_adv_targ"].reshape(-1),
                       dd["factor"].reshape(-1), res)
    torch.cuda.synchronize()
    old_net = MA.OracleMANet(su.oa.state())
    with torch.no_grad():
        otr.update_model(su.oa, otr.flat_params() + _unpacked(net, step.to(dev)))
        lp = MA.ma_actor_dist(su.oa, su.obs).log_prob(su.actions)
        ratio = torch.prod(torch.exp(lp - s["old_action_log_probs"]), dim=-1, keepdim=True)
        terms = (ratio * s["factor"] * s["adv_targ"], ratio * s["factor"] * s["cost_adv_targ"], otr.kl_divergence(su.obs, su.actions, su.oa, old_net))
        want3 = (-terms[0].mean(), terms[1].mean(), terms[2].mean())
    # the means cancel (advantages of both signs; KL terms of size ~1/2 per dimension): 2e-5 relative to the size of the summed terms
    for i, w in enumerate(want3):
        scale = max(abs(float(w)), float(terms[i].abs().mean()), 0.05 * A if i == 2 else 0.0)
        assert abs(float(res[i]) - float(w)) <= 2e-5 * scale + 1e-9, (i, float(res[i]), float(w), scale)
    net.flat.copy_(old_flat)
    print(f"\nMACPO N={N} D={D} A={A} H={H}: layer tangent {worst_layer:.2e}, FVP {fvp_err:.2e} (log_std block {ls_err:.2e}), g/b {worst_g:.2e}, "
          f"CG residual {res_dev:.3e} (oracle {res_or:.3e}), line search {[float(res[i]) for i in range(3)]}")


@pytest.mark.gpu
@pytest.mark.parametrize("N,D,A,H", SHAPES)
def test_trpo_update_vs_oracle(N, D, A, H):
    """Consecutive trpo_update calls through the device kernels against the oracle, one per scenario: the expected case (0-4)
    and accepted trial of each, including a search that accepts at a later trial and one that accepts nothing, after which the
    actor must be bit-identical to the one before."""
    dev = _cuda()
    su = Setup(N, D, D, A, H, dev, seed=3 * N + D)
    for aver, cs, tkl, steps, case, acc in SCENARIOS:
        su.set_search(tkl, steps)
        s = su.sample(aver, cs)
        before = su.nets.actor.flat.clone()
        o_before = su.otr.flat_params().clone()
        want, got = su.otr.trpo_update(s), su.tr.trpo_update(s)
        torch.cuda.synchronize()
        tag = (N, aver, cs, tkl, steps)
        assert (got["optim_case"], got["accepted"]) == (want["optim_case"], want["accepted"]), (tag, got["optim_case"], got["accepted"],
                                                                                              want["optim_case"], want["accepted"])
        assert want["optim_case"] == case, (tag, want["optim_case"])
        assert (want["accepted"] >= 1) if acc == "later" else want["accepted"] == acc, (tag, want["accepted"])
        for k in ("q", "r", "s", "lam", "nu"):
            assert float(got[k]) == pytest.approx(float(want[k]), rel=1e-4, abs=1e-7), (tag, k, float(got[k]), float(want[k]))
        if want["accepted"] < 0:
            assert torch.equal(su.nets.actor.flat, before), tag
        step = float((su.otr.flat_params() - o_before).abs().max())
        err = max(float((su.nets.actor.p[k].cpu() - p.detach()).abs().max()) for k, p in su.oa.p.items())
        assert err <= 1e-4 * max(step, 1e-12) + 1e-6, (tag, err, step)
        for net, onet in ((su.nets.critic, su.oc), (su.nets.cost_critic, su.ok)):
            for k, p in onet.p.items():
                e = float((net.p[k].cpu() - p.detach()).abs().max())
                assert e < 0.05 * su.cfg["critic_lr"] + 1e-6, (tag, k, e)
        print(f"\nMACPO trpo_update N={N}: case {got['optim_case']} trial {got['accepted']} actor err {err:.2e} (step {step:.2e}) "
              f"q {float(got['q']):.6g}/{float(want['q']):.6g}")
        # re-synchronise the actors so that the next scenario starts from the same weights on both sides
        with torch.no_grad():
            su.otr.update_model(su.oa, _unpacked(su.nets.actor, su.nets.actor.flat))


@pytest.mark.gpu
def test_macpo_cli_synthetic(tmp_path):
    _cuda()
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    pkg = os.path.join(root, "safe-policy-optimization_b200")
    code = ("import sys, math; from safepo.multi_agent import macpo; rows = macpo.main(sys.argv[1:]); "
            "assert rows and all(math.isfinite(v) for r in rows for v in r.values() if isinstance(v, float)), rows; print(rows[-1])")
    r = subprocess.run([sys.executable, "-c", code, "--env", "synthetic", "--iterations", "2", "--num-envs", "64", "--hidden-size", "128",
                        "--log-dir", str(tmp_path)], cwd=pkg, capture_output=True, text=True, env=dict(os.environ, PYTHONPATH=pkg))
    assert r.returncode == 0, r.stdout + r.stderr
    print(r.stdout[-2000:])


def _runner_iteration(device):
    """Two iterations of safepo/multi_agent/macpo.py's Runner (two agents) against tests/macpo_oracle.py's OracleMACPORunner on a
    synthetic stream with the same injected eps, agent order and row orders: buffers after compute(), and after train() each
    agent's case and accepted trial, the cross-agent factor and all weights."""
    import macpo_oracle as MO
    from safepo.common.ma_model import MultiAgentNets
    from safepo.multi_agent.macpo import DEFAULT_CONFIG, Runner
    T, N, D, DS, A, H, NA = 4, 16, 10, 14, 3, 128, 2
    cfg = dict(DEFAULT_CONFIG, episode_length=T, n_rollout_threads=N, hidden_size=H)
    g = torch.Generator().manual_seed(31)
    init = [(_state(g, D, H, A, "actor"), _state(g, DS, H, A, "critic"), _state(g, DS, H, A, "critic")) for _ in range(NA)]
    onets = [tuple(MA.OracleMANet(st) for st in sts) for sts in init]
    orun = MO.OracleMACPORunner(onets, cfg, T, N, D, DS, A)
    nets = [MultiAgentNets(*sts, device, layer_N=2) for sts in init]
    run = Runner(nets, cfg, D, DS, A)
    obs0, share0 = torch.randn(N, NA, D, generator=g) * 2 + 0.5, torch.randn(N, NA, DS, generator=g) * 3
    orun.warmup(obs0, share0)
    run.warmup(obs0, share0)

    def near(a, b, tol):
        return float((a.cpu() - b).abs().max()) <= tol * (1.0 + float(b.abs().max()))
    seen = []
    for it in range(2):
        for step in range(T):
            eps = [torch.randn(N, A, generator=g) for _ in range(NA)]
            ov, oact, olp, ocp = orun.collect(step, eps=eps)
            v, act, lp, cp = run.collect(step, eps=eps)
            assert near(v, ov, 5e-5) and all(near(act[a], oact[a], 5e-5) for a in range(NA)), (it, step)
            obs, share = torch.randn(N, NA, D, generator=g) * 2 + 0.5, torch.randn(N, NA, DS, generator=g) * 3
            rew, cost = torch.randn(N, NA, 1, generator=g), (torch.rand(N, NA, 1, generator=g) < 0.3).float()
            dones = (torch.rand(N, generator=g) < 0.2)[:, None].expand(N, NA).clone()
            orun.insert(obs, share, rew, cost, dones, ov, oact, olp, ocp)
            run.insert(obs, share, rew, cost, dones, v, act, lp, cp)
        orun.compute()
        run.compute()
        for a in range(NA):
            for k in ("returns", "cost_returns"):
                assert near(getattr(run.buffer[a], k), getattr(orun.buffer[a], k), 5e-5), (it, a, k)
        order = torch.randperm(NA, generator=g)
        perms = [[torch.randperm(T * N, generator=g)] for _ in range(NA)]
        want = orun.train(agent_order=order, perms=perms)
        got = run.train(agent_order=order, perms=perms, collect_outputs=True)
        for a in range(NA):
            assert (got[a]["optim_case"], got[a]["accepted"]) == (want[a]["optim_case"], want[a]["accepted"]), (it, a)
            seen.append((want[a]["optim_case"], want[a]["accepted"]))
            assert near(run.buffer[a].factor, orun.buffer[a].factor, 1e-4), (it, a)
            for net, onet, tol in zip((nets[a].actor, nets[a].critic, nets[a].cost_critic), onets[a], (1e-5, 0.05 * cfg["critic_lr"], 0.05 * cfg["critic_lr"])):
                for k, pt in onet.p.items():
                    assert float((net.p[k].cpu() - pt.detach()).abs().max()) < tol, (it, a, k)
            row = run.log_agent(a, got[a])
            # the KL is a mean of per-dimension terms of size ~1/2 that cancel: the line-search rule, 2e-5 of 0.05 A
            assert row[f"Misc/KL/agent{a}"] == pytest.approx(float(want[a]["kl"]), rel=1e-3, abs=1e-6 * A)
            assert row[f"Misc/Entropy/agent{a}"] == pytest.approx(float(want[a]["dist_entropy"]), rel=1e-5)
        if it == 0:                                   # finished episodes above the limit for the second iteration
            run.return_aver_cost(torch.tensor(31.5))
            for b in orun.buffer:
                b.aver_episode_costs = torch.tensor(31.5)
    assert any(bool((run.buffer[a].factor != 1).any()) for a in range(NA))
    return seen


def test_runner_iteration_host_path_vs_oracle(monkeypatch):
    """The MACPO Runner's host logic (emulated C-ABI) against the oracle's runner: two iterations of two agents."""
    import macpo_emulator
    macpo_emulator.install(monkeypatch)
    threads = torch.get_num_threads()
    torch.set_num_threads(1)
    try:
        print(_runner_iteration("cpu"))
    finally:
        torch.set_num_threads(threads)


@pytest.mark.gpu
def test_runner_iteration_vs_oracle():
    """The MACPO Runner on the device against the oracle's runner: two iterations of two agents."""
    print("\nMACPO runner (case, trial) per agent update:", _runner_iteration(_cuda()))
