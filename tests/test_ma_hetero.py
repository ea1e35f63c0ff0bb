"""Multi-agent runs whose agents differ in observation and action size, and MAPPO-Lag with its policy active masks.

CPU: tests/hetero_oracle.py replays the reference runners' own iterations of tests/golden/hetero.pt bit for bit (the 9|8
Humanoid's padded actions, the Freight-Franka per-agent observations; MAPPO-Lag with the mamujoco flags and HAPPO) and two
masked MAPPO_L_Trainer.ppo_update calls; the runners' host path through the emulated C-ABI against that oracle; padding,
trimming and the list observations; the refusal of a bad agent and of a checkpoint of another agent's shape; the CLI's
per-agent flags.
GPU: two runner iterations of each algorithm with heterogeneous agents against the oracle, MultiAgentTrainer.ppo_update with
the policy masks at config 5's layers and at the MAMuJoCo shape, save -> restore -> eval, and the four CLIs."""
import importlib
import math
import os
import subprocess
import sys

import pytest
import torch

import hetero_oracle as HO
from oracle import ma_oracle as MA
from oracle import ppo_oracle as PO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "safe-policy-optimization_b200")
CASES = {"humanoid": dict(obs=(10, 10), act=(9, 8), pad=9, obs_list=False), "franka": dict(obs=(10, 14), act=(4, 3), pad=None, obs_list=True)}
ALGOS = ("mappolag", "macpo", "mappo", "happo")
TWO_NET = {"mappo": PO.OracleMAPPOTrainer, "happo": PO.OracleHAPPOTrainer}
MASKS = dict(use_policy_active_masks=True, use_value_active_masks=True, entropy_coef=0.01)


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs CUDA")
    return torch.device("cuda:0")


def _single_thread():
    threads = torch.get_num_threads()
    torch.set_num_threads(1)        # the fixture was written with one intra-op thread (LayerNorm's backward reductions)
    return threads


# ============================================================ CPU: the fixture ============================================================
def _oracle_runner(algo, cfg, T, N, obs_dims, DS, act_dims, pad, nets):
    if algo == "mappolag":
        return HO.OracleHeteroMARunner(nets, cfg, T, N, obs_dims, DS, act_dims, pad)
    if algo == "macpo":
        return HO.OracleHeteroMACPORunner(nets, cfg, T, N, obs_dims, DS, act_dims, pad)
    return HO.OracleHeteroTwoNetRunner(nets, cfg, T, N, obs_dims, DS, act_dims, TWO_NET[algo], pad)


@pytest.mark.parametrize("algo", ["mappolag", "happo"])
@pytest.mark.parametrize("case", list(CASES))
def test_oracle_replays_reference_runs_bit_for_bit(golden, algo, case):
    """The oracle runners replay the reference Runner's two iterations of hetero.pt exactly: the actions as the environment gets
    them (the 9|8 case's zero column included), log-probs, values, the buffers after compute() (trimmed actions, per-agent
    observations), and after train() the factor, lamda_lagr, the PopArt state and every state dict."""
    fx = golden("hetero")["runs"][(algo, case)]
    T, N, DS, H, NA = fx["dims"]
    cfg, lag = dict(fx["cfg"]), algo == "mappolag"
    names = ("actor", "critic", "cost_critic") if lag else ("actor", "critic")
    threads = _single_thread()
    try:
        init = HO.initial_states(fx["init_seed"], fx["obs_dims"], DS, fx["act_dims"], H, cfg["layer_N"], lag)
        nets = [tuple(MA.OracleMANet(s, cfg["layer_N"]) for s in sts) for sts in init]
        orun = _oracle_runner(algo, cfg, T, N, fx["obs_dims"], DS, fx["act_dims"], fx["pad"], nets)
        orun.warmup(fx["obs0"], fx["share_obs0"])
        torch.manual_seed(fx["seed"])
        for it, (steps, want_it) in enumerate(zip(fx["stream"], fx["iters"])):
            for step, st in enumerate(steps):
                out = orun.collect(step)
                values, actions, logps = out[:3]
                assert HO.digest(values) == st["values"], (it, step)
                assert HO.digests(actions) == st["actions"], (it, step)
                assert HO.digests(logps) == st["action_log_probs"], (it, step)
                if fx["pad"] is not None:
                    assert bool((actions[1][:, 8] == 0).all())
                if lag:
                    assert HO.digest(out[3]) == st["cost_preds"]
                    orun.insert(st["obs"], st["share_obs"], st["rewards"], st["costs"], st["dones"], values, actions, logps, out[3])
                else:
                    orun.insert(st["obs"], st["share_obs"], st["rewards"], st["dones"], values, actions, logps)
            orun.compute()
            for b, want in zip(orun.buffer, want_it["after_compute"]):
                for k, v in want.items():
                    assert HO.digest(getattr(b, k)) == v, (it, k)
            orun.train()
            for a, want in enumerate(want_it["agents"]):
                tr = orun.trainer[a]
                assert HO.digest(orun.buffer[a].factor) == want["factor"], (it, a)
                if lag:
                    assert HO.digest(torch.as_tensor(tr.lamda_lagr).reshape(-1)) == want["lamda_lagr"], (it, a)
                pop = [x.reshape(-1) for x in (tr.popart.running_mean, tr.popart.running_mean_sq, tr.popart.debiasing_term)]
                assert HO.digests(pop) == want["popart"], (it, a)
                for net, name in zip(nets[a], names):
                    for k, v in want["state"][name].items():
                        assert HO.digest(net.p[k]) == v, (it, a, name, k)
            if it == 0 and lag:
                for b in orun.buffer:
                    b.aver_episode_costs = torch.tensor(fx["aver_cost_after_first"])
        assert any(bool((b.factor != 1).any()) for b in orun.buffer)
    finally:
        torch.set_num_threads(threads)


def test_oracle_masked_update_matches_reference_bit_for_bit(golden):
    """OracleMaskedMATrainer replays two masked MAPPO_L_Trainer.ppo_update calls of hetero.pt exactly (a quarter of the rows
    inactive): the eight returned values, lamda_lagr, the PopArt state and the three state dicts."""
    fx = golden("hetero")["masked_update"]
    threads = _single_thread()
    try:
        cfg = dict(fx["cfg"])
        D, DS, A, H, _ = fx["dims"]
        init = HO.initial_states(fx["init_seed"], [D], DS, [A], H, cfg["layer_N"], True)[0]
        nets = [MA.OracleMANet(s, cfg["layer_N"]) for s in init]
        tr = HO.OracleMaskedMATrainer(*nets, cfg)
        for call in fx["calls"]:
            out = tr.ppo_update(fx["sample"])
            for k, v in call["out"].items():
                assert HO.digest(out[k]) == v, k
            assert HO.digest(torch.as_tensor(tr.lamda_lagr).reshape(-1)) == call["lamda_lagr"]
            pop = [x.reshape(-1) for x in (tr.popart.running_mean, tr.popart.running_mean_sq, tr.popart.debiasing_term)]
            assert HO.digests(pop) == call["popart"]
            for net, name in zip(nets, ("actor", "critic", "cost_critic")):
                for k, v in call["state"][name].items():
                    assert HO.digest(net.p[k]) == v, (name, k)
        am = fx["sample"]["active_masks"]
        assert 0 < int((am == 0).sum()) < am.numel()
    finally:
        torch.set_num_threads(threads)


def test_hetero_fixture_regenerates_identically(tmp_path):
    """make_hetero_golden.py writes the committed hetero.pt byte for byte (only where the reference is checked out)."""
    gen = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "make_hetero_golden.py")
    sys.path.insert(0, os.path.dirname(gen))
    import make_golden
    if not os.path.isdir(make_golden.REF):
        pytest.skip("the reference checkout is not present")
    out = tmp_path / "hetero.pt"
    r = subprocess.run([sys.executable, gen, str(out)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    with open(out, "rb") as f1, open(os.path.join(os.path.dirname(gen), "hetero.pt"), "rb") as f2:
        assert f1.read() == f2.read()


# ============================================================ runner vs oracle (CPU host path / GPU) ============================================================
def _config(algo, T, N, H, layer_N=2):
    M = importlib.import_module(f"safepo.multi_agent.{algo}")
    cfg = dict(M.DEFAULT_CONFIG, episode_length=T, n_rollout_threads=N, hidden_size=H, learning_iters=2, layer_N=layer_N)
    if algo == "mappolag":                          # the yaml's mamujoco section at the test's sizes
        cfg.update({k: v for k, v in M.MAMUJOCO.items() if k not in ("episode_length", "n_rollout_threads", "n_eval_rollout_threads", "hidden_size")})
    elif algo != "macpo":
        cfg.update(MASKS)
    return M, cfg


def _build(algo, case, dev, T, N, DS, H, seed, layer_N=2):
    """The device runner and the oracle runner of two agents of the case's sizes from the same weights."""
    from safepo.common.ma_model import MultiAgentNets
    M, cfg = _config(algo, T, N, H, layer_N)
    c = CASES[case]
    cost = M.Runner.cost_critic
    g = torch.Generator().manual_seed(seed)
    states = [[HO.random_state(g, D, H, A, "actor", layer_N), HO.random_state(g, DS, H, 0, "critic", layer_N)] + ([HO.random_state(g, DS, H, 0, "critic", layer_N)] if cost else [])
              for D, A in zip(c["obs"], c["act"])]
    onets = [tuple(MA.OracleMANet(s, layer_N) for s in sts) for sts in states]
    orun = _oracle_runner(algo, cfg, T, N, c["obs"], DS, c["act"], c["pad"], onets)
    nets = [MultiAgentNets(*sts, *([] if cost else [None]), dev, layer_N=layer_N, std_x_coef=cfg["std_x_coef"], std_y_coef=cfg["std_y_coef"])
            for sts in states]
    run = M.Runner(nets, cfg, list(c["obs"]), DS, list(c["act"]), pad_actions_to=c["pad"])
    return cfg, orun, run, onets, g


def _obs(g, case, N, NA):
    c = CASES[case]
    if c["obs_list"]:
        return [torch.randn(N, d, generator=g) * 2 + 0.5 for d in c["obs"]]
    return torch.randn(N, NA, c["obs"][0], generator=g) * 2 + 0.5


def _to(x, dev):
    return [t.to(dev) for t in x] if isinstance(x, list) else x.to(dev)


def _iterations(algo, case, dev, T=4, N=16, DS=14, H=128, seed=7, layer_N=2):
    """Two runner iterations of two agents of the case's sizes, device runner against the oracle runner, with the same eps, agent
    order and row orders.  Every agent of env 1 finishes at step 2; for the algorithms whose advantages stay finite when an agent
    finishes alone (all but MAPPO-Lag, whose NaN standardisation is the reference's), agent 1 of env 0 also finishes alone at step
    1.  The device runner stores its own actions (equal to the oracle's within fp32 noise, checked), padded for the environment
    where the case pads.  Returns the runners and both sides' outputs per iteration."""
    NA, c = 2, CASES[case]
    cfg, orun, run, onets, g = _build(algo, case, dev, T, N, DS, H, seed, layer_N)
    lag = run.cost_critic
    obs0, share0 = _obs(g, case, N, NA), torch.randn(N, NA, DS, generator=g) * 3
    orun.warmup(obs0, share0)
    run.warmup(_to(obs0, dev), share0.to(dev))
    outs = []
    for it in range(2):
        for step in range(T):
            eps = [torch.randn(N, A, generator=g) for A in c["act"]]
            o = orun.collect(step, eps)
            v, act, lp, cp = run.collect(step, [e.to(dev) for e in eps])
            env_act = run.env_actions(act)
            for a in range(NA):
                assert act[a].shape == (N, c["act"][a])
                assert env_act[a].shape == o[1][a].shape
                assert float((env_act[a].cpu() - o[1][a]).abs().max()) < 1e-4, (it, step, a)
                if c["pad"] is not None:
                    assert bool((env_act[a][:, c["act"][a]:] == 0).all())
            obs, share = _obs(g, case, N, NA), torch.randn(N, NA, DS, generator=g) * 3
            rew, cost = torch.randn(N, NA, 1, generator=g), (torch.rand(N, NA, 1, generator=g) < 0.3).float()
            dones = torch.zeros(N, NA, dtype=torch.bool)
            if step == 2:
                dones[1, :] = True
            if step == 1 and algo != "mappolag":
                dones[0, 1] = True
            if lag:
                orun.insert(obs, share, rew, cost, dones, *o)
            else:
                orun.insert(obs, share, rew, dones, *o)
            run.insert(_to(obs, dev), share.to(dev), rew.to(dev), cost.to(dev), dones.to(dev), v, env_act, lp, cp)
        orun.compute()
        run.compute()
        for a in range(NA):
            assert run.buffer[a].actions.shape[-1] == c["act"][a] and run.buffer[a].obs.shape[-1] == c["obs"][a]
        order = torch.randperm(NA, generator=g).tolist()
        iters = 1 if algo == "macpo" else cfg["learning_iters"]
        perms = [[torch.randperm(T * N, generator=g) for _ in range(iters)] for _ in range(NA)]
        want = orun.train(order, perms)
        got = run.train(order, [[p.to(dev) for p in ps] for ps in perms], collect_outputs=True)
        outs.append((got, want))
        if it == 0 and lag:
            run.return_aver_cost(torch.tensor(31.5))
            for b in orun.buffer:
                b.aver_episode_costs = torch.tensor(31.5)
    return cfg, orun, run, onets, outs


_NAMES = {"mappolag": ("value_loss", "critic_grad_norm", "policy_loss", "dist_entropy", "actor_grad_norm", "imp_weights", "cost_loss",
                       "cost_grad_norm"),
          "mappo": ("value_loss", "critic_grad_norm", "policy_loss", "dist_entropy", "actor_grad_norm", "imp_weights"),
          "happo": ("value_loss", "critic_grad_norm", "policy_loss", "dist_entropy", "actor_grad_norm", "imp_weights")}


def _check_iterations(algo, cfg, orun, run, onets, outs, rtol, lr_frac):
    """The runner tests' bars: returned values within rtol of the largest |value| (+1e-5) (MAPPO-Lag, whose oracle runner returns
    nothing: lamda_lagr and the PopArt state), MACPO's case and accepted trial, the factor, and every weight within lr_frac learning
    rates of the oracle's (a wrong gradient sign would be 2 lr per update; MACPO's actor within 1e-5)."""
    for got, want in outs:
        for a in got:
            if algo == "macpo":
                assert (got[a]["optim_case"], got[a]["accepted"]) == (want[a]["optim_case"], want[a]["accepted"]), a
            elif algo != "mappolag":
                for gv, k in zip(got[a], _NAMES[algo]):
                    wv = want[a][k].reshape(-1).double()
                    err = float((gv.detach().cpu().reshape(-1).double() - wv).abs().max())
                    assert err <= rtol * float(wv.abs().max()) + 1e-5, (a, k, err)
    for a in range(run.num_agents):
        f_got, f_want = run.buffer[a].factor.cpu(), orun.buffer[a].factor
        assert float((f_got - f_want).abs().max()) <= 1e-3 * (1 + float(f_want.abs().max())), a
        pop = orun.trainer[a].popart
        for got_s, want_s in zip(run.trainer[a].popart_state.cpu(), (pop.running_mean, pop.running_mean_sq, pop.debiasing_term)):
            assert abs(float(got_s) - float(want_s)) <= 1e-4 * abs(float(want_s)) + 1e-12, a
        if algo == "mappolag":
            assert abs(float(run.trainer[a].lamda_lagr) - float(orun.trainer[a].lamda_lagr)) < 1e-5, a
        lrs = (cfg["actor_lr"], cfg["critic_lr"], cfg["critic_lr"])
        for i, (net, onet, lr) in enumerate(zip((run.nets[a].actor, run.nets[a].critic, run.nets[a].cost_critic), onets[a], lrs)):
            tol = (1e-5 if algo == "macpo" and i == 0 else lr_frac * lr) + 2e-6
            for k, pt in onet.p.items():
                err = float((net.p[k].cpu() - pt.detach()).abs().max())
                assert err < tol, (a, k, err, tol)


def _emulate(monkeypatch, algo):
    import ppo_emulator
    if algo == "macpo":
        import macpo_emulator
        return macpo_emulator.install(monkeypatch)
    return ppo_emulator.install(monkeypatch)


@pytest.mark.parametrize("algo", ALGOS)
@pytest.mark.parametrize("case", list(CASES))
def test_runner_host_path_through_emulated_abi_vs_oracle(monkeypatch, algo, case):
    """Two iterations of each runner with agents of different sizes through the emulated C-ABI against the oracle runner:
    padding for the environment and trimming on insert, per-agent observations, per-agent buffers, the cross-agent factor
    across agents of different act_dim, masks on where the algorithm has them."""
    _emulate(monkeypatch, algo)
    threads = _single_thread()
    try:
        cfg, orun, run, onets, outs = _iterations(algo, case, "cpu", N=6, H=128 if algo == "macpo" else 32,   # MACPO's emulation checks H
                                                  layer_N=1 if algo == "macpo" else 2)
        _check_iterations(algo, cfg, orun, run, onets, outs, rtol=1e-3, lr_frac=0.2)
    finally:
        torch.set_num_threads(threads)


# ============================================================ CPU: conventions, refusals, CLI ============================================================
def _nets_for(dev, obs_dims, DS, act_dims, H=32, cost=True, seed=3):
    from safepo.common.ma_model import MultiAgentNets
    g = torch.Generator().manual_seed(seed)
    return [MultiAgentNets(HO.random_state(g, D, H, A, "actor", 2), HO.random_state(g, DS, H, 0, "critic", 2), HO.random_state(g, DS, H, 0, "critic", 2) if cost else None, dev)
            for D, A in zip(obs_dims, act_dims)]


def test_padding_trimming_and_list_observations(monkeypatch):
    """env_actions pads with exact zero columns only with pad_actions_to; insert cuts padded actions back and reads either
    observation convention; warmup takes the list form."""
    import ma_emulator
    from safepo.multi_agent.mappolag import DEFAULT_CONFIG, Runner
    ma_emulator.install(monkeypatch)
    T, N, DS = 3, 5, 6
    cfg = dict(DEFAULT_CONFIG, episode_length=T, n_rollout_threads=N, hidden_size=32)
    run = Runner(_nets_for("cpu", (4, 8), DS, (9, 8)), cfg, [4, 8], DS, [9, 8], pad_actions_to=9)
    acts = [torch.randn(N, 9), torch.randn(N, 8)]
    env = run.env_actions(acts)
    assert env[0] is acts[0] and env[1].shape == (N, 9) and torch.equal(env[1][:, :8], acts[1]) and bool((env[1][:, 8] == 0).all())
    assert Runner(_nets_for("cpu", (4, 8), DS, (9, 8)), cfg, [4, 8], DS, [9, 8]).env_actions(acts) is acts
    obs = [torch.randn(N, 4), torch.randn(N, 8)]
    run.warmup(obs, torch.randn(N, 2, DS))
    assert torch.equal(run.buffer[0].obs[0], obs[0]) and torch.equal(run.buffer[1].obs[0], obs[1])
    obs = [torch.randn(N, 4), torch.randn(N, 8)]
    z = torch.zeros(N, 2, 1)
    run.insert(obs, torch.randn(N, 2, DS), z, z, torch.zeros(N, 2, dtype=torch.bool), z, env, [torch.zeros(N, 9), torch.zeros(N, 8)], z)
    assert torch.equal(run.buffer[1].actions[0], acts[1]) and torch.equal(run.buffer[1].obs[1], obs[1])
    with pytest.raises(Exception):
        run.warmup([torch.randn(N, 4)], torch.randn(N, 2, DS))


def test_synthetic_env_per_agent_sizes():
    """Equal per-agent sizes give the stacked form and the same draws as the int form; different observation sizes give one
    tensor per agent; step checks each agent's actions against its own width."""
    from safepo.common.synthetic_env import SyntheticMultiAgentEnv
    a = SyntheticMultiAgentEnv(4, 2, 6, 8, 3, 5, 11, "cpu", agent_done_prob=0.1)
    b = SyntheticMultiAgentEnv(4, 2, [6, 6], 8, [3, 3], 5, 11, "cpu", agent_done_prob=0.1)
    for x, y in zip(a.reset(), b.reset()):
        assert (x is None and y is None) or torch.equal(x, y)
    for _ in range(3):
        for x, y in zip(a.step([torch.zeros(4, 3)] * 2), b.step([torch.zeros(4, 3)] * 2)):
            assert (x is None and y is None) or torch.equal(x, y)
    h = SyntheticMultiAgentEnv(4, 2, [6, 10], 8, [9, 8], 5, 11, "cpu")
    obs, share, _ = h.reset()
    assert isinstance(obs, list) and [o.shape for o in obs] == [(4, 6), (4, 10)] and share.shape == (4, 2, 8)
    obs = h.step([torch.zeros(4, 9), torch.zeros(4, 8)])[0]
    assert [o.shape for o in obs] == [(4, 6), (4, 10)]
    with pytest.raises(ValueError):
        h.step([torch.zeros(4, 9), torch.zeros(4, 9)])
    with pytest.raises(ValueError):
        SyntheticMultiAgentEnv(4, 2, [6, 10, 12], 8, 3, 5, 11, "cpu")


def test_bad_agent_is_refused_before_any_launch(monkeypatch):
    """A per-agent size outside the kernels' limits, or one its nets do not have, raises SpoError naming the agent and the
    dimension when the runner is built, before anything is launched."""
    import ma_emulator
    from safepo._lib import SpoError
    from safepo.multi_agent.mappolag import DEFAULT_CONFIG, Runner
    lib = ma_emulator.install(monkeypatch)
    calls = []
    for name in dir(lib):
        if name.startswith("spo_ma") or name.startswith("spo_gae"):
            fn = getattr(lib, name)
            monkeypatch.setattr(lib, name, (lambda fn, name: (lambda *a: calls.append(name) or fn(*a)))(fn, name), raising=False)
    cfg = dict(DEFAULT_CONFIG, episode_length=2, n_rollout_threads=3, hidden_size=32)
    with pytest.raises(SpoError, match=r"agent 1: obs_dim=7 must be even"):
        Runner(_nets_for("cpu", (4, 7), 6, (3, 3)), cfg, [4, 7], 6, [3, 3])
    with pytest.raises(SpoError, match=r"agent 0: act_dim=33 must be in 1\.\.32"):
        Runner(_nets_for("cpu", (4, 4), 6, (33, 3)), cfg, [4, 4], 6, [33, 3])
    with pytest.raises(SpoError, match=r"agent 1: act_dim=8, but its actor has 9 actions"):
        Runner(_nets_for("cpu", (4, 4), 6, (9, 9)), cfg, [4, 4], 6, [9, 8])
    with pytest.raises(SpoError, match=r"agent 0: obs_dim=4, but its actor takes 10 inputs"):
        Runner(_nets_for("cpu", (10, 4), 6, (3, 3)), cfg, [4, 4], 6, 3)
    with pytest.raises(SpoError, match=r"agent 0: share_obs_dim=8, but its critic takes 6 inputs"):
        Runner(_nets_for("cpu", (4, 4), 6, (3, 3)), cfg, 4, 8, 3)
    with pytest.raises(SpoError, match=r"act_dim: 3 entries for 2 agents"):
        Runner(_nets_for("cpu", (4, 4), 6, (3, 3)), cfg, 4, 6, [3, 3, 3])
    with pytest.raises(SpoError, match=r"pad_actions_to=8 is narrower"):
        Runner(_nets_for("cpu", (4, 4), 6, (9, 8)), cfg, 4, 6, [9, 8], pad_actions_to=8)
    assert calls == []


def test_checkpoint_of_another_shape_is_refused(monkeypatch, tmp_path):
    """save -> restore of agents of different sizes keeps each agent's shapes; the same files restored into agents of swapped
    sizes raise SpoError naming the file and the key, and nothing is copied."""
    import ma_emulator
    from safepo._lib import SpoError
    from safepo.multi_agent.mappolag import DEFAULT_CONFIG, Runner
    ma_emulator.install(monkeypatch)
    cfg = dict(DEFAULT_CONFIG, episode_length=2, n_rollout_threads=3, hidden_size=32)
    src = Runner(_nets_for("cpu", (4, 8), 6, (9, 8), seed=1), cfg, [4, 8], 6, [9, 8], pad_actions_to=9)
    src.save(str(tmp_path), train_state=True)
    assert torch.load(tmp_path / "actor_agent1.pt")["act.action_out.fc_mean.weight"].shape == (8, 32)
    same = Runner(_nets_for("cpu", (4, 8), 6, (9, 8), seed=2), cfg, [4, 8], 6, [9, 8], pad_actions_to=9)
    same.restore(str(tmp_path), train_state=True)
    for a in range(2):
        assert torch.equal(same.nets[a].actor.flat, src.nets[a].actor.flat)
    swapped = Runner(_nets_for("cpu", (8, 4), 6, (8, 9), seed=2), cfg, [8, 4], 6, [8, 9], pad_actions_to=9)
    before = swapped.nets[0].actor.flat.clone()
    with pytest.raises(SpoError, match=r"actor_agent0\.pt: 'base\.feature_norm\.weight' has shape \(4,\), expected \(8,\)"):
        swapped.restore(str(tmp_path))
    assert torch.equal(swapped.nets[0].actor.flat, before)
    with pytest.raises(SpoError, match=r"train_state_agent0\.pt.*'obs' has shape \(3, 4\), expected \(3, 8\)"):
        swapped.buffer[0].load_carried_state(torch.load(tmp_path / "train_state_agent0.pt")["buffer"], str(tmp_path / "train_state_agent0.pt"))


def test_cli_per_agent_sizes_through_emulated_abi(monkeypatch, tmp_path):
    """--obs-dims / --act-dims / --pad-actions-to build agents of those sizes and train them on the synthetic environments (list
    observations, padded actions); a list of the wrong length is refused; --mamujoco applies MAPPO-Lag's mask flags."""
    import ppo_emulator
    from safepo.multi_agent import mappolag as M
    ppo_emulator.install(monkeypatch)
    built = []
    real_init = M.Runner.__init__

    def spy(self, *a, **k):
        real_init(self, *a, **k)
        built.append(self)
    monkeypatch.setattr(M.Runner, "__init__", spy)
    common = ["--num-envs", "6", "--share-obs-dim", "14", "--hidden-size", "32", "--episode-len", "3", "--device", "cpu", "--iterations", "1"]
    rows = M.main(common + ["--obs-dims", "10,14", "--act-dims", "9,8", "--pad-actions-to", "9", "--log-dir", str(tmp_path / "a")])
    run = built[-1]
    assert (run.obs_dims, run.act_dims, run.pad_actions_to) == ([10, 14], [9, 8], 9)
    assert [b.actions.shape[-1] for b in run.buffer] == [9, 8] and [b.obs.shape[-1] for b in run.buffer] == [10, 14]
    assert len(rows) == 1 and all(math.isfinite(rows[0][f"Loss/Loss_actor/agent{a}"]) for a in range(2))
    rows = M.main(common + ["--mamujoco", "--act-dims", "3,2", "--log-dir", str(tmp_path / "b")])
    run = built[-1]
    assert run.config["use_policy_active_masks"] and run.config["gamma"] == 0.99 and run.obs_dims == [398, 398] and run.act_dims == [3, 2]
    with pytest.raises(SystemExit):
        M.main(common + ["--obs-dims", "10,14,16", "--log-dir", str(tmp_path / "c")])


def test_macpo_mamujoco_section_builds_one_block_nets(monkeypatch, tmp_path):
    """MACPO's --mamujoco builds nets with layer_N 1 (fc1 and one fc2 block) of 128 and trains them (emulated C-ABI)."""
    import macpo_emulator
    from safepo.multi_agent import macpo as M
    macpo_emulator.install(monkeypatch)
    built = []
    real_init = M.Runner.__init__

    def spy(self, *a, **k):
        real_init(self, *a, **k)
        built.append(self)
    monkeypatch.setattr(M.Runner, "__init__", spy)
    rows = M.main(["--mamujoco", "--num-envs", "4", "--obs-dims", "10,14", "--act-dims", "3,2", "--share-obs-dim", "14", "--episode-len", "3",
                   "--device", "cpu", "--iterations", "1", "--log-dir", str(tmp_path)])
    run = built[-1]
    p = run.nets[0].actor.p
    assert run.nets[0].actor.layer_N == 1 and run.nets[0].actor.H == 128 and "base.mlp.fc2.0.0.weight" in p and "base.mlp.fc2.1.0.weight" not in p
    assert run.config["target_kl"] == 0.01 and run.T == 1000
    assert all(math.isfinite(rows[0][f"Misc/KL/agent{a}"]) for a in range(2))


# ============================================================ GPU ============================================================
@pytest.mark.gpu
@pytest.mark.parametrize("algo", ALGOS)
@pytest.mark.parametrize("case", list(CASES))
def test_runner_iterations_vs_oracle(algo, case):
    """Two iterations of each runner with heterogeneous agents on the device against the oracle runner, at the bars of the
    existing multi-agent runner tests (MAPPO-Lag with the mamujoco mask flags; MACPO with layer_N 1, as its mamujoco section
    has)."""
    dev = _cuda()
    cfg, orun, run, onets, outs = _iterations(algo, case, dev, T=5, N=64, H=128, seed=21, layer_N=1 if algo == "macpo" else 2)
    torch.cuda.synchronize()
    _check_iterations(algo, cfg, orun, run, onets, outs, rtol=1e-3, lr_frac=0.2)


UPDATE_SHAPES = {"config5": (2048, 398, 398, 20, 512), "mamujoco": (1000, 10, 14, 8, 128)}


@pytest.mark.gpu
@pytest.mark.parametrize("shape", list(UPDATE_SHAPES))
def test_masked_ppo_update_vs_oracle(shape):
    """MultiAgentTrainer.ppo_update with use_policy_active_masks (about a fifth of the rows inactive) against
    OracleMaskedMATrainer: two consecutive updates, the eight returned values, lamda_lagr, every gradient before the clip and all
    weights, at config 5's layers and at the MAMuJoCo shape (hidden 128)."""
    from safepo.common.ma_model import MultiAgentNets, MultiAgentTrainer
    from safepo.multi_agent import mappolag as M
    dev = _cuda()
    n, D, DS, A, H = UPDATE_SHAPES[shape]
    cfg = dict(M.DEFAULT_CONFIG, **{k: v for k, v in M.MAMUJOCO.items() if k not in ("episode_length", "n_rollout_threads", "hidden_size")},
               hidden_size=H)
    g = torch.Generator().manual_seed(n + D)
    sts = [HO.random_state(g, D, H, A, "actor", 2), HO.random_state(g, DS, H, 0, "critic", 2), HO.random_state(g, DS, H, 0, "critic", 2)]
    onets = [MA.OracleMANet(s, 2) for s in sts]
    otr = HO.OracleMaskedMATrainer(*onets, cfg)
    nets = MultiAgentNets(*sts, dev)
    tr = MultiAgentTrainer(nets, cfg)
    obs, share = torch.randn(n, D, generator=g) * 2 + 0.5, torch.randn(n, DS, generator=g) * 3
    with torch.no_grad():
        dist = MA.ma_actor_dist(onets[0], obs)
        actions = dist.mean + dist.stddev * torch.randn(n, A, generator=g)
        logp = dist.log_prob(actions)
    sample = dict(share_obs=share, obs=obs, actions=actions, value_preds=0.1 * torch.randn(n, 1, generator=g),
                  returns=torch.randn(n, 1, generator=g) * 4 + 1, old_action_log_probs=logp + 0.3 * torch.randn(n, A, generator=g) / A ** 0.5,
                  adv_targ=torch.randn(n, 1, generator=g), factor=torch.rand(n, 1, generator=g) + 0.5,
                  active_masks=(torch.rand(n, 1, generator=g) >= 0.2).float(), cost_preds=0.1 * torch.randn(n, 1, generator=g),
                  cost_returns=torch.randn(n, 1, generator=g) * 2, cost_adv_targ=torch.randn(n, 1, generator=g), aver_episode_costs=torch.tensor(30.0))
    names = _NAMES["mappolag"]
    for it in range(2):
        want = otr.ppo_update(sample)
        got = dict(zip(names, tr.ppo_update(dict(sample))))
        slack = 1.0 if it == 0 else 10.0
        for k in names:
            gv, wv = got[k].detach().cpu().reshape(-1).double(), want[k].reshape(-1).double()
            err = float((gv - wv).abs().max())
            assert err <= (1e-4 * float(wv.abs().max()) + 2e-6) * slack, (it, k, err, float(wv.abs().max()))
        assert abs(float(tr.lamda_lagr) - float(otr.lamda_lagr)) < 1e-6
        for net, onet, nk in ((nets.actor, onets[0], "actor_grad_norm"), (nets.critic, onets[1], "critic_grad_norm"),
                              (nets.cost_critic, onets[2], "cost_grad_norm")):
            coef = min(1.0, float(cfg["max_grad_norm"]) / (float(want[nk]) + 1e-6))
            for k, pt in onet.p.items():
                wg = pt.grad / coef
                err = float((net.g[k].cpu() - wg).abs().max())
                assert err <= (5e-5 * float(wg.abs().max()) + 1e-7) * slack, (it, k, err)
        for net, onet, lr in ((nets.actor, onets[0], cfg["actor_lr"]), (nets.critic, onets[1], cfg["critic_lr"]), (nets.cost_critic, onets[2], cfg["critic_lr"])):
            for k, pt in onet.p.items():
                assert float((net.p[k].cpu() - pt.detach()).abs().max()) < 0.05 * lr + 1e-6, (it, k)


@pytest.mark.gpu
def test_save_restore_eval_round_trip(tmp_path):
    """Agents of different sizes on the device: save -> restore into fresh nets is bit-exact per agent, and eval of the restored
    runner on the list-observation, padded-action environment equals eval of the saved one."""
    from safepo.common.synthetic_env import SyntheticMultiAgentEnv
    from safepo.multi_agent.mappolag import DEFAULT_CONFIG, Runner
    dev = _cuda()
    cfg = dict(DEFAULT_CONFIG, episode_length=4, n_rollout_threads=32, hidden_size=128)
    src = Runner(_nets_for(dev, (10, 14), 14, (9, 8), H=128, seed=1), cfg, [10, 14], 14, [9, 8], pad_actions_to=9)
    src.save(str(tmp_path), train_state=True)
    dst = Runner(_nets_for(dev, (10, 14), 14, (9, 8), H=128, seed=2), cfg, [10, 14], 14, [9, 8], pad_actions_to=9)
    dst.restore(str(tmp_path), train_state=True)
    for a in range(2):
        for n in ("actor", "critic", "cost_critic"):
            assert torch.equal(getattr(src.nets[a], n).flat, getattr(dst.nets[a], n).flat), (a, n)
    env = lambda: SyntheticMultiAgentEnv(8, 2, [10, 14], 14, 9, 3, 5, dev)      # noqa: E731
    assert src.eval(env(), 10) == dst.eval(env(), 10)
    assert src.last_eval == dst.last_eval and src.last_eval["episodes"] >= 10


@pytest.mark.gpu
@pytest.mark.parametrize("algo,extra", [(a, []) for a in ALGOS] + [("mappolag", ["--mamujoco"]), ("macpo", ["--mamujoco"])],
                         ids=list(ALGOS) + ["mappolag-mamujoco", "macpo-mamujoco"])
def test_cli_heterogeneous_agents(algo, extra, tmp_path):
    """Each CLI trains agents of 10 / 14 observations and 9 / 8 actions (padded to 9 for the environments) for two iterations
    and logs finite rows; MAPPO-Lag and MACPO also with their mamujoco sections."""
    _cuda()
    code = ("import sys, math; from safepo.multi_agent import %s as M; rows = M.main(sys.argv[1:]); "
            "assert len(rows) == 2 and all(math.isfinite(v) for r in rows for v in r.values() if isinstance(v, float)), rows; print(rows[-1])") % algo
    cmd = [sys.executable, "-c", code, "--iterations", "2", "--num-envs", "64", "--hidden-size", "128", "--share-obs-dim", "36",
           "--obs-dims", "10,14", "--act-dims", "9,8", "--pad-actions-to", "9", "--episode-len", "7", "--log-dir", str(tmp_path)] + extra
    if algo in ("mappo", "happo"):
        cmd += ["--agent-done-prob", "0.01"]
    r = subprocess.run(cmd, cwd=PKG, capture_output=True, text=True, env=dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, PKG])), timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
