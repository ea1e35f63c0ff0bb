"""Saving, restoring and evaluating multi-agent runs (safepo/multi_agent/mappolag.py: Runner.save / restore / eval / run, shared by
MAPPO-Lag, MACPO, MAPPO and HAPPO; safepo/common/ma_model.py: MultiAgentNets.save / load, the trainers' training state).

CPU: tests/ma_ckpt_oracle.py replays the reference's own save / restore / eval of tests/golden/ma_ckpt.pt bit for bit; the files
MultiAgentNets.save writes have the reference's keys, shapes and dtypes; malformed checkpoints raise SpoError; the host logic of
eval, resume and the CLI through the emulated C-ABI (tests/ma_emulator.py).  GPU: the same against the kernels, for all four
algorithms."""
import importlib
import os
import subprocess
import sys

import pytest
import torch

from ma_ckpt_oracle import OracleMACkptRunner, StubMAEnv
from oracle import ma_oracle as MA

ALGOS = ("mappolag", "macpo", "mappo", "happo")


def _fixture(golden):
    return golden("ma_ckpt")["ckpt"]


def _write_reference_files(fx, directory):
    os.makedirs(directory, exist_ok=True)
    for a, st in enumerate(fx["saved"]):
        for n in ("actor", "critic"):
            torch.save(st[n], os.path.join(directory, f"{n}_agent{a}.pt"))


def _single_thread():
    threads = torch.get_num_threads()
    torch.set_num_threads(1)            # the fixture was written with one intra-op thread
    return threads


def _cfg(fx):
    from safepo.multi_agent.mappolag import DEFAULT_CONFIG
    D, DS, A, H, NA = fx["dims"]
    xc, yc, layer_N = fx["std"]
    return dict(DEFAULT_CONFIG, hidden_size=H, layer_N=layer_N, std_x_coef=xc, std_y_coef=yc, episode_length=4,
                n_rollout_threads=len(fx["env"]["periods"]))


def _stub_env(fx, device="cpu"):
    D, DS, A, H, NA = fx["dims"]
    e = fx["env"]
    return StubMAEnv(NA, D, DS, e["periods"], e["seed"], alone=e["alone"], device=device)


def _random_state(g, din, H, layer_N, head, A=0):
    from safepo.multi_agent.mappolag import init_state
    st = init_state(din, H, layer_N, head, A, generator=g)
    return {k: v + 0.1 * torch.randn(v.shape, generator=g) for k, v in st.items()}


def _nets(fx, device, seed, cost_critic=True):
    from safepo.common.ma_model import MultiAgentNets
    D, DS, A, H, NA = fx["dims"]
    xc, yc, layer_N = fx["std"]
    g = torch.Generator().manual_seed(seed)
    return [MultiAgentNets(_random_state(g, D, H, layer_N, "actor", A), _random_state(g, DS, H, layer_N, "critic"),
                           _random_state(g, DS, H, layer_N, "critic") if cost_critic else None, device, layer_N=layer_N,
                           std_x_coef=xc, std_y_coef=yc) for _ in range(NA)]


# ============================================================ CPU ============================================================
def test_oracle_replays_reference_save_restore_eval_bit_for_bit(golden, tmp_path):
    """The oracle runner restores the reference-saved state dicts of ma_ckpt.pt, evaluates them on the stub environment to the
    reference's eval results exactly (one episode: environment 1 alone; four: three steps, two environments finishing at the
    last), and saving them again writes the same state dicts."""
    fx = _fixture(golden)
    D, DS, A, H, NA = fx["dims"]
    cfg = _cfg(fx)
    threads = _single_thread()
    try:
        g = torch.Generator().manual_seed(5)
        onets = [(MA.OracleMANet(_random_state(g, D, H, cfg["layer_N"], "actor", A), cfg["layer_N"]),
                  MA.OracleMANet(_random_state(g, DS, H, cfg["layer_N"], "critic"), cfg["layer_N"]),
                  MA.OracleMANet(_random_state(g, DS, H, cfg["layer_N"], "critic"), cfg["layer_N"])) for a in range(NA)]
        orun = OracleMACkptRunner(onets, cfg, cfg["episode_length"], cfg["n_rollout_threads"], D, DS, A)
        _write_reference_files(fx, tmp_path / "ref")
        orun.restore(str(tmp_path / "ref"))
        for k, want in fx["evals"].items():
            got = orun.eval(_stub_env(fx), k)
            assert (float(got[0]), float(got[1])) == want, (k, got, want)
            assert orun.last_eval["episodes"] == {1: 1, 4: 5}[k]
        orun.save(str(tmp_path / "again"))
        for a in range(NA):
            for n in ("actor", "critic"):
                st = torch.load(tmp_path / "again" / f"{n}_agent{a}.pt")
                assert list(st) == list(fx["saved"][a][n])
                assert all(torch.equal(st[k], v) for k, v in fx["saved"][a][n].items()), (a, n)
    finally:
        torch.set_num_threads(threads)


def test_saved_files_have_the_reference_format(golden, monkeypatch, tmp_path):
    """MultiAgentNets.save writes actor_agent{i}.pt / critic_agent{i}.pt with exactly the key set, shapes and dtypes of the
    reference-saved ones, as separate CPU tensors (not the packed buffer); load puts the reference's values into the packed
    buffers in place (same storage, Adam moments untouched) and leaves the cost critic alone."""
    import ma_emulator
    ma_emulator.install(monkeypatch)
    fx = _fixture(golden)
    nets = _nets(fx, "cpu", 1)
    for a, n_ in enumerate(nets):
        n_.save(str(tmp_path / "ours"), a)
        for n in ("actor", "critic"):
            st = torch.load(tmp_path / "ours" / f"{n}_agent{a}.pt", weights_only=True)
            ref = fx["saved"][a][n]
            assert set(st) == set(ref)
            for k, v in st.items():
                assert v.shape == ref[k].shape and v.dtype == ref[k].dtype == torch.float32 and v.device.type == "cpu", k
                assert v.untyped_storage().nbytes() == v.numel() * 4, k
    _write_reference_files(fx, tmp_path / "ref")
    for a, n_ in enumerate(nets):
        ptr, cost = n_.actor.flat.data_ptr(), n_.cost_critic.cpu_state_dict()
        n_.actor.exp_avg.fill_(0.25)
        n_.load(str(tmp_path / "ref"), a)
        assert n_.actor.flat.data_ptr() == ptr and bool((n_.actor.exp_avg == 0.25).all())
        for n, net in (("actor", n_.actor), ("critic", n_.critic)):
            for k, v in fx["saved"][a][n].items():
                assert torch.equal(net.p[k], v), (a, n, k)
                assert net.p[k].data_ptr() >= net.flat.data_ptr()
        assert all(torch.equal(v, n_.cost_critic.p[k]) for k, v in cost.items())


def test_malformed_checkpoints_raise(golden, monkeypatch, tmp_path):
    """A missing file, a missing or extra key, a wrong shape or a non-float tensor raises SpoError naming it, before anything is
    copied; so does a malformed training state."""
    import ma_emulator
    from safepo._lib import SpoError
    from safepo.multi_agent.mappolag import Runner
    ma_emulator.install(monkeypatch)
    fx = _fixture(golden)
    nets = _nets(fx, "cpu", 2)
    before = [n.actor.flat.clone() for n in nets]

    def case(name, edit, match):
        d = tmp_path / name
        _write_reference_files(fx, d)
        st = dict(fx["saved"][0]["actor"])
        edit(st)
        torch.save(st, d / "actor_agent0.pt")
        with pytest.raises(SpoError, match=match):
            nets[0].load(str(d), 0)
        assert torch.equal(nets[0].actor.flat, before[0])
    case("missing", lambda st: st.pop("act.action_out.log_std"), "missing key 'act.action_out.log_std'")
    case("extra", lambda st: st.update(extra=torch.zeros(1)), "unexpected key 'extra'")
    case("shape", lambda st: st.update({"base.mlp.fc1.0.weight": torch.zeros(3, 3)}), r"'base.mlp.fc1.0.weight' has shape \(3, 3\)")
    case("dtype", lambda st: st.update({"base.mlp.fc1.0.bias": torch.zeros(fx["dims"][3], dtype=torch.int64)}),
         "'base.mlp.fc1.0.bias' is not a floating-point tensor")
    (tmp_path / "nofile").mkdir()
    with pytest.raises(SpoError, match="no checkpoint"):
        nets[0].load(str(tmp_path / "nofile"), 0)
    run = Runner(nets, _cfg(fx), fx["dims"][0], fx["dims"][1], fx["dims"][2])
    run.save(str(tmp_path / "ts"), train_state=True)
    with pytest.raises(SpoError, match="no training state"):
        run.restore(str(tmp_path / "ref"), train_state=True)
    st = torch.load(tmp_path / "ts" / "train_state_agent1.pt", weights_only=True)
    st["trainer"]["nets"]["critic"]["exp_avg"].pop("v_out.bias")
    torch.save(st, tmp_path / "ts" / "train_state_agent1.pt")
    with pytest.raises(SpoError, match="missing key 'v_out.bias'"):
        run.restore(str(tmp_path / "ts"), train_state=True)


def _stream(g, T, N, D, DS, NA, alone):
    """One iteration of environment outputs: an environment finishing at step 1, with ``alone`` an agent finishing alone."""
    steps = []
    for t in range(T):
        dones = torch.zeros(N, NA, dtype=torch.bool)
        if t == 1:
            dones[1] = True
        if alone and t == T - 1:
            dones[0, 1] = True                       # carried into the next iteration's first active mask
        steps.append(dict(obs=torch.randn(N, NA, D, generator=g), share_obs=torch.randn(N, NA, DS, generator=g) * 2,
                          rewards=0.1 * torch.randn(N, NA, 1, generator=g), costs=(torch.rand(N, NA, 1, generator=g) < 0.3).float(),
                          dones=dones))
    return steps


def _draws(g, T, N, A, NA, iters):
    return dict(eps=[[torch.randn(N, A, generator=g) for _ in range(NA)] for _ in range(T)],
                order=torch.randperm(NA, generator=g).tolist(),
                perms=[[torch.randperm(T * N, generator=g) for _ in range(iters)] for _ in range(NA)])


def _iteration(run, steps, draws):
    dev = run.device
    for t, s in enumerate(steps):
        v, act, lp, cp = run.collect(t, eps=[e.to(dev) for e in draws["eps"][t]])
        run.insert(*(s[k].to(dev) for k in ("obs", "share_obs", "rewards", "costs", "dones")), v, act, lp, cp)
    run.compute()
    run.train(agent_order=draws["order"], perms=[[p.to(dev) for p in ps] for ps in draws["perms"]])
    run.return_aver_cost(torch.tensor(0.4 + 0.1 * len(steps)))
    run.iterations_done += 1


def _check_resume(algo, device, tmp_path, N=6, D=10, DS=14, A=3, H=32, NA=2, T=4):
    """Two iterations straight against one iteration, save with the training state, a fresh runner (other initial weights)
    restored from it and one more iteration, with the same injected draws: everything the runner carries must be equal."""
    M = importlib.import_module(f"safepo.multi_agent.{algo}")
    from safepo.common.ma_model import MultiAgentNets
    cfg = dict(M.DEFAULT_CONFIG, episode_length=T, n_rollout_threads=N, hidden_size=H, learning_iters=2)
    alone = algo in ("mappo", "happo")               # MAPPO-Lag / MACPO standardise with NaN on inactive entries (reference quirk)
    if alone:
        cfg.update(use_policy_active_masks=True, use_value_active_masks=True)

    def runner(seed):
        g = torch.Generator().manual_seed(seed)
        nets = [MultiAgentNets(_random_state(g, D, H, 2, "actor", A), _random_state(g, DS, H, 2, "critic"),
                               _random_state(g, DS, H, 2, "critic") if M.Runner.cost_critic else None, device) for _ in range(NA)]
        return M.Runner(nets, cfg, D, DS, A)
    g = torch.Generator().manual_seed(17)
    obs0, share0 = torch.randn(N, NA, D, generator=g), torch.randn(N, NA, DS, generator=g)
    streams = [_stream(g, T, N, D, DS, NA, alone) for _ in range(2)]
    draws = [_draws(g, T, N, A, NA, cfg["learning_iters"] if algo != "macpo" else 1) for _ in range(2)]
    straight = runner(1)
    straight.warmup(obs0.to(device), share0.to(device))
    for it in range(2):
        _iteration(straight, streams[it], draws[it])
    first = runner(1)
    first.warmup(obs0.to(device), share0.to(device))
    _iteration(first, streams[0], draws[0])
    first.save(str(tmp_path), train_state=True)
    resumed = runner(99)
    resumed.restore(str(tmp_path), train_state=True)
    assert resumed.iterations_done == 1
    _iteration(resumed, streams[1], draws[1])
    for a in range(NA):
        want, got = straight.trainer[a], resumed.trainer[a]
        for (name, wn), (_, gn) in zip(want._named_nets(), got._named_nets()):
            for k in ("flat", "exp_avg", "exp_avg_sq"):
                assert torch.equal(getattr(wn, k), getattr(gn, k)), (algo, a, name, k)
            assert wn.step == gn.step, (algo, a, name)
        assert torch.equal(want.popart_state, got.popart_state) and torch.equal(want.lamda_lagr, got.lamda_lagr), (algo, a)
        for k in ("obs", "share_obs", "masks", "active_masks", "returns", "factor"):
            assert torch.equal(getattr(straight.buffer[a], k), getattr(resumed.buffer[a], k)), (algo, a, k)
    if alone:
        assert float(straight.buffer[1].active_masks[0].min()) == 0.0       # the carried first step had an inactive agent
    assert any(float((straight.nets[a].actor.flat - first.nets[a].actor.flat).abs().max()) > 0 for a in range(NA))


def test_resume_through_emulated_abi(monkeypatch, tmp_path):
    """The resume check of MAPPO-Lag's runner with the emulated C-ABI (host logic: what is saved, what is restored)."""
    import ma_emulator
    ma_emulator.install(monkeypatch)
    _check_resume("mappolag", "cpu", tmp_path)


def test_eval_through_emulated_abi_vs_fixture(golden, monkeypatch, tmp_path):
    """Runner.eval with the emulated C-ABI on the reference-saved weights: the reference's results within float32 reordering,
    the finished-episode counts exactly."""
    import ma_emulator
    from safepo.multi_agent.mappolag import Runner
    ma_emulator.install(monkeypatch)
    fx = _fixture(golden)
    run = Runner(_nets(fx, "cpu", 3), _cfg(fx), *fx["dims"][:3])
    _write_reference_files(fx, tmp_path)
    run.restore(str(tmp_path))
    for k, (r, c) in fx["evals"].items():
        got = run.eval(_stub_env(fx), k)
        assert abs(got[0] - r) <= 1e-5 * abs(r) + 1e-6 and abs(got[1] - c) <= 1e-5 * abs(c) + 1e-6, (k, got, r, c)
        assert run.last_eval["episodes"] == {1: 1, 4: 5}[k]


def test_cli_save_eval_model_dir_resume_through_emulated_abi(monkeypatch, tmp_path):
    """The MAPPO-Lag CLI saves every iteration into <log-dir>/models_seed<seed> and logs Eval/EpRet with --use-eval;
    --model-dir restores and evaluates without training; --resume continues the iteration count from the training state."""
    import ma_emulator
    from safepo.multi_agent import mappolag as M
    ma_emulator.install(monkeypatch)
    common = ["--num-envs", "6", "--obs-dim", "10", "--share-obs-dim", "14", "--act-dim", "3", "--hidden-size", "32", "--episode-len", "3",
              "--device", "cpu"]
    log = tmp_path / "log"
    rows = M.main(common + ["--iterations", "2", "--use-eval", "--eval-interval", "1", "--save-train-state", "--log-dir", str(log)])
    assert len(rows) == 2 and all(r["Eval/EpRet"] != 0.0 for r in rows)
    saved = log / "models_seed0"
    assert sorted(os.listdir(saved)) == sorted(f"{n}_agent{a}.pt" for n in ("actor", "critic", "train_state") for a in range(2))
    rows = M.main(common + ["--iterations", "1", "--log-dir", str(tmp_path / "noeval")])
    assert rows[0]["Eval/EpRet"] == 0.0 and rows[0]["Eval/EpCost"] == 0.0         # no evaluation yet: 0.0, as in the reference

    def no_training(*a, **k):
        raise AssertionError("--model-dir must not train")
    with monkeypatch.context() as m:
        m.setattr(M.Runner, "train", no_training)
        out = M.main(common + ["--model-dir", str(saved), "--eval-episodes", "3", "--log-dir", str(tmp_path / "evalonly")])
    assert len(out) == 1 and set(out[0]) == {"Eval/EpRet", "Eval/EpCost", "Eval/Episodes"}
    assert not (tmp_path / "evalonly").exists()
    rows = M.main(common + ["--iterations", "1", "--resume", str(saved), "--save-dir", str(tmp_path / "resumed"), "--log-dir", str(log)])
    assert rows[0]["Train/Epoch"] == 2 and rows[0]["Train/TotalSteps"] == 3 * 8 * 6
    with pytest.raises(SystemExit):
        M.main(common + ["--model-dir", str(saved), "--resume", str(saved)])


def test_ma_ckpt_fixture_regenerates_identically(tmp_path):
    """make_ma_ckpt_golden.py writes the committed ma_ckpt.pt byte for byte (only where the reference is checked out)."""
    gen = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "make_ma_ckpt_golden.py")
    sys.path.insert(0, os.path.dirname(gen))
    import make_golden
    if not os.path.isdir(make_golden.REF):
        pytest.skip("the reference checkout is not present")
    out = tmp_path / "ma_ckpt.pt"
    r = subprocess.run([sys.executable, gen, str(out)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    with open(out, "rb") as f1, open(os.path.join(os.path.dirname(gen), "ma_ckpt.pt"), "rb") as f2:
        assert f1.read() == f2.read()


# ============================================================ GPU ============================================================
def _cuda():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    return torch.device("cuda:0")


def _close(got, want, rtol=2e-5, atol=1e-5):
    """The forward bar of the multi-agent nets (tests/test_gpu_parity.py: test_ma_get_actions_vs_oracle)."""
    got, want = torch.as_tensor(got).double().cpu(), torch.as_tensor(want).double().cpu()
    return bool(((got - want).abs() <= atol + rtol * want.abs()).all())


@pytest.mark.gpu
def test_reference_checkpoint_on_device(golden, tmp_path):
    """The reference-saved weights loaded into MultiAgentNets: deterministic get_actions / act and the values match the oracle
    on the same weights within the forward bar."""
    dev = _cuda()
    fx = _fixture(golden)
    D, DS, A, H, NA = fx["dims"]
    xc, yc, layer_N = fx["std"]
    _write_reference_files(fx, tmp_path)
    nets = _nets(fx, dev, 4)
    g = torch.Generator().manual_seed(6)
    obs, cent = torch.randn(257, D, generator=g) * 2 + 0.3, torch.randn(257, DS, generator=g) * 3
    for a, n_ in enumerate(nets):
        n_.load(str(tmp_path), a)
        oa, oc = MA.OracleMANet(fx["saved"][a]["actor"], layer_N), MA.OracleMANet(fx["saved"][a]["critic"], layer_N)
        with torch.no_grad():
            want_act, want_v = MA.ma_actor_dist(oa, obs, xc, yc).mean, MA.ma_critic_value(oc, cent)
        v, act, _, _ = n_.get_actions(cent.to(dev), obs.to(dev), deterministic=True)
        assert _close(act, want_act) and _close(v, want_v) and _close(n_.act(obs.to(dev)), want_act), a


@pytest.mark.gpu
def test_device_disk_device_round_trip(golden, tmp_path):
    """Save, load into fresh nets of other weights: every parameter identical bit for bit."""
    dev = _cuda()
    fx = _fixture(golden)
    src, dst = _nets(fx, dev, 7), _nets(fx, dev, 8)
    for a, (s, d) in enumerate(zip(src, dst)):
        s.save(str(tmp_path), a)
        d.load(str(tmp_path), a)
        for sn, dn in ((s.actor, d.actor), (s.critic, d.critic)):
            assert all(torch.equal(sn.p[k], dn.p[k]) for k in sn.p)


@pytest.mark.gpu
@pytest.mark.parametrize("algo", ALGOS)
def test_resume_equals_straight_run(algo, tmp_path):
    """One iteration, save with the training state, a fresh runner restored from it, one more iteration == two iterations
    straight, bit for bit: weights, Adam moments and steps, PopArt, lamda_lagr and the buffers (injected eps / perms / order)."""
    _check_resume(algo, _cuda(), tmp_path, N=64, D=18, DS=36, H=128)


class _CPUView:
    """An environment on the device seen from the CPU oracle: outputs to the CPU, actions to the device."""

    def __init__(self, env, dev):
        self.env, self.dev = env, dev

    def reset(self):
        return tuple(x.cpu() if torch.is_tensor(x) else x for x in self.env.reset())

    def step(self, actions):
        return tuple(x.cpu() if torch.is_tensor(x) else x for x in self.env.step([a.to(self.dev) for a in actions]))


@pytest.mark.gpu
def test_eval_matches_oracle(golden, tmp_path):
    """Runner.eval on the device against the oracle's eval: on the stub environment with the reference-saved weights (the
    reference's own results), and on the synthetic stream with agents finishing alone (--agent-done-prob > 0) -- the means
    within the forward bar, the finished-episode counts exactly."""
    from safepo.common.synthetic_env import SyntheticMultiAgentEnv
    from safepo.multi_agent.mappolag import Runner
    dev = _cuda()
    fx = _fixture(golden)
    D, DS, A, H, NA = fx["dims"]
    cfg = _cfg(fx)
    _write_reference_files(fx, tmp_path)
    run = Runner(_nets(fx, dev, 9), cfg, D, DS, A)
    run.restore(str(tmp_path))
    for k, (r, c) in fx["evals"].items():
        got = run.eval(_stub_env(fx, dev), k)
        assert _close(got[0], r) and _close(got[1], c) and run.last_eval["episodes"] == {1: 1, 4: 5}[k], (k, got, r, c)
    g = torch.Generator().manual_seed(10)
    onets = [(MA.OracleMANet(s["actor"], cfg["layer_N"]), MA.OracleMANet(s["critic"], cfg["layer_N"]),
              MA.OracleMANet(_random_state(g, DS, H, cfg["layer_N"], "critic"), cfg["layer_N"])) for s in fx["saved"]]
    orun = OracleMACkptRunner(onets, cfg, cfg["episode_length"], cfg["n_rollout_threads"], D, DS, A)

    def env():
        return SyntheticMultiAgentEnv(16, NA, D, DS, A, 7, 10003, dev, agent_done_prob=0.3)
    got, want = run.eval(env(), 20), orun.eval(_CPUView(env(), dev), 20)
    assert run.last_eval["episodes"] == orun.last_eval["episodes"] >= 20
    assert _close(run.last_eval["rewards"], orun.last_eval["rewards"]) and _close(run.last_eval["costs"], orun.last_eval["costs"])
    assert _close(got[0], want[0]) and _close(got[1], want[1])


@pytest.mark.gpu
@pytest.mark.parametrize("algo", ALGOS)
def test_cli_eval_save_and_model_dir(algo, tmp_path):
    """Each CLI trains with --use-eval --eval-interval 1 (finite Eval/EpRet every iteration, checkpoints written), then
    evaluates the run just saved with --model-dir."""
    import math
    M = importlib.import_module(f"safepo.multi_agent.{algo}")
    _cuda()
    common = ["--num-envs", "64", "--hidden-size", "128", "--obs-dim", "18", "--share-obs-dim", "36", "--act-dim", "3", "--episode-len", "5",
              "--agent-done-prob", "0.01"]
    rows = M.main(common + ["--iterations", "2", "--use-eval", "--eval-interval", "1", "--log-dir", str(tmp_path)])
    assert len(rows) == 2 and all(math.isfinite(r["Eval/EpRet"]) and r["Eval/EpRet"] != 0.0 for r in rows), rows
    out = M.main(common + ["--model-dir", str(tmp_path / "models_seed0"), "--eval-episodes", "5", "--log-dir", str(tmp_path / "e")])
    assert math.isfinite(out[0]["Eval/EpRet"]) and math.isfinite(out[0]["Eval/EpCost"])
