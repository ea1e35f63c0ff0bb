"""CPU-side checks: the C-ABI library loads and exports every symbol include/spo.h
declares, host logic (Lagrange, logger, minibatch order, synthetic env) against the golden
fixtures.  No kernel is launched here."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    from safepo import _lib as L
    lib = L.lib()
    header = open(os.path.join(ROOT, "include", "spo.h")).read()
    declared = set(re.findall(r"\b(spo_[a-z_]+)\s*\(", header))
    declared -= {"spo_status"}
    assert declared, "no declarations parsed"
    assert declared == set(L.EXPORTS)
    for name in declared:
        assert hasattr(lib, name), name
    assert lib.spo_version() == 100


def test_param_layout_matches_reference_counts():
    from safepo import _lib as L
    assert L.param_count(L.dims(60, 2)) == (8196, 8129, 24454)       # SURVEY Appendix B.4
    assert L.param_count(L.dims(88, 2)) == (9988, 9921, 9988 + 2 * 9921)
    assert L.param_count(L.dims(27, 8)) == (6480, 6017, 6480 + 2 * 6017)
    o = L.param_offsets(L.dims(60, 2), 0)
    assert (o["log_std"], o["w1"]) == (0, 2)                          # log_std first (cpo.py:70-78)
    with pytest.raises(L.SpoError):
        L.param_count(L.dims(60, 2, hidden=128))                      # no silent fallback


def test_lagrange_bit_exact(golden):
    from safepo.common.lagrange import Lagrange
    g = golden("lagrange")["lagrange"]
    lag = Lagrange(25.0, 0.001, 0.035)
    got = []
    for jc in g["jc"]:
        lag.update_lagrange_multiplier(jc)
        got.append(lag.lagrangian_multiplier)
    assert got == g["lam"]
    capped = Lagrange(25.0, 0.001, 0.035, lagrangian_upper_bound=2.0)
    got = []
    for _ in g["capped"]:
        capped.update_lagrange_multiplier(500.0)
        got.append(capped.lagrangian_multiplier)
    assert got == g["capped"]
    nan = Lagrange(25.0, 0.001, 0.035)
    nan.update_lagrange_multiplier(float("nan"))
    assert np.isnan(nan.lagrangian_multiplier)                        # reference quirk A3


def test_reference_minibatch_order(golden):
    from safepo.single_agent._engine import reference_order, LinearDecay
    g = golden("dataloader")["dataloader"]
    torch.manual_seed(g["seed"])
    for want in g["orders"]:
        assert torch.equal(reference_order(g["S"]), want)
    s = LinearDecay(3e-4, 2)
    assert s.step() == 0.00015 and s.step() == 0.0


def test_logger_semantics(tmp_path):
    from safepo.common.logger import EpochLogger
    lg = EpochLogger(str(tmp_path / "exp" / "task" / "algo" / "run"), seed="0", verbose=False, use_tensorboard=False)
    assert lg.get_stats("Metrics/EpCost") == 0.0                      # before the key was ever logged
    lg.store(**{"Metrics/EpCost": 3.0})
    lg.store(**{"Metrics/EpCost": 5.0})
    assert lg.get_stats("Metrics/EpCost") == 0.0
    lg.log_tabular("Metrics/EpCost")
    lg.log_tabular("Train/Epoch", 1)
    lg.dump_tabular()
    assert np.isnan(lg.get_stats("Metrics/EpCost"))                   # nothing stored since (A3)
    lg.store(**{"Metrics/EpCost": 7.0})
    assert lg.get_stats("Metrics/EpCost") == 7.0
    lg.close()
    rows = open(tmp_path / "exp" / "task" / "algo" / "run" / "progress.csv").read().strip().splitlines()
    assert rows[0] == "Metrics/EpCost,Train/Epoch" and rows[1].startswith("4.0,1")


def test_synthetic_env_contract():
    from safepo.common.synthetic_env import SyntheticVecEnv
    env = SyntheticVecEnv(4, 6, 2, episode_len=5, seed=1, stagger=True, p_terminate=0.1)
    obs, _ = env.reset()
    assert obs.shape == (4, 6) and obs.dtype == np.float32
    seen_final = False
    for _ in range(40):
        o, r, c, term, trunc, info = env.step(np.zeros((4, 2)))
        assert o.shape == (4, 6) and r.shape == (4,) and term.dtype == bool and not (term & trunc).any()
        if (term | trunc).any():
            fin = info["final_observation"]
            assert fin.dtype == object and all((f is not None) == d for f, d in zip(fin, term | trunc))
            seen_final = True
    assert seen_final
    env2 = SyntheticVecEnv(4, 6, 2, episode_len=5, seed=1, stagger=True, p_terminate=0.1)
    env2.reset()
    assert np.array_equal(env2.step(np.zeros((4, 2)))[0], SyntheticVecEnv(4, 6, 2, episode_len=5, seed=1, stagger=True, p_terminate=0.1).step(np.zeros((4, 2)))[0])


def test_gae_np_oracle_equals_path_oracle(golden):
    from oracle import spo_oracle as O
    for c in golden("gae")["gae_cases"]:
        a = O.gae_dual(c["rew"], c["cost"], c["v_r"], c["v_c"], c["seg_end"], c["boot_r"], c["boot_c"], c["gamma"], c["lam"], c["lam_c"])
        b = O.gae_dual_np(c["rew"], c["cost"], c["v_r"], c["v_c"], c["seg_end"], c["boot_r"], c["boot_c"], c["gamma"], c["lam"], c["lam_c"])
        for x, y in zip(a, b):
            assert torch.equal(x, y)


def test_no_cpu_fallback():
    from safepo import _lib as L
    from safepo.common.buffer import VectorizedOnPolicyBuffer
    from safepo.common.model import ActorVCritic

    class Sp:
        def __init__(self, d):
            self.shape = (d,)
    with pytest.raises(L.SpoError):
        VectorizedOnPolicyBuffer(Sp(4), Sp(2), size=8, device="cpu", num_envs=2)
    pol = ActorVCritic(4, 2)
    with pytest.raises(L.SpoError):
        pol.step(torch.zeros(3, 4))


def test_oracle_running_mean_std_matches_pooled_moments():
    """oracle/envio.py (restated gymnasium RunningMeanStd, parity unpinned): after any sequence of batch
    updates the statistics equal the pooled moments of all rows plus the prior pseudo-observations
    (count 1e-4 at mean 0, var 1) -- the defining property of the parallel-variance update."""
    import numpy as np
    from oracle import envio
    rng = np.random.default_rng(0)
    norm = envio.NormalizeObservation(5)
    xs = [rng.normal(2.0, 3.0, size=(n, 5)) for n in (7, 1, 64)]
    for x in xs:
        out = norm.normalize(x)
        np.testing.assert_allclose(out, (x - norm.obs_rms.mean) / np.sqrt(norm.obs_rms.var + 1e-8), rtol=0, atol=0)
    allx = np.concatenate(xs)
    c0, n = 1e-4, allx.shape[0]
    mean = allx.sum(0) / (n + c0)                      # prior mean 0
    ex2 = ((allx ** 2).sum(0) + c0 * 1.0) / (n + c0)   # prior E[x^2] = var + mean^2 = 1
    np.testing.assert_allclose(norm.obs_rms.mean, mean, rtol=1e-12)
    np.testing.assert_allclose(norm.obs_rms.var, ex2 - mean ** 2, rtol=1e-10)
    assert abs(norm.obs_rms.count - (n + c0)) < 1e-9
    frozen = norm.normalize(xs[0], update=False)
    assert abs(norm.obs_rms.count - (n + c0)) < 1e-9 and frozen.shape == xs[0].shape


def test_oracle_rescale_action_known_answers():
    import numpy as np
    from oracle import envio
    low, high = np.array([-2.0, 0.0]), np.array([2.0, 10.0])
    got = envio.rescale_action(np.array([[-1.0, -1.0], [0.0, 0.5], [1.0, 1.0], [3.0, -7.0]]), low, high)
    np.testing.assert_allclose(got, [[-2.0, 0.0], [0.0, 7.5], [2.0, 10.0], [2.0, 0.0]])


def test_pid_lagrangian_host_class_matches_reference(golden):
    """safepo.common.lagrange.PIDLagrangian (cppo_pid) against the sequence the reference's class produced."""
    from safepo.common.lagrange import PIDLagrangian
    c = golden("siblings")["pid"]
    P = PIDLagrangian(25.0, 0.001)
    for jc, want in zip(c["jc"], c["lam"]):
        P.update_lagrange_multiplier(jc)
        assert P.lagrangian_multiplier == want, (jc, P.lagrangian_multiplier, want)


def test_sibling_cli_modules_expose_reference_entry_points():
    import importlib
    for name in ("ppo", "pg", "cppo_pid", "trpo", "natural_pg", "rcpo", "pcpo", "cup", "ppo_lag", "focops", "cpo", "trpo_lag"):
        m = importlib.import_module(f"safepo.single_agent.{name}")
        assert callable(m.main) and isinstance(m.default_cfg, dict) and m.default_cfg["hidden_sizes"] == [64, 64]


def test_bench_reference_arm_prints_contract_line():
    """bench.py --impl reference runs without a GPU and prints ONE JSON line with the keys the driver reads."""
    import json
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "0",
                          "--cpu-seconds", "3", "--num-envs", "64", "--horizon", "50"], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [l for l in out.stdout.strip().splitlines() if l.startswith("{")]
    assert len(lines) == 1
    d = json.loads(lines[0])
    for k in ("impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline",
              "dtype", "data", "config", "cpu_baseline", "e2e"):
        assert k in d, k
    assert d["impl"] == "reference" and d["value"] > 0 and d["e2e"]["value"] == d["value"]
    assert d["cpu_baseline"]["kind"] == "port" and 1 <= d["cpu_baseline"]["cores"] <= 16


def test_bench_spo_arm_refuses_to_run_without_cuda():
    import os
    import subprocess
    import sys
    import torch
    if torch.cuda.is_available():
        pytest.skip("needs a host without CUDA")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--steps", "1", "--warmup", "0"], capture_output=True, text=True,
                         timeout=300)
    assert out.returncode != 0 and "no CPU fallback" in (out.stderr + out.stdout)


def test_c_abi_rejects_bad_arguments_before_touching_the_device():
    """Error behaviour of the C-ABI (include/spo.h): invalid arguments return a status code and leave a message in
    spo_last_error() without launching anything -- checked here without a GPU."""
    import ctypes as C
    from safepo import _lib as L
    lib = L.lib()
    OK = 0
    d_bad = L.dims(60, 2, hidden=32)
    a, c, t = C.c_int(), C.c_int(), C.c_int()
    assert lib.spo_param_count(C.byref(d_bad), C.byref(a), C.byref(c), C.byref(t)) != OK
    assert b"hidden" in lib.spo_last_error()
    d_big = L.dims(4096, 2)
    assert lib.spo_param_count(C.byref(d_big), C.byref(a), C.byref(c), C.byref(t)) != OK and b"obs_dim" in lib.spo_last_error()
    d = L.dims(60, 2)
    assert lib.spo_param_count(C.byref(d), C.byref(a), C.byref(c), C.byref(t)) == OK and (a.value, c.value) == (8196, 8129)
    # null pointers / empty batches
    assert lib.spo_policy_step(C.byref(d), None, None, None, 0, 0, 0, 0, None, None, None, None, None, 0, None) != OK
    assert b"spo_policy_step" in lib.spo_last_error()
    assert lib.spo_gae_dual(None, None, None, None, None, None, None, 0.99, 0.94, 0.94, None, None, None, None, 4, 5, 0, None) != OK
    assert lib.spo_adv_stats(None, None, 0, None, None) != OK and b"spo_adv_stats" in lib.spo_last_error()
    assert lib.spo_obs_normalize(None, 4, 3, None, None, 1.0, None, 1, 1e-8, None, None) != OK
    assert lib.spo_action_rescale(None, 4, 3, None, None, -1.0, 1.0, None, None) != OK
    assert lib.spo_gae_masked(None, None, None, 0.0, 1.0, 0.96, 0.9, None, 4, 8, None) != OK and b"spo_gae_masked" in lib.spo_last_error()
    assert lib.spo_ma_mlp_layer(None, 4, 10, None, None, None, None, 128, None, None, None, None) != OK and b"spo_ma_mlp_layer" in lib.spo_last_error()
    assert lib.spo_ma_head(None, 4, 128, None, None, 3, None, 1.0, 0.5, None, None, None, None) != OK
    # the multi-agent update entry points (second slice of SURVEY 8f rank 3)
    assert lib.spo_ma_mlp_layer_train(None, 4, 10, None, None, None, None, 128, None, None, None, None, None, None) != OK
    assert lib.spo_ma_ln_elu_bwd(None, None, None, 4, 128, None, None, None) != OK and b"spo_ma_ln_elu_bwd" in lib.spo_last_error()
    assert lib.spo_ma_ln_in_bwd(None, None, 4, 10, None, None) != OK
    assert lib.spo_ma_partial_reduce(None, 1, 4, 1, 4, None, None, None, 1.0, None) != OK
    assert lib.spo_ma_gemm_nn(None, None, None, 4, 4, 4, None) != OK and lib.spo_ma_gemm_tn(None, None, None, 4, 4, 4, 1, None) != OK
    assert lib.spo_ma_actor_loss(None, 4, 128, None, None, None, 3, None, None, None, None, None, None, 0.8, 1.2, 1.0, 0.5, None, None, None, None) != OK
    assert lib.spo_ma_actor_finalize(None, 1, 4, None, 3, 1.0, 0.5, 0.01, None, None, None, None) != OK
    assert lib.spo_ma_value_loss(None, None, None, None, 4, 0.2, 10.0, 0.25, None, None, None) != OK
    assert lib.spo_ma_popart_normalize(None, 4, None, 0.99999, 1e-5, None, None) != OK
    assert lib.spo_ma_lagrange_step(None, None, None, 4, 1.0, 0.96, 1e-5, None, None) != OK
    assert lib.spo_ma_clip_adam(None, None, None, None, 4, 10.0, 5e-4, 0.9, 0.999, 1e-5, 0.0, 1, None, None, None) != OK and b"spo_ma_clip_adam" in lib.spo_last_error()
    assert lib.spo_cg_begin(C.byref(d), None, None, None, None) != OK and lib.spo_cg_update(C.byref(d), None, None, 1e-10, 1e-6, None) != OK
    assert lib.spo_actor_forward(C.byref(d), None, None, 0, None, None) != OK
    assert lib.spo_fvp(C.byref(d), None, None, 0, None, 0.1, None, None) != OK
    # obs that is 4-byte but not 16-byte aligned at obs_dim % 4 == 0 (rows read as float4): refused before any launch.
    # The pointers are never dereferenced; any launch with them would fault.
    P, X, BAD = 0x100000, 0x200000, 0x300004
    n = 4
    step = lambda obs, st: lib.spo_policy_step(C.byref(d), P, obs, None, 1, 1, 0, n, X, X, X, X, st, 0, None)
    refusals = {
        "spo_policy_step": lambda: step(BAD, None),
        "spo_critic_values": lambda: lib.spo_critic_values(C.byref(d), P, BAD, n, X, X, None),
        "spo_actor_forward": lambda: lib.spo_actor_forward(C.byref(d), P, BAD, n, X, None),
        "spo_actor_kl": lambda: lib.spo_actor_kl(C.byref(d), P, BAD, X, X, n, 0, 0.02, X, None),
        "spo_actor_kl_accumulate": lambda: lib.spo_actor_kl_accumulate(C.byref(d), P, BAD, X, X, n, X, None),
        "spo_surrogate_grad": lambda: lib.spo_surrogate_grad(C.byref(d), P, BAD, X, X, X, n, X, X, None),
        "spo_fvp": lambda: lib.spo_fvp(C.byref(d), P, BAD, n, X, 0.1, X + 64, None),
        "spo_linesearch_eval": lambda: lib.spo_linesearch_eval(C.byref(d), P, BAD, X, X, X, X, X, X, n, X, None),
        "spo_conjugate_gradient": lambda: lib.spo_conjugate_gradient(C.byref(d), P, BAD, n, X, 10, 0.1, 1e-10, 1e-8, X, X, None),
    }
    for who, call in refusals.items():
        assert call() == -1, who                                                     # SPO_ERR_INVALID_ARG
        msg = lib.spo_last_error()
        assert who.encode() in msg and b"16-byte aligned" in msg, (who, msg)
    store = L.Rollout(obs=BAD, act=X, reward=X, cost=X, value_r=X, value_c=X, logp=X, seg_end=X, boot_r=X, boot_c=X,
                      num_envs=n, steps=3)
    assert step(X, C.byref(store)) == -1 and b"store->obs must be 16-byte aligned" in lib.spo_last_error()


def test_env_factory_imports_and_fails_loudly_without_safety_gymnasium():
    """ADVICE r1: `--env mujoco` must resolve to a real factory (safepo/common/env.py), not to a missing module."""
    import importlib.util
    from safepo import _lib as L
    from safepo.common.env import make_sa_mujoco_env
    if importlib.util.find_spec("safety_gymnasium") is None:
        with pytest.raises(L.SpoError, match="safety_gymnasium"):
            make_sa_mujoco_env(num_envs=2, env_id="SafetyPointGoal1-v0", seed=0)


def test_checkpoint_normalizer_object_has_gymnasium_surface():
    """ADVICE r1: the checkpointed "Normalizer" must be an object evaluate.py:56-57 can assign to eval_env.obs_rms:
    picklable, with numpy mean / var, count and update() (the pooled-moments merge of gymnasium's RunningMeanStd)."""
    import pickle
    import numpy as np
    from oracle import envio
    from safepo.common.normalizer import HostRunningMeanStd
    rng = np.random.default_rng(0)
    h, o = HostRunningMeanStd((5,)), envio.RunningMeanStd(shape=(5,))
    for _ in range(4):
        x = rng.normal(size=(7, 5)) * 3 + 1
        h.update(x); o.update(x)
    h2 = pickle.loads(pickle.dumps(h))
    assert np.array_equal(h2.mean, o.mean) and np.array_equal(h2.var, o.var) and h2.count == o.count
    h2.update(rng.normal(size=(3, 5)))
    assert h2.count == o.count + 3 and h2.mean.shape == (5,)


def test_vectorised_episode_accounting_is_bit_identical_to_the_per_env_loop():
    """SURVEY 8f rank 4: the per-step bookkeeping of finished episodes (50-episode deques, one logged running mean per finished
    episode, ascending env index) without a Python loop over envs -- same numbers, bit for bit, as the reference-style loop."""
    from collections import deque
    import numpy as np
    from safepo.single_agent._engine import Rollout

    class Log:
        def __init__(self):
            self.epoch_dict, self.logged = {}, True

        def store(self, **kw):
            for k, v in kw.items():
                self.epoch_dict.setdefault(k, []).append(v)

    rng = np.random.default_rng(0)
    N = 300
    fast = Rollout.__new__(Rollout)            # only the accounting state, no device objects
    fast.logger = Log()
    fast.ep_ret, fast.ep_cost, fast.ep_len = rng.normal(size=N) * 10, rng.random(N) * 50, rng.integers(1, 1000, N).astype(float)
    fast.rew_deque, fast.cost_deque, fast.len_deque = deque(maxlen=50), deque(maxlen=50), deque(maxlen=50)
    ref_ret, ref_cost, ref_len = fast.ep_ret.copy(), fast.ep_cost.copy(), fast.ep_len.copy()
    rd, cd, ld = deque(maxlen=50), deque(maxlen=50), deque(maxlen=50)
    want = {"Metrics/EpRet": [], "Metrics/EpCost": [], "Metrics/EpLen": []}
    for step in range(12):
        k = [3, 40, 9, 120, 300, 1, 0, 64, 300, 2, 51, 299][step]
        finished = np.sort(rng.choice(N, size=k, replace=False))
        for idx in finished:                    # the reference's loop, ppo_lag.py:216-230
            rd.append(ref_ret[idx]); cd.append(ref_cost[idx]); ld.append(ref_len[idx])
            want["Metrics/EpRet"].append(np.mean(rd)); want["Metrics/EpCost"].append(np.mean(cd)); want["Metrics/EpLen"].append(np.mean(ld))
            ref_ret[idx] = ref_cost[idx] = ref_len[idx] = 0.0
        fast._account_finished(finished)
        bump = rng.normal(size=N)
        fast.ep_ret += bump; ref_ret += bump
        fast.ep_cost += np.abs(bump); ref_cost += np.abs(bump)
        fast.ep_len += 1; ref_len += 1
    for key in want:
        got = np.asarray(fast.logger.epoch_dict[key], dtype=np.float64)
        assert got.shape == (len(want[key]),) and np.array_equal(got, np.asarray(want[key])), key
    assert list(fast.rew_deque) == list(rd) and list(fast.len_deque) == list(ld)
    assert np.array_equal(fast.ep_ret, ref_ret) and not fast.logger.logged


def test_multi_agent_net_packing_and_no_cpu_path():
    """safepo/common/ma_model.py host logic: one packed fp32 buffer per net with every tensor on a 16-byte boundary, parameters and
    gradients as views under the reference's state_dict names; the nets refuse a CPU device (no fallback)."""
    from safepo import _lib as L
    from safepo.common.ma_model import MultiAgentNets, _Net
    g = torch.Generator().manual_seed(0)
    D, H, A = 10, 128, 3
    st = {"base.feature_norm.weight": torch.randn(D, generator=g), "base.feature_norm.bias": torch.randn(D, generator=g)}
    dims = [D, H, H]
    for li, name in enumerate(("fc1", "fc2.0")):
        st[f"base.mlp.{name}.0.weight"] = torch.randn(H, dims[li], generator=g)
        st[f"base.mlp.{name}.0.bias"] = torch.randn(H, generator=g)
        st[f"base.mlp.{name}.2.weight"] = torch.randn(H, generator=g)
        st[f"base.mlp.{name}.2.bias"] = torch.randn(H, generator=g)
    st["act.action_out.log_std"] = torch.randn(A, generator=g)
    st["act.action_out.fc_mean.weight"] = torch.randn(A, H, generator=g)
    st["act.action_out.fc_mean.bias"] = torch.randn(A, generator=g)
    net = _Net(st, torch.device("cpu"), layer_N=1)
    assert (net.D, net.H, len(net.blocks)) == (D, H, 2)
    base = net.flat.data_ptr()
    for k, v in st.items():
        assert torch.equal(net.p[k], v) and net.p[k].shape == v.shape
        assert (net.p[k].data_ptr() - base) % 16 == 0 and (net.g[k].data_ptr() - net.gflat.data_ptr()) == (net.p[k].data_ptr() - base)
    net.flat.zero_()                                    # the parameters are views of the packed buffer
    assert all(float(t.abs().sum()) == 0.0 for t in net.p.values())
    assert net.flat.numel() >= sum(v.numel() for v in st.values()) and net.flat.numel() % 4 == 0
    sd = net.state_dict()
    assert list(sd) == list(st)                        # state_dict order and names of the reference
    with pytest.raises(L.SpoError, match="CUDA"):
        MultiAgentNets(st, st, st, "cpu")



# ---- host orchestration of the multi-agent path, with the C-ABI emulated on the CPU (tests/ma_emulator.py: test infrastructure) ----
def _ma_small_state(g, din, H, A, head):
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


def test_multi_agent_trainer_call_sequence_vs_oracle(golden, monkeypatch):
    """MultiAgentTrainer.ppo_update driven through the emulated C-ABI: the sequence of entry points, the buffers handed to each
    and the partial-sum layouts the host relies on reproduce the oracle's update (gradients, returned quantities, lamda, PopArt,
    weights after two updates).  The kernels behind the real entry points are checked on the GPU by test_ma_ppo_update_vs_oracle."""
    import ma_emulator
    from oracle import ma_oracle as MA
    from safepo.common.ma_model import MultiAgentNets, MultiAgentTrainer
    ma_emulator.install(monkeypatch)
    cfg = dict(golden("ma_update")["ma_update"]["cfg"])
    cfg["entropy_coef"] = 0.01
    N, D, DS, A, H = 300, 10, 14, 3, 32
    g = torch.Generator().manual_seed(4)
    sa, sc, sk = _ma_small_state(g, D, H, A, "actor"), _ma_small_state(g, DS, H, A, "critic"), _ma_small_state(g, DS, H, A, "critic")
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
                  cost_adv_targ=torch.randn(N, 1, generator=g), aver_episode_costs=torch.rand(7, 5, generator=g) * 60)   # only its mean is used
    otr = MA.OracleMATrainer(oa, oc, ok_, cfg)
    nets = MultiAgentNets(sa, sc, sk, "cpu", layer_N=cfg["layer_N"], std_x_coef=cfg["std_x_coef"], std_y_coef=cfg["std_y_coef"])
    tr = MultiAgentTrainer(nets, cfg)
    got_v, got_a, got_lp, got_k = nets.get_actions(share, obs, deterministic=True)
    assert torch.allclose(got_v, v0, atol=2e-6) and torch.allclose(got_a, dist.mean, atol=2e-6) and torch.allclose(got_k, k0, atol=2e-6)
    assert torch.allclose(nets.evaluate_actions(obs, actions), logp, atol=1e-5)
    names = ("value_loss", "critic_grad_norm", "policy_loss", "dist_entropy", "actor_grad_norm", "imp_weights", "cost_loss", "cost_grad_norm")
    for it in range(2):
        want = otr.ppo_update(sample)
        got = dict(zip(names, tr.ppo_update(sample)))
        for k in names:
            assert torch.allclose(got[k].reshape(-1), torch.as_tensor(want[k]).reshape(-1), rtol=2e-4, atol=2e-6), (it, k, got[k], want[k])
        for net, onet, nk in ((nets.actor, oa, "actor_grad_norm"), (nets.critic, oc, "critic_grad_norm"), (nets.cost_critic, ok_, "cost_grad_norm")):
            coef = min(1.0, float(cfg["max_grad_norm"]) / (float(want[nk]) + 1e-6))
            for k, pt in onet.p.items():
                wg = pt.grad / coef
                assert float((net.g[k] - wg).abs().max()) <= 1e-4 * float(wg.abs().max()) + 1e-7, (it, k)
                assert float((net.p[k] - pt.detach()).abs().max()) < 2e-5, (it, k)
        assert abs(float(tr.lamda_lagr) - float(otr.lamda_lagr)) < 1e-6
        for got_s, want_s in zip(tr.popart_state, (otr.popart.running_mean, otr.popart.running_mean_sq, otr.popart.debiasing_term)):
            assert abs(float(got_s) - float(want_s)) <= 1e-5 * abs(float(want_s)) + 1e-12


def test_multi_agent_runner_iteration_vs_oracle(golden, monkeypatch):
    """safepo/multi_agent/mappolag.py Runner (collect / insert / compute / train) with SeparatedReplayBuffer and
    MultiAgentTrainer.train through the emulated C-ABI, against the oracle's runner (itself pinned bit for bit to the reference's
    Runner by tests/golden/ma_epoch.pt) on the fixture's environment stream with the same injected draws: two iterations of two
    agents -- buffers after compute(), the cross-agent factor, lamda, PopArt and all weights after train()."""
    import ma_emulator
    from oracle import ma_oracle as MA
    from safepo.common.ma_model import MultiAgentNets
    from safepo.multi_agent.mappolag import Runner
    ma_emulator.install(monkeypatch)
    c = golden("ma_epoch")["ma_epoch"]
    T, N, D, DS, A, H, NA = c["dims"]
    cfg = dict(c["cfg"])
    onets = [tuple(MA.OracleMANet(st[n], layer_N=cfg["layer_N"]) for n in ("actor", "critic", "cost_critic")) for st in c["init"]]
    orun = MA.OracleMARunner(onets, cfg, T, N, D, DS, A)
    nets = [MultiAgentNets(st["actor"], st["critic"], st["cost_critic"], "cpu", layer_N=cfg["layer_N"], std_x_coef=cfg["std_x_coef"],
                           std_y_coef=cfg["std_y_coef"]) for st in c["init"]]
    run = Runner(nets, cfg, D, DS, A)
    orun.warmup(c["obs0"], c["share_obs0"])
    run.warmup(c["obs0"], c["share_obs0"])
    g = torch.Generator().manual_seed(9)

    def near(a, b, tol=2e-5):
        return float((a - b).abs().max()) <= tol * (1.0 + float(b.abs().max()))
    for it in range(2):
        for step in range(T):
            s = c["stream"][it][step]
            eps = [torch.randn(N, A, generator=g) for _ in range(NA)]
            ov, oact, olp, ocp = orun.collect(step, eps=eps)
            v, act, lp, cp = run.collect(step, eps=eps)
            assert near(v, ov) and near(cp, ocp) and all(near(act[a], oact[a]) and near(lp[a], olp[a]) for a in range(NA)), (it, step)
            orun.insert(s["obs"], s["share_obs"], s["rewards"], s["costs"], s["dones"], ov, oact, olp, ocp)
            run.insert(s["obs"], s["share_obs"], s["rewards"], s["costs"], s["dones"], v, act, lp, cp)
        orun.compute()
        run.compute()
        for a in range(NA):
            for k in ("returns", "cost_returns", "value_preds", "cost_preds", "masks", "active_masks", "rewards", "costs", "actions", "obs", "share_obs"):
                assert near(getattr(run.buffer[a], k), getattr(orun.buffer[a], k), 5e-5), (it, a, k)
        order = torch.randperm(NA, generator=g)
        perms = [[torch.randperm(T * N, generator=g) for _ in range(cfg["learning_iters"])] for _ in range(NA)]
        orun.train(agent_order=order, perms=perms)
        assert run.train(agent_order=order, perms=perms) == [int(a) for a in order]
        for a in range(NA):
            assert near(run.buffer[a].factor, orun.buffer[a].factor, 1e-4), (it, a)
            assert abs(float(run.trainer[a].lamda_lagr) - float(orun.trainer[a].lamda_lagr)) < 1e-6
            pop = orun.trainer[a].popart
            for got_s, want_s in zip(run.trainer[a].popart_state, (pop.running_mean, pop.running_mean_sq, pop.debiasing_term)):
                assert abs(float(got_s) - float(want_s)) <= 1e-5 * abs(float(want_s)) + 1e-12
            for net, onet in zip((nets[a].actor, nets[a].critic, nets[a].cost_critic), onets[a]):
                for k, pt in onet.p.items():
                    assert float((net.p[k] - pt.detach()).abs().max()) < 5e-5, (it, a, k)
            assert near(run.buffer[a].obs[0], orun.buffer[a].obs[0]) and near(run.buffer[a].masks[0], orun.buffer[a].masks[0])    # after_update
        if it == 0:
            run.return_aver_cost(torch.tensor(c["aver_cost_after_first"]))
            for b in orun.buffer:
                b.aver_episode_costs = torch.tensor(c["aver_cost_after_first"])
    assert any(bool((run.buffer[a].factor != 1).any()) for a in range(NA))


def test_multi_agent_run_loop_and_cli_through_emulated_abi(monkeypatch, tmp_path):
    """Runner.run (the loop of mappolag.py:300-373) on the synthetic multi-agent environment and the module's CLI, host logic only
    (emulated C-ABI): episode sums and finished-episode means, the average episode cost handed to the buffers, per-agent log
    columns, weights that move, a progress.csv; the reference's initialisation (orthogonal weights, zero biases, log_std = x_coef)."""
    import ma_emulator
    from safepo.common.ma_model import MultiAgentNets
    from safepo.common.synthetic_env import SyntheticMultiAgentEnv
    from safepo.multi_agent import mappolag as M
    ma_emulator.install(monkeypatch)
    g = torch.Generator().manual_seed(0)
    st = M.init_state(10, 32, 2, "actor", act_dim=3, generator=g)
    w = st["base.mlp.fc2.0.0.weight"]
    gain2 = float(torch.nn.init.calculate_gain("relu")) ** 2
    assert torch.allclose(w @ w.t(), gain2 * torch.eye(32), atol=1e-4)                   # orthogonal with the ReLU gain
    assert float(st["base.mlp.fc1.0.bias"].abs().max()) == 0.0 and torch.equal(st["act.action_out.log_std"], torch.ones(3))
    assert float((st["act.action_out.fc_mean.weight"] @ st["act.action_out.fc_mean.weight"].t() - 1e-4 * torch.eye(3)).abs().max()) < 1e-6
    cfg = dict(M.DEFAULT_CONFIG, episode_length=4, n_rollout_threads=6, hidden_size=32, learning_iters=2, entropy_coef=0.01)
    T, N, D, DS, A, NA = 4, 6, 10, 14, 3, 2

    def build(seed):
        gg = torch.Generator().manual_seed(seed)
        nets = [MultiAgentNets(M.init_state(D, 32, 2, "actor", A, generator=gg), M.init_state(DS, 32, 2, "critic", generator=gg),
                               M.init_state(DS, 32, 2, "critic", generator=gg), "cpu") for _ in range(NA)]
        return M.Runner(nets, cfg, D, DS, A), SyntheticMultiAgentEnv(N, NA, D, DS, A, episode_len=3, seed=seed, device="cpu")
    run, envs = build(1)
    w0 = run.nets[0].actor.flat.clone()
    torch.manual_seed(5)
    rows = run.run(envs, 3)
    assert [r["Train/TotalSteps"] for r in rows] == [24, 48, 72]
    assert all("Metrics/EpCost" in r and "Loss/Loss_actor/agent1" in r and "Misc/Lagrange/agent0" in r for r in rows)
    assert run.buffer[0].aver_episode_costs.numel() == 1                                  # replaced by the finished episodes' mean cost
    assert abs(float(run.buffer[0].aver_episode_costs) - rows[-1]["Metrics/EpCost"]) < 1e-6
    assert 0.0 <= rows[0]["Metrics/EpCost"] <= 3.0                                        # episodes of 3 steps, cost in {0, 1} per step
    assert float((run.nets[0].actor.flat - w0).abs().max()) > 0
    assert torch.equal(run.buffer[1].obs[0], run.buffer[1].obs[-1])                       # after_update rolled the last observation over
    run2, envs2 = build(1)
    torch.manual_seed(5)
    rows2 = run2.run(envs2, 3)
    drop = ("Time/Total", "Time/FPS")
    assert [{k: v for k, v in r.items() if k not in drop} for r in rows] == [{k: v for k, v in r.items() if k not in drop} for r in rows2]
    out = M.main(["--num-envs", "6", "--obs-dim", "10", "--share-obs-dim", "14", "--act-dim", "3", "--hidden-size", "32", "--iterations", "2",
                  "--episode-len", "5", "--device", "cpu", "--log-dir", str(tmp_path / "exp" / "synthetic" / "mappolag" / "seed0")])
    assert len(out) == 2
    csv_text = (tmp_path / "exp" / "synthetic" / "mappolag" / "seed0" / "progress.csv").read_text()
    assert "Loss/Loss_reward_critic/agent0" in csv_text and len(csv_text.strip().splitlines()) == 3
    with pytest.raises(ValueError):
        envs.step([torch.zeros(N, A)])                                                     # one action tensor per agent
