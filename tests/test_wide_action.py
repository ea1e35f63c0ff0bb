"""Action dimensions 9..16 (the Doggo robot has 12 actuators): the kernels' AC = 16 instantiations against float64 and
the oracle, the trainers at the SafetyDoggoGoal1-v0 shape, and the refusals at the edges.

The checks reuse the per-tensor machinery of test_update_gradients.py (float64 reference step, gradient readout through
Adam's first moment, trust-region comparisons) and the forward checks of test_gpu_parity.py at act_dim > 8; the bars
are theirs (DESIGN section 5).  Run the GPU part with ``-s`` to see the measured maxima."""
import csv
import ctypes as C
import importlib
import os
import subprocess
import sys

import pytest
import torch

from oracle import spo_oracle as O
from oracle import trainers as TR

import test_gpu_parity as GP
import test_update_gradients as T

WIDE_A = (9, 12, 16)
WIDE_D = (1, 64, 65, 104, 128)
SPO_ERR_UNSUPPORTED = -2     # include/spo.h

# Bars: those of test_update_gradients.py except two, each at most 4x the largest error measured over this file's matrix
# on one H100 80 GB.  loss 2.2e-6: the cost critic's loss of one row (focops-128-9-1), a squared difference of nearly equal
# numbers; tr_loss 1.1e-6: the surrogate of a single row at act 16, whose log-density sums 16 terms before the exp.
WIDE_BAR = dict(T.BAR, loss=8e-6, tr_loss=4e-6)


@pytest.fixture(autouse=True)
def _wide_bars(monkeypatch):
    for k, v in WIDE_BAR.items():
        monkeypatch.setitem(T.BAR, k, v)


# ---------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("A", [12, 16])
@pytest.mark.parametrize("kind", ["ppo", "pg", "focops", "critic"])
def test_reference_step_matches_oracle_bit_for_bit_wide(kind, A):
    """The float64 reference step, run in float32, equals the oracle's minibatch step bit for bit at act_dim 12 / 16."""
    D, B = 23, 48
    torch.manual_seed(21 + A)
    pol = O.OraclePolicy(D, A)
    with torch.no_grad():
        pol.nets["actor"]["log_std"].copy_(torch.linspace(-0.4, 0.3, A))
    b = T._cpu_batch(pol, B, torch.Generator().manual_seed(5 + A), D, A)
    mine = T.unpack(T.pack(pol), D, A)
    got = T.ref_step(mine, b, kind, T.HP_REF)
    want = O.minibatch_step(pol, O.OracleOptim(pol), b, kind, max_grad_norm=40.0, target_kl=T.HP_REF["focops_kl"])
    for w, g_ in zip(want, got["losses"]):
        if g_ is not None:
            assert w == g_, (kind, A, w, g_)
    for net in T.ACTIVE[kind]:
        for p, g_ in zip(pol.params(net), got["grads"][net]):
            assert torch.equal(p.grad, g_), (kind, A, net)


@pytest.mark.parametrize("A", [12, 16])
def test_reference_cup_step_matches_oracle_bit_for_bit_wide(A):
    D, B = 9, 40
    torch.manual_seed(31 + A)
    pol = O.OraclePolicy(D, A)
    data = T._cpu_batch(pol, B, torch.Generator().manual_seed(7 + A), D, A)
    data["adv_c"] = data["adv"]
    lam, gamma = 0.7, 0.99
    mine = T.unpack(T.pack(pol), D, A)
    with torch.no_grad():
        om, os_ = O.actor_mean_std(mine, data["obs"])
    b = dict(data, old_mean=om.clone(), old_std=os_.expand_as(om).clone())
    got = T.ref_step(mine, b, "cup", dict(T.HP_REF, cup_coef=lam * ((1 - gamma * 0.95) / (1 - gamma))))
    O.cup_second_stage(pol, O.OracleOptim(pol), data, lam, gamma=gamma, batch_size=B, learning_iters=1, target_kl=1e9,
                       perms=[torch.arange(B)])
    for p, g_ in zip(pol.params("actor"), got["grads"]["actor"]):
        assert torch.equal(p.grad, g_)


def test_doggo_task_dims():
    from safepo.common import synthetic_env as senv
    assert senv.TASK_DIMS["SafetyDoggoGoal1-v0"] == (104, 12)
    assert all(1 <= d <= 128 and 1 <= a <= 16 for d, a in senv.TASK_DIMS.values())


def test_act_dim_17_is_refused():
    from safepo import _lib as L
    assert L.param_count(L.dims(104, 16))[0] == 16 + 64 * 104 + 64 + 64 * 64 + 64 + 16 * 64 + 16
    with pytest.raises(L.SpoError, match="act_dim=17"):
        L.param_count(L.dims(104, 17))


def test_data_parallel_update_refuses_act_dim_above_8():
    """spo_pg_update_dp across GPUs sizes its gradient slots for act_dim <= 8; wider actors are refused before any launch
    (the pointers below are never dereferenced)."""
    from safepo import _lib as L
    fake = C.c_void_p(256)
    bt = L.Batch(fake, fake, fake, fake, fake, fake, None, None, 1024)
    hp = T._hparams(L, "ppo", T.make_hp())
    comm = L.Comm(2, 0, fake, None, 0, 0)
    for A, want in ((12, SPO_ERR_UNSUPPORTED), (16, SPO_ERR_UNSUPPORTED)):
        d = L.dims(104, A)
        rc = L.lib().spo_pg_update_dp(C.byref(d), fake, fake, fake, fake, C.byref(bt), fake, 1024, 64, 0, C.byref(hp), fake,
                                      C.byref(comm), None)
        assert rc == want, (A, rc)
        assert b"act_dim" in L.lib().spo_last_error()


# ---------------------------------------------------------------------------------------------------------------
# GPU: the minibatch update kernel (AC = 16) against float64
# ---------------------------------------------------------------------------------------------------------------

READOUT_WIDE = [
    ("ppo", 1, 9, 1, dict(clip_lo=0.7, clip_hi=1.3, critic_l2=0.1, value_coef=2.0)),
    ("ppo", 64, 12, 64, dict()),
    ("ppo", 65, 16, 100, dict(critic_l2=0.0, value_coef=2.0)),
    ("ppo", 104, 12, 100, dict(clip_lo=0.7, clip_hi=1.3, critic_l2=0.1)),
    ("ppo", 128, 16, 64, dict(value_coef=2.0)),
    ("ppo", 104, 9, 64, dict()),
    ("pg", 104, 12, 64, dict()),
    ("pg", 128, 9, 100, dict(critic_l2=0.1, value_coef=2.0)),
    ("focops", 104, 12, 64, dict(focops_kl=0.05)),
    ("focops", 65, 16, 64, dict(focops_lam=0.3, focops_kl=0.05, critic_l2=0.1, value_coef=2.0)),
    ("focops", 128, 9, 1, dict(focops_lam=0.3, focops_kl=0.05, critic_l2=0.0, value_coef=2.0)),
    ("focops", 1, 16, 64, dict(focops_kl=0.05)),
    ("cup", 104, 12, 64, dict(cup_coef=0.7)),
    ("cup", 64, 16, 1, dict(cup_coef=2.5)),
    ("critic", 104, 12, 100, dict(value_coef=2.0)),
    ("critic", 65, 16, 64, dict(critic_l2=0.1)),
    ("critic", 1, 9, 1, dict(critic_l2=0.0, value_coef=2.0)),
]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,D,A,B,extra", READOUT_WIDE, ids=[f"{k}-{d}-{a}-{b}" for k, d, a, b, _ in READOUT_WIDE])
def test_wide_update_gradient_readout_vs_float64(kind, D, A, B, extra):
    T.test_update_gradient_readout_vs_float64(kind, D, A, B, extra)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,D,A,B,extra", [
    ("ppo", 104, 12, 100, dict(value_coef=2.0)),
    ("pg", 128, 16, 64, dict()),
    ("focops", 65, 16, 64, dict(focops_kl=0.05)),
    ("cup", 104, 12, 64, dict(cup_coef=0.7)),
])
def test_wide_update_clip_coefficient_vs_float64(kind, D, A, B, extra):
    T.test_update_clip_coefficient_vs_float64(kind, D, A, B, extra)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,D,A,batch,K,extra", [
    ("ppo", 104, 12, 100, 5, dict(critic_l2=0.1, value_coef=2.0)),
    ("ppo", 128, 16, 64, 5, dict()),
    ("critic", 65, 16, 128, 5, dict()),
])
def test_wide_update_multistep_fixed_weights_emas(kind, D, A, batch, K, extra):
    T.test_update_multistep_fixed_weights_emas(kind, D, A, batch, K, extra)


CLUSTER_CASES = [READOUT_WIDE[3], READOUT_WIDE[9], READOUT_WIDE[13]]   # PPO (104, 12, 100), FOCOPS (65, 16, 64), CUP (64, 16, 1)


def dump_cluster_cases(path):
    out = {}
    for kind, D, A, B, extra in CLUSTER_CASES:
        st, _, res, _ = T.run_readout(kind, D, A, B, extra)
        out[f"{kind}-{D}-{A}-{B}"] = (st["m"].cpu(), st["v"].cpu(), torch.tensor(res["loss_sum"], dtype=torch.float64))
    torch.save(out, path)


@pytest.mark.gpu
def test_wide_update_16_cta_cluster_matches_12(tmp_path):
    """The 16-CTA cluster fallback (four CTAs idle) against the 12-CTA cluster at act_dim 12 / 16: bit-identical moments
    and losses.  The cluster size is cached per process, so the 16-CTA run is a subprocess with SPO_CLUSTER=16."""
    here = os.path.dirname(os.path.abspath(__file__))
    root = os.path.dirname(here)
    path = str(tmp_path / "c16.pt")
    code = ("import sys; sys.path[:0] = {!r}; import test_wide_action as W; W.dump_cluster_cases({!r})"
            .format([root, os.path.join(root, "safe-policy-optimization_b200"), here], path))
    r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, SPO_CLUSTER="16"), cwd=root, capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    got = torch.load(path)
    for kind, D, A, B, extra in CLUSTER_CASES:
        st, _, res, _ = T.run_readout(kind, D, A, B, extra)
        m16, v16, l16 = got[f"{kind}-{D}-{A}-{B}"]
        assert torch.equal(st["m"].cpu(), m16) and torch.equal(st["v"].cpu(), v16), kind
        assert l16.tolist() == res["loss_sum"], (kind, l16.tolist(), res["loss_sum"])


# ---------------------------------------------------------------------------------------------------------------
# GPU: trust-region kernels (AC = 16) against float64
# ---------------------------------------------------------------------------------------------------------------

TR_WIDE = [(D, A, "many") for D in WIDE_D for A in WIDE_A] + [(D, A, S) for D, A in ((1, 9), (65, 16), (104, 12), (128, 16))
                                                               for S in (1, 63, 65)]


@pytest.mark.gpu
@pytest.mark.parametrize("D,A,S", TR_WIDE, ids=[f"{d}-{a}-{s}" for d, a, s in TR_WIDE])
def test_wide_trust_region_kernels_per_tensor_vs_float64(D, A, S):
    """spo_surrogate_grad, spo_fvp and spo_linesearch_eval; "many" = 128 x SMs + 37 rows (two tiles per CTA, a partial
    last tile).  obs_dim 128 / act_dim 16 is the largest FVP layout (230 272 B of shared memory)."""
    T.test_trust_region_kernels_per_tensor_vs_float64(D, A, S)


@pytest.mark.gpu
@pytest.mark.parametrize("D,A", [(104, 12), (128, 16)])
def test_wide_conjugate_gradient_equals_split_solver_bit_for_bit(D, A):
    """spo_conjugate_gradient against spo_cg_begin / spo_fvp / spo_cg_update at act_dim > 8 (S = 127: two CTAs, whose
    atomic adds into a zeroed vector commute exactly)."""
    L = T._L()
    dev = T._dev()
    S, iters = 127, 10
    flat, c, P = T.trust_case(D, A, S, 19 + A)
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
    assert torch.equal(x1, x2) and float(x1.abs().max()) > 0
    # and the solve itself: residual of (H + 0.1 I) x = b with the float64 autograd FVP
    p64 = T.unpack(flat.double(), D, A)
    r = O.fvp_autograd(p64, c["obs"].double(), x1.double().cpu()).detach() - c["v"].double()
    assert float(r.norm()) < 1e-2 * float(c["v"].norm()), float(r.norm())


# ---------------------------------------------------------------------------------------------------------------
# GPU: forward kernels (the FFMA kernel's AC = 16 instantiation) against the oracle
# ---------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("N,D,A", [(1024, 60, 12), (129, 64, 16), (300, 104, 9), (1000, 104, 12), (7, 1, 16), (200, 128, 16)])
def test_wide_rollout_step_critic_values_and_store(N, D, A):
    """Rollout step (sample, log-prob, both critics, the slot write) and bootstrap critic values; obs_dim <= 64 with
    obs_dim % 4 == 0 and >= 128 rows would take the wgmma kernel at act_dim <= 8."""
    GP.test_tensor_core_rollout_step_and_store(N, D, A)


@pytest.mark.gpu
@pytest.mark.parametrize("D,A,S", [(60, 12, 4096 + 37), (64, 16, 1500), (104, 12, 4096 + 37), (128, 9, 2048 + 5), (1, 16, 1024)])
def test_wide_actor_forward_and_kl(D, A, S):
    GP.test_tensor_core_forward_and_kl_large_batch(D, A, S)


@pytest.mark.gpu
def test_wide_forward_takes_the_ffma_kernel():
    """At obs_dim 60 / 64 (where act_dim <= 8 runs the wgmma kernel) act_dim 12 runs the FFMA kernel, for the step and the
    full-batch means alike."""
    dev = GP._cuda()
    from safepo.common.model import ActorVCritic
    from torch.profiler import ProfilerActivity, profile

    def kernels(fn):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        return [e.name for e in prof.events() if "spo_" in e.name]

    for D, A, wide in ((64, 12, True), (64, 8, False)):
        pol = ActorVCritic(D, A).to(dev)
        obs = torch.randn(4096, D, device=dev)
        names = kernels(lambda: (pol.actor_mean(obs), pol.step(obs, eps=torch.zeros(4096, A, device=dev))))
        ffma = [n for n in names if "spo_ffma_forward_kernel" in n]
        assert (len(ffma) == 2) if wide else (len(ffma) == 0), (D, A, names)


# ---------------------------------------------------------------------------------------------------------------
# GPU: trainers at the SafetyDoggoGoal1-v0 shape (obs 104, act 12) against the oracle trainer
# ---------------------------------------------------------------------------------------------------------------

TRUST = ("cpo", "trpo_lag")


@pytest.mark.gpu
@pytest.mark.parametrize("algo", ["ppo_lag", "focops", "cup", "cpo", "trpo_lag"])
def test_wide_trainer_tracks_oracle_trainer(tmp_path, algo):
    """Two epochs of the CLI entry (main) on the synthetic stream in host-RNG mode against oracle.trainers.train, with the
    bounds of test_trainer_tracks_oracle_trainer (policy-gradient family) / test_trust_region_trainer_tracks_oracle."""
    from safepo.common import synthetic_env as senv
    from safepo.utils.config import single_agent_args
    GP._cuda()
    task = "SafetyDoggoGoal1-v0"
    mod = importlib.import_module(f"safepo.single_agent.{algo}")
    N, Tn, L_ep = (5, 160, 40) if algo in TRUST else (6, 120, 40)
    extra = ["--cost-limit", "0.2"] if algo == "cup" else []
    argv = ["--seed", "3", "--num-envs", str(N), "--steps-per-epoch", str(N * Tn), "--total-steps", str(2 * N * Tn), "--task", task,
            "--rng", "host", "--gae", "exact", "--log-dir", str(tmp_path)] + extra
    args, _ = single_agent_args(argv)
    args.log_dir = str(tmp_path / "exp" / task / algo / "run")
    D, A = senv.TASK_DIMS[task]
    assert (D, A) == (104, 12)
    env = senv.SyntheticVecEnv(N, D, A, episode_len=L_ep, seed=3, stagger=True, p_terminate=0.01)
    pol, _, _, _ = mod.main(args, env=env, quiet=True)
    oargs = TR.default_args(seed=3, num_envs=N, steps_per_epoch=N * Tn, total_steps=2 * N * Tn, task=task,
                            cost_limit=args.cost_limit)
    oenv = senv.SyntheticVecEnv(N, D, A, episode_len=L_ep, seed=3, stagger=True, p_terminate=0.01)
    opol, olog, _ = TR.train(algo, oargs, oenv)
    rows = list(csv.DictReader(open(tmp_path / "exp" / task / algo / "run" / "progress.csv")))
    assert len(rows) == len(olog.rows) == 2
    for got, want in zip(rows, olog.rows):
        for k in ("Metrics/EpRet", "Metrics/EpCost", "Metrics/EpLen", "Train/Epoch", "Train/TotalSteps"):
            assert float(got[k]) == pytest.approx(float(want[k]), rel=1e-6, abs=1e-9), k
        if algo in TRUST:
            assert int(float(got["Misc/AcceptanceStep"])) == int(want["Misc/AcceptanceStep"])
            keys = ("Misc/Alpha", "Misc/xHx", "Misc/gradient_norm", "Misc/H_inv_g", "Misc/FinalStepNorm", "Loss/Loss_actor",
                    "Train/KL", "Loss/Loss_reward_critic", "Loss/Loss_cost_critic")
            for k in keys:
                assert float(got[k]) == pytest.approx(float(want[k]), rel=5e-3, abs=5e-5), (k, got[k], want[k])
        else:
            assert int(float(got["Train/StopIter"])) == int(want["Train/StopIter"])
            if "Train/LagragianMultiplier" in want:
                assert float(got["Train/LagragianMultiplier"]) == pytest.approx(float(want["Train/LagragianMultiplier"]),
                                                                                 rel=1e-5, abs=1e-8)
            for k in ("Loss/Loss_reward_critic", "Loss/Loss_cost_critic", "Loss/Loss_actor", "Train/KL"):
                assert float(got[k]) == pytest.approx(float(want[k]), rel=2e-3, abs=2e-5), (k, got[k], want[k])
    if algo not in TRUST:
        for k, v in opol.nets["actor"].items():
            assert float((pol.actor.state_dict()[k].cpu() - v.detach()).abs().max()) < 5e-3, k


@pytest.fixture(scope="module", autouse=True)
def _print_measured():
    yield
    if T.MEASURED:
        print("\nmeasured maxima at act_dim 9..16 (error / scale) vs bars:")
        for k in sorted(T.MEASURED):
            print(f"  {k:9s} {T.MEASURED[k]:.3e}   bar {WIDE_BAR[k]:.1e}")
