"""--use-eval in the single-agent trainers and safepo.evaluate (saved runs, single- and multi-agent).

CPU: the evaluation oracle (tests/sa_eval_oracle.py) against the reference's own main() with ``use_eval=True``
(tests/golden/sa_eval.pt), the engine's evaluation host logic against that oracle, checkpoint selection, state-dict checks and
the eval_result.txt line.  GPU: main() of the four algorithms with --use-eval against the fixture, a CLI run evaluated with
``python -m safepo.evaluate`` against the reference's eval_single_agent, and a multi-agent run directory."""
import csv
import json
import os
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import sa_eval_oracle as EO
from oracle import spo_oracle as O
from oracle import trainers as TR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "safe-policy-optimization_b200")


def _senv():
    from safepo.common import synthetic_env
    return synthetic_env


def _num(v):
    # cpo logs Train/KL as a fp32 tensor (cpo.py:529): the csv holds its repr
    return float(v.replace("tensor(", "").rstrip(")")) if isinstance(v, str) else float(v)


def _envs(run):
    senv = _senv()
    a = run["args"]
    D, A = senv.TASK_DIMS[a["task"]]
    env = senv.SyntheticVecEnv(a["num_envs"], D, A, seed=a["seed"], **run["env"])
    eval_env = senv.SyntheticVecEnv(1, D, A, seed=0, **run["env"])       # make_sa_mujoco_env(num_envs=1, seed=None)
    return env, eval_env


def _check_columns(got, want):
    """The same columns as the reference, the episode and eval columns first and in its order (the order of the later
    columns is the trainers' own, unchanged by the evaluation)."""
    assert set(got) == set(want)
    assert got[:6] == want[:6] == ["Metrics/EpRet", "Metrics/EpCost", "Metrics/EpLen", "Metrics/EvalEpRet", "Metrics/EvalEpCost",
                                   "Metrics/EvalEpLen"]


CASES = [(algo, n) for algo in ("ppo_lag", "focops", "cpo", "trpo_lag") for n in (1, 3)]


# ---------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------

@pytest.mark.parametrize("algo,n", CASES)
def test_eval_oracle_matches_reference_main(golden, algo, n):
    """The oracle's main() with the evaluation block against the reference's, every logged number bit for bit, the eval
    columns where the reference puts them."""
    run = golden("sa_eval")["runs"][algo][n]
    env, eval_env = _envs(run)
    _, log, _ = EO.train(algo, TR.default_args(**run["args"]), env, eval_env)
    assert len(log.rows) == len(run["rows"])
    _check_columns([k for k in log.log_headers if not k.startswith("Time/")], list(run["rows"][0].keys()))
    for got, want in zip(log.rows, run["rows"]):
        for k, v in want.items():
            g, w = float(got[k]), _num(v)
            assert g == w or np.float32(g) == np.float32(w) or (np.isnan(g) and np.isnan(w)), (algo, n, k, g, w)


def test_fixture_steps_the_training_env_across_episode_ends(golden):
    """The fixture exercises what it is for: evaluations that last longer than the time to the next episode end of some
    training env (3 envs) and per-env sums whose mean is not one env's value."""
    runs = golden("sa_eval")["runs"]
    lens = [float(r["Metrics/EvalEpLen"]) for a in runs for r in runs[a][3]["rows"]]
    assert max(lens) > 1
    costs = [float(r["Metrics/EvalEpCost"]) for a in runs for r in runs[a][3]["rows"]]
    assert any(0 < c < 1 for c in costs)            # a third or two thirds: the mean over the three envs


class _Policy:
    """ActorVCritic.step on the oracle's CPU arithmetic: the evaluation's host logic is what is tested here."""

    def __init__(self, opol):
        self.opol = opol

    def step(self, obs, deterministic=False):
        assert deterministic
        with torch.no_grad():
            return O.policy_step(self.opol, obs, deterministic=True)


@pytest.mark.parametrize("n", [1, 3])
def test_engine_evaluation_matches_oracle(n):
    """safepo.single_agent._engine.Evaluation against the oracle's block: the logged columns, the returned sums and the state of
    the training env afterwards (which env was stepped, how far)."""
    from safepo.single_agent._engine import Evaluation, eval_episode_count
    senv = _senv()
    D, A = senv.TASK_DIMS["SafetyPointGoal1-v0"]
    kw = dict(episode_len=9, stagger=True, p_terminate=0.05)
    torch.manual_seed(1)
    opol = O.OraclePolicy(D, A, [64, 64])
    logs = []
    envs = []
    for engine in (True, False):
        env, eval_env = senv.SyntheticVecEnv(n, D, A, seed=4, **kw), senv.SyntheticVecEnv(1, D, A, seed=0, **kw)
        for _ in range(5):
            env.step(None)
        log = TR.StatLog()
        sums = []
        for epoch in range(3):
            episodes = eval_episode_count(epoch, 3)
            if engine:
                roll = SimpleNamespace(policy=_Policy(opol), env=env, logger=log, obs_norm=None, act_rescale=None, D=D)
                sums.append(Evaluation(roll, eval_env, "cpu").run(episodes))
            else:
                sums.append(EO.evaluate(opol, env, eval_env, episodes, log))
        logs.append((log.epoch_dict, sums))
        envs.append((env._k, env._age.copy()))
    (got, gs), (want, ws) = logs
    assert set(got) == set(EO.EVAL_KEYS) == set(want)
    for k in EO.EVAL_KEYS:
        assert got[k] == want[k], k
    for g, w in zip(gs, ws):
        for a, b in zip(g, w):
            assert np.array_equal(np.asarray(a), np.asarray(b))
    assert envs[0][0] == envs[1][0] and np.array_equal(envs[0][1], envs[1][1])
    assert envs[0][0] > 5 + 1 + 1 + 10      # every episode took at least one step of the training env


def test_eval_columns_are_logged_only_with_use_eval():
    """Off means unchanged: without an evaluation the loops log exactly the columns they logged before, and Time/Total is
    the same sum; with one the columns sit where the reference puts them (ppo_lag.py:353-373)."""
    from safepo.single_agent._engine import _log_metrics, _log_times

    class Rec:
        def __init__(self):
            self.keys, self.vals = [], {}

        def log_tabular(self, k, v=None):
            self.keys.append(k)
            self.vals[k] = v

    off, on = Rec(), Rec()
    for rec, ev in ((off, None), (on, object())):
        _log_metrics(rec, ev)
        _log_times(rec, ev, 0.25, 0.0 if ev is None else 0.5, 1.125)
    assert off.keys == ["Metrics/EpRet", "Metrics/EpCost", "Metrics/EpLen", "Time/Rollout", "Time/Update", "Time/Total"]
    assert off.vals["Time/Total"] == 0.25 + 1.125
    assert on.keys == ["Metrics/EpRet", "Metrics/EpCost", "Metrics/EpLen", "Metrics/EvalEpRet", "Metrics/EvalEpCost",
                       "Metrics/EvalEpLen", "Time/Rollout", "Time/Eval", "Time/Update", "Time/Total"]
    assert on.vals["Time/Eval"] == 0.5 and on.vals["Time/Total"] == 0.25 + 0.5 + 1.125


def test_checkpoint_selection_is_the_references_string_sort(tmp_path):
    """sorted(...)[-1] (evaluate.py:36,41): model99.pt after model100.pt, state99.pkl after state100.pkl."""
    from safepo import evaluate as E
    from safepo._lib import SpoError
    (tmp_path / "torch_save").mkdir()
    for name in ("model0.pt", "model100.pt", "model99.pt", "notes.txt"):
        (tmp_path / "torch_save" / name).write_bytes(b"")
    for name in ("state0.pkl", "state100.pkl", "state99.pkl"):
        (tmp_path / name).write_bytes(b"")
    assert os.path.basename(E._last(str(tmp_path / "torch_save"), ".pt")) == "model99.pt"
    assert os.path.basename(E._last(str(tmp_path), ".pkl")) == "state99.pkl"
    with pytest.raises(SpoError, match="no \\*.pt"):
        E._last(str(tmp_path / "missing"), ".pt")


def test_bad_checkpoints_raise_spo_error_naming_the_key(tmp_path):
    import joblib
    from safepo import evaluate as E
    from safepo._lib import SpoError
    from safepo.common.model import ActorVCritic
    from safepo.common.normalizer import HostRunningMeanStd
    torch.manual_seed(0)
    pol = ActorVCritic(60, 2)                      # state_dict shapes only: nothing here touches a device
    good = {k: v.clone() for k, v in pol.actor.state_dict().items()}
    cases = {"missing": ({k: v for k, v in good.items() if k != "mean.2.bias"}, "missing key 'mean.2.bias'"),
             "shape": (dict(good, **{"mean.0.weight": torch.zeros(64, 59)}), "'mean.0.weight' has shape \\(64, 59\\)"),
             "extra": (dict(good, bogus=torch.zeros(1)), "unexpected key 'bogus'")}
    for name, (sd, msg) in cases.items():
        path = tmp_path / f"{name}.pt"
        torch.save(sd, path)
        with pytest.raises(SpoError, match=msg):
            E._load_actor(pol, str(path))
    path = tmp_path / "good.pt"
    torch.save({k: v + 1 for k, v in good.items()}, path)
    E._load_actor(pol, str(path))
    assert torch.equal(pol.actor.log_std.detach(), good["log_std"] + 1)
    joblib.dump({"Other": 1}, tmp_path / "state0.pkl")
    with pytest.raises(SpoError, match="missing key 'Normalizer'"):
        E._load_normalizer(str(tmp_path / "state0.pkl"), 60, "cpu")
    joblib.dump({"Normalizer": HostRunningMeanStd((59,))}, tmp_path / "state1.pkl")
    with pytest.raises(SpoError, match="Normalizer.mean has shape \\(59,\\)"):
        E._load_normalizer(str(tmp_path / "state1.pkl"), 60, "cpu")


def test_benchmark_eval_writes_the_references_line(tmp_path, monkeypatch):
    """benchmark_eval over a runs/<env>/<algo>/<seed> tree: one line per (env, algo) in the format of evaluate.py:179-184,
    default save directory runs -> results."""
    from safepo import evaluate as E
    bench = tmp_path / "runs" / "exp"
    pairs = {("SafetyPointGoal1-v0", "ppo_lag"): [(1.234, 10.0), (2.0, 30.0)], ("SafetyPointGoal1-v0", "cpo"): [(-0.5, 0.0)],
             ("SafetyCarButton1-v0", "focops"): [(0.125, 2.5), (0.375, 7.5), (0.25, 5.0)]}
    lookup = {}
    for (env, algo), runs in pairs.items():
        for i, pair in enumerate(runs):
            d = bench / env / algo / f"seed-{i:03d}-x"
            d.mkdir(parents=True)
            lookup[str(d)] = pair
    monkeypatch.setattr(E, "single_runs_eval", lambda d, n: lookup[d])
    E.benchmark_eval(["--benchmark-dir", str(bench), "--eval-episodes", "4"])
    lines = open(tmp_path / "results" / "exp" / "eval_result.txt").read().splitlines(keepends=True)
    want = []
    for env in sorted({e for e, _ in pairs}):
        for algo in sorted(a for e, a in pairs if e == env):
            r, c = zip(*pairs[(env, algo)])
            want.append(f"After 4 episodes evaluation, the {algo} in {env} evaluation reward: {round(np.mean(r), 2)}±"
                        f"{round(np.std(r), 2)}, cost: {round(np.mean(c), 2)}±{round(np.std(c), 2)} \n")
    assert lines == want
    assert lines[0] == "After 4 episodes evaluation, the focops in SafetyCarButton1-v0 evaluation reward: 0.25±0.1, cost: 5.0±2.04 \n"


def test_run_dispatch_and_unknown_multi_agent_algorithm(tmp_path, monkeypatch):
    from safepo import evaluate as E
    from safepo._lib import SpoError
    (tmp_path / "config.json").write_text(json.dumps({"algorithm_name": "mappolag", "seed": 0}))
    monkeypatch.setattr(E, "eval_multi_agent", lambda d, n: ("ma", n))
    monkeypatch.setattr(E, "eval_single_agent", lambda d, n: ("sa", n))
    assert E.single_runs_eval(str(tmp_path), 2) == ("ma", 2)
    (tmp_path / "config.json").write_text(json.dumps({"task": "SafetyPointGoal1-v0", "seed": 0}))
    assert E.single_runs_eval(str(tmp_path), 2) == ("sa", 2)
    monkeypatch.undo()
    (tmp_path / "config.json").write_text(json.dumps({"algorithm_name": "qmix", "seed": 0}))
    with pytest.raises(SpoError, match="'qmix'"):
        E.eval_multi_agent(str(tmp_path), 1)
    with pytest.raises(SpoError, match="no config.json"):
        E.eval_multi_agent(str(tmp_path / "nowhere"), 1)


# ---------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("algo,n", CASES)
def test_main_with_use_eval_tracks_reference(golden, tmp_path, algo, n):
    """main() with --use-eval True in host-RNG mode against the reference's main(), with the bars of
    test_gpu_parity.py's trainer tests; the eval columns are sums of the env's float64 rewards like Metrics/EpRet."""
    import importlib
    from safepo.utils.config import single_agent_args
    run = golden("sa_eval")["runs"][algo][n]
    a = run["args"]
    argv = ["--seed", str(a["seed"]), "--task", a["task"], "--num-envs", str(n), "--steps-per-epoch", str(a["steps_per_epoch"]),
            "--total-steps", str(a["total_steps"]), "--use-eval", "True", "--rng", "host", "--gae", "exact", "--log-dir", str(tmp_path)]
    args, _ = single_agent_args(argv)
    args.log_dir = str(tmp_path / "run")
    env, _ = _envs(run)
    importlib.import_module(f"safepo.single_agent.{algo}").main(args, env=env, quiet=True)
    with open(tmp_path / "run" / "progress.csv") as f:
        rows = list(csv.DictReader(f))
    assert len(rows) == len(run["rows"])
    _check_columns([k for k in rows[0] if not k.startswith("Time/")], list(run["rows"][0].keys()))
    assert "Time/Eval" in rows[0]
    trust = algo in ("cpo", "trpo_lag")
    for got, want in zip(rows, run["rows"]):
        for k in ("Metrics/EpRet", "Metrics/EpCost", "Metrics/EpLen") + EO.EVAL_KEYS + ("Train/Epoch", "Train/TotalSteps"):
            assert float(got[k]) == pytest.approx(_num(want[k]), rel=1e-6, abs=1e-9), k
        if "Train/LagragianMultiplier" in want:
            assert float(got["Train/LagragianMultiplier"]) == pytest.approx(_num(want["Train/LagragianMultiplier"]), rel=1e-5, abs=1e-8)
        if trust:
            assert int(float(got["Misc/AcceptanceStep"])) == int(_num(want["Misc/AcceptanceStep"]))
            keys, rel, abs_ = ("Misc/Alpha", "Misc/xHx", "Misc/gradient_norm", "Misc/H_inv_g", "Misc/FinalStepNorm", "Loss/Loss_actor",
                               "Train/KL", "Loss/Loss_reward_critic", "Loss/Loss_cost_critic"), 5e-3, 5e-5
        else:
            assert int(float(got["Train/StopIter"])) == int(_num(want["Train/StopIter"]))
            assert float(got["Train/LR"]) == pytest.approx(_num(want["Train/LR"]), rel=1e-6, abs=1e-9)
            keys, rel, abs_ = ("Loss/Loss_reward_critic", "Loss/Loss_cost_critic", "Loss/Loss_actor", "Train/KL"), 2e-3, 2e-5
        for k in keys:
            assert float(got[k]) == pytest.approx(_num(want[k]), rel=rel, abs=abs_), (k, got[k], want[k])


def _run(cmd, cwd):
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([PKG, ROOT]))
    r = subprocess.run([sys.executable] + cmd, cwd=cwd, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return r.stdout


@pytest.mark.gpu
def test_cli_run_then_evaluate_returns_the_references_pair(golden, tmp_path):
    """A short ppo_lag CLI run with the fixture's settings, then ``python -m safepo.evaluate --benchmark-dir``: the run
    directory evaluates to the pair the reference's eval_single_agent returned on its own run directory."""
    from safepo import evaluate as E
    ref = golden("sa_eval")["single_agent"]
    a = ref["args"]
    _run(["-m", "safepo.single_agent.ppo_lag", "--seed", str(a["seed"]), "--num-envs", str(a["num_envs"]),
          "--steps-per-epoch", str(a["steps_per_epoch"]), "--total-steps", str(a["total_steps"]), "--env", a["env"],
          "--episode-len", str(a["episode_len"]), "--log-dir", str(tmp_path / "runs")], tmp_path)
    algo_dir = tmp_path / "runs" / "single_agent_exp" / "SafetyPointGoal1-v0" / "ppo_lag"
    (run_dir,) = list(algo_dir.iterdir())
    assert {"config.json", "progress.csv", "state0.pkl", "torch_save"} <= set(os.listdir(run_dir))
    out = _run(["-m", "safepo.evaluate", "--benchmark-dir", str(tmp_path / "runs" / "single_agent_exp"),
                "--eval-episodes", str(ref["eval_episodes"])], tmp_path)
    line = open(tmp_path / "results" / "single_agent_exp" / "eval_result.txt").read()
    assert line == E.result_line(ref["eval_episodes"], "ppo_lag", "SafetyPointGoal1-v0", [ref["reward"]], [ref["cost"]]), (line, out)
    reward, cost = E.eval_single_agent(str(run_dir), ref["eval_episodes"])
    assert reward == pytest.approx(ref["reward"], rel=1e-12, abs=1e-15) and cost == ref["cost"]


@pytest.mark.gpu
def test_normalised_run_installs_its_statistics(tmp_path):
    """A run trained with --normalize-obs: eval_single_agent installs the saved Normalizer (its statistics, not fresh ones)."""
    from safepo import evaluate as E
    from safepo.common import normalizer as N
    seen = []
    real = N.SafeNormalizeObservation.normalize

    def spy(self, obs, update=True, out=None):
        if not seen:
            seen.append((self.obs_rms.mean.cpu().numpy().copy(), self.obs_rms.count))
        return real(self, obs, update, out)
    _run(["-m", "safepo.single_agent.ppo_lag", "--num-envs", "2", "--steps-per-epoch", "40", "--total-steps", "80",
          "--episode-len", "9", "--normalize-obs", "--log-dir", str(tmp_path / "runs")], tmp_path)
    (run_dir,) = list((tmp_path / "runs" / "single_agent_exp" / "SafetyPointGoal1-v0" / "ppo_lag").iterdir())
    import joblib
    saved = joblib.load(os.path.join(run_dir, "state0.pkl"))["Normalizer"]
    N.SafeNormalizeObservation.normalize = spy
    try:
        E.eval_single_agent(str(run_dir), 1)
    finally:
        N.SafeNormalizeObservation.normalize = real
    np.testing.assert_array_equal(seen[0][0], saved.mean)
    assert seen[0][1] == saved.count and saved.count > 1


@pytest.mark.gpu
@pytest.mark.parametrize("algo", ["mappolag", "macpo"])
def test_multi_agent_run_directory_evaluates(tmp_path, algo):
    """A multi-agent CLI run writes config.json; eval_multi_agent (and benchmark_eval) restore models_seed{seed} and return
    what the CLI's own --model-dir evaluation returns."""
    import importlib
    from safepo import evaluate as E
    mod = importlib.import_module(f"safepo.multi_agent.{algo}")
    sizes = ["--num-envs", "8", "--num-agents", "2", "--obs-dim", "10", "--share-obs-dim", "14", "--act-dim", "3",
             "--hidden-size", "128", "--episode-len", "4", "--seed", "0"]
    run_dir = tmp_path / "runs" / "synthetic" / algo / "seed0"
    mod.main(sizes + ["--iterations", "2", "--log-dir", str(run_dir)])
    cfg = json.load(open(run_dir / "config.json"))
    assert cfg["algorithm_name"] == algo and cfg["hidden_size"] == 128
    got = E.eval_multi_agent(str(run_dir), 2)
    (row,) = mod.main(sizes + ["--model-dir", str(run_dir / "models_seed0"), "--eval-episodes", "2"])
    assert float(got[0]) == row["Eval/EpRet"] and float(got[1]) == row["Eval/EpCost"]
    E.benchmark_eval(["--benchmark-dir", str(tmp_path / "runs"), "--eval-episodes", "2", "--save-dir", str(tmp_path)])
    assert open(tmp_path / "eval_result.txt").read() == E.result_line(2, algo, "synthetic", [got[0]], [got[1]])
