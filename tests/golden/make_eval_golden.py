"""Generate tests/golden/sa_eval.pt from the REAL reference: ``--use-eval True`` in the single-agent scripts' main() and
safepo/evaluate.py's eval_single_agent.

Runs only where the reference tree is available (read-only); reuses make_golden.py's import shims.  Stored:

* ``runs[algo][num_envs]``: main() of ppo_lag / focops / cpo / trpo_lag with ``use_eval=True`` on the synthetic vector env,
  1 and 3 envs (3 exercises the per-env sums of the evaluation, which steps the training env), episodes short enough that
  every evaluation steps the training env across episode ends; every progress.csv value that is not a time.
* ``single_agent``: eval_single_agent on the run directory of one ppo_lag run, and the returned (reward, cost) pair.

    python tests/golden/make_eval_golden.py
"""
from __future__ import annotations

import csv
import importlib
import importlib.util
import os
import sys
import tempfile

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)

from make_golden import import_reference  # noqa: E402

CFGS = {
    "ppo_lag": dict(seed=3, task="SafetyPointGoal1-v0", episode_len=13, T=40),
    "focops": dict(seed=4, task="SafetyPointGoal1-v0", episode_len=11, T=45),
    "cpo": dict(seed=5, task="SafetyCarButton1-v0", episode_len=12, T=40),
    "trpo_lag": dict(seed=6, task="SafetyPointGoal1-v0", episode_len=14, T=50),
}
EPOCHS = 3
EVAL_EPISODES = 3


def _synthetic_env_module():
    spec = importlib.util.spec_from_file_location(
        "spo_synthetic_env", os.path.join(ROOT, "safe-policy-optimization_b200", "safepo", "common", "synthetic_env.py"))
    senv = importlib.util.module_from_spec(spec)
    sys.modules["spo_synthetic_env"] = senv          # so that the logger can pickle the env's obs_rms (state*.pkl)
    spec.loader.exec_module(senv)
    return senv


def run_main(ref, senv, algo, args_kw, env_kw):
    from oracle.trainers import default_args
    mod = ref[algo]
    args = default_args(**args_kw)
    args.log_dir = os.path.join(tempfile.mkdtemp(), "exp", args.task, algo, "run")
    D, A = senv.TASK_DIMS[args.task]

    def fake_make(num_envs, env_id, seed=None):
        env = senv.SyntheticVecEnv(num_envs, D, A, seed=0 if seed is None else seed, **env_kw)
        return env, env.observation_space, env.action_space

    mod.make_sa_mujoco_env = fake_make
    mod.main(args, {})
    with open(os.path.join(args.log_dir, "progress.csv")) as f:
        rows = [{k: v for k, v in r.items() if not k.startswith("Time/")} for r in csv.DictReader(f)]
    return args.log_dir, rows, fake_make


def main():
    ref = import_reference()
    senv = _synthetic_env_module()
    runs = {}
    for algo, c in CFGS.items():
        runs[algo] = {}
        for N in (1, 3):
            T = c["T"]
            akw = dict(seed=c["seed"], task=c["task"], num_envs=N, steps_per_epoch=N * T, total_steps=N * T * EPOCHS, use_eval=True)
            ekw = dict(episode_len=c["episode_len"], stagger=True, p_terminate=0.02)
            _, rows, _ = run_main(ref, senv, algo, akw, ekw)
            assert len(rows) == EPOCHS and all("Metrics/EvalEpRet" in r for r in rows), (algo, N)
            runs[algo][N] = dict(args=akw, env=ekw, rows=rows)
            print(algo, N, [r["Metrics/EvalEpRet"] for r in rows])
    # eval_single_agent on a run whose config names the synthetic env the way the CLI records it (--env, --episode-len)
    akw = dict(seed=2, num_envs=3, steps_per_epoch=3 * 30, total_steps=3 * 30 * 2, env="synthetic", episode_len=17)
    run_dir, _, fake_make = run_main(ref, senv, "ppo_lag", akw, dict(episode_len=17))
    evaluate = importlib.import_module("safepo.evaluate")
    evaluate.make_sa_mujoco_env = fake_make
    pair = evaluate.eval_single_agent(run_dir, EVAL_EPISODES)
    single = dict(args=akw, eval_episodes=EVAL_EPISODES, files=sorted(os.listdir(run_dir)), reward=float(pair[0]), cost=float(pair[1]))
    print("eval_single_agent", single)
    path = os.path.join(HERE, "sa_eval.pt")
    torch.save({"runs": runs, "epochs": EPOCHS, "single_agent": single}, path)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
