"""Time PPO-Lag and CPO at the Doggo shape (SafetyDoggoGoal1-v0: obs 104, act 12; 1024 envs, T = 1000, the synthetic
stream of bench.py) against the same obs at act 8, alternating the two shapes epoch by epoch so that both see the same
card state.  act 12 runs the kernels' AC = 16 instantiations, act 8 the AC = 8 ones; the difference is what the wider
action capacity costs.

Per shape and algorithm: the median over --reps epochs of the whole epoch (rollout, GAE, update) in env-steps/s, and of the
update alone in microseconds per minibatch step (PPO-Lag: spo_pg_update passes, PPO clip + both critics; CPO: the critic
regression's minibatch steps, the trust-region part reported per call).  Prints the card's name and power limit.

    python tools/wide_act_bench.py [--reps 5] [--warmup 2]"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "safe-policy-optimization_b200"), os.path.join(ROOT, "tools")]

import torch  # noqa: E402

import bench  # noqa: E402
from macpo_bench import power_limit  # noqa: E402


def build(algo, D, A, envs, horizon):
    name = f"{algo}_{D}_{A}"
    bench.WORKLOADS[name] = dict(bench.WORKLOADS[algo], D=D, A=A, envs=envs,
                                 task="SafetyDoggoGoal1-v0" if A == 12 else bench.WORKLOADS[algo]["task"])
    bench.select_workload(name)
    args = argparse.Namespace(num_envs=envs, horizon=horizon)
    return bench.build_trainer(args, torch.device("cuda:0"), 0, resident=True)


def timed_epoch(tr):
    """One epoch (bench.one_epoch) and, on the batch it produced, the update part once more on its own."""
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    ev[0].record()
    bench.one_epoch(tr)
    ev[1].record()
    data, _ = tr["last"]
    ev[2].record()
    if tr["algo"] == "cpo":
        tr["trust"].run_cpo(data, 0.0)
        ev[3].record()
        torch.cuda.synchronize()
        t_trust = ev[2].elapsed_time(ev[3])
        ev[2].record()
        c = tr["critics"].run(data)
        ev[3].record()
        torch.cuda.synchronize()
        return ev[0].elapsed_time(ev[1]), ev[2].elapsed_time(ev[3]), c["steps"], t_trust
    u = tr["upd"].run(data)
    ev[3].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]), ev[2].elapsed_time(ev[3]), u["steps"], None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--envs", type=int, default=1024)
    ap.add_argument("--horizon", type=int, default=1000)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs the GPU"
    out = {"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit(), "envs": args.envs, "horizon": args.horizon,
           "obs": 104}
    for algo in ("ppo_lag", "cpo"):
        trs = {A: build(algo, 104, A, args.envs, args.horizon) for A in (12, 8)}
        for _ in range(args.warmup):
            for A, tr in trs.items():
                timed_epoch(tr)
        rec = {A: [] for A in trs}
        for _ in range(args.reps):
            for A, tr in trs.items():             # alternate the two shapes
                rec[A].append(timed_epoch(tr))
        for A, rs in rec.items():
            med = lambda xs: sorted(xs)[len(xs) // 2]
            ep_ms = med([r[0] for r in rs])
            per_step = med([1e3 * r[1] / max(r[2], 1) for r in rs])
            key = f"{algo}_act{A}"
            out[f"{key}_env_steps_per_s"] = round(args.envs * args.horizon / (ep_ms / 1e3))
            out[f"{key}_epoch_ms"] = round(ep_ms, 2)
            out[f"{key}_us_per_minibatch_step"] = round(per_step, 3)
            out[f"{key}_minibatch_steps"] = med([r[2] for r in rs])
            if algo == "cpo":
                out[f"{key}_trust_region_ms"] = round(med([r[3] for r in rs]), 3)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
