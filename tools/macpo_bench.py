"""Time MACPO's trust-region pieces at config 5's shape on the device (CUDA events, after warm-up): one Fisher-vector product,
one conjugate-gradient solve, one line-search trial and one whole MACPOTrainer.train, for 2 agents x 1024 envs x 8 steps
(8192 rows per agent), obs 398, act 20, hidden 512.  Prints the FVP's FLOPs from the shapes and the card's name and power limit.

    python tools/macpo_bench.py [--reps 10]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "safe-policy-optimization_b200")]

import torch  # noqa: E402


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ts = []
    for _ in range(reps):
        ev[0].record()
        fn()
        ev[1].record()
        torch.cuda.synchronize()
        ts.append(ev[0].elapsed_time(ev[1]))
    ts.sort()
    return ts[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    from safepo.common.buffer import SeparatedReplayBuffer
    from safepo.common.ma_model import MACPOTrainer, MultiAgentNets
    from safepo.multi_agent.macpo import DEFAULT_CONFIG
    from safepo.multi_agent.mappolag import init_state
    dev = torch.device("cuda:0")
    T, E, D, A, H = 8, 1024, 398, 20, 512
    n = T * E
    cfg = dict(DEFAULT_CONFIG, n_rollout_threads=E, episode_length=T)
    g = torch.Generator().manual_seed(0)
    nets = MultiAgentNets(init_state(D, H, 2, "actor", A, 1.0, 0.01, g), init_state(D, H, 2, "critic", generator=g),
                          init_state(D, H, 2, "critic", generator=g), dev)
    tr = MACPOTrainer(nets, cfg)
    obs = torch.randn(n, D, generator=g).to(dev)
    mean_old = tr.actor_forward(obs)
    P = tr.P
    v = torch.randn(P, device=dev) * 1e-2
    v[nets.actor.flat == 0] = 0            # keeps the padding (and, harmlessly for a timing, the zero-initialised biases) at 0
    out = torch.empty_like(v)
    x = torch.empty_like(v)
    t_fvp = timed(lambda: tr.fvp(v, out), args.reps)
    t_cg = timed(lambda: tr.conjugate_gradient(v, x), max(3, args.reps // 3))
    act = torch.randn(n, A, device=dev) * 0.3
    old_lp = torch.randn(n, A, device=dev) * 0.1 - 0.5
    adv, cadv, fac = torch.randn(n, device=dev), torch.randn(n, device=dev), torch.ones(n, device=dev)
    tr.old_flat.copy_(nets.actor.flat)
    res = torch.zeros(8, device=dev)

    from safepo import _lib as L
    tr._v["x"].copy_(v)

    def trial():               # exactly the launches of one trial in MACPOTrainer.trpo_update, and its 8-float read
        L.check(L.lib().spo_ma_dots(L.ptr(tr._v["x"]), L.ptr(tr._v["x"]), None, None, None, None, None, None, 1, P, L.ptr(tr._work),
                                    L.ptr(res[5:]), L.stream()), "spo_ma_dots")
        L.check(L.lib().spo_ma_ls_trial(L.ptr(tr.old_flat), L.ptr(tr._v["x"]), L.ptr(res[5:]), 0.05, L.ptr(nets.actor.flat), P, L.stream()),
                "spo_ma_ls_trial")
        tr.linesearch_eval(obs, mean_old, act, old_lp, adv, cadv, fac, res)
        res.cpu()
    t_ls = timed(trial, args.reps)
    nets.actor.flat.copy_(tr.old_flat)
    buf = SeparatedReplayBuffer(cfg, D, D, A, dev)
    buf.obs.copy_(torch.randn(T + 1, E, D, device=dev))
    buf.share_obs.copy_(buf.obs)
    buf.actions.copy_(torch.randn(T, E, A, device=dev) * 0.3)
    buf.action_log_probs.copy_(torch.randn(T, E, A, device=dev) * 0.1 - 0.5)
    buf.returns.copy_(torch.randn(T + 1, E, 1, device=dev))
    buf.cost_returns.copy_(torch.randn(T + 1, E, 1, device=dev).abs() * 30)
    buf.return_aver_insert(torch.tensor(30.0))
    t_train = timed(lambda: tr.train(buf), max(3, args.reps // 3))
    K0, K = D, H
    flops = 2 * n * (2 * K0 * H + 2 * 2 * K * H + 2 * A * H)          # JVP: dx W^T + x dW^T per layer, mean layer
    flops += 2 * n * (2 * K0 * H + 2 * 2 * K * H + 2 * A * H)         # VJP: dW = dz^T x and dx = dz W per layer, mean layer
    print(json.dumps(dict(gpu=torch.cuda.get_device_name(0), power_limit=power_limit(), rows=n, params=P, fvp_flops=flops,
                          fvp_ms=round(t_fvp, 4), fvp_tflops=round(flops / t_fvp / 1e9, 2), cg_solve_ms=round(t_cg, 3),
                          linesearch_trial_ms=round(t_ls, 4), train_ms=round(t_train, 3))))


if __name__ == "__main__":
    main()
