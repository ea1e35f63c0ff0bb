"""Per-phase cycle breakdown of one spo_update_kernel pass (needs tools/libspo_timers.so:
`python safe-policy-optimization_b200/build.py --timers`)."""
import ctypes as C
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "safe-policy-optimization_b200"))
from safepo import _lib as L  # noqa: E402

L.LIB_PATH = os.path.join(ROOT, "tools", "libspo_timers.so")
from safepo.single_agent._engine import PolicyGradientUpdate  # noqa: E402
from safepo.common.model import ActorVCritic  # noqa: E402

dev = torch.device("cuda:0")
S, D, A = int(os.environ.get("S", 1024000)), 60, 2
steps = min(int(os.environ.get("STEPS", 4000)), S // 64)
torch.manual_seed(0)
pol = ActorVCritic(D, A).to(dev)
data = {"obs": torch.randn(S, D, device=dev), "act": torch.randn(S, A, device=dev), "log_prob": torch.full((S,), -2.5, device=dev),
        "target_value_r": torch.randn(S, device=dev), "target_value_c": torch.randn(S, device=dev), "adv": torch.randn(S, device=dev)}
cfg = dict(hidden_sizes=[64, 64], gamma=0.99, target_kl=1e9, batch_size=64, learning_iters=1, max_grad_norm=40.0)
upd = PolicyGradientUpdate(pol, cfg, L.LOSS_PPO_CLIP, epochs=100, host_rng=False, device=dev)
perm = torch.randperm(S, device=dev)[: steps * 64]
upd.run(data, perms=[perm])
torch.cuda.synchronize()
lib = L.lib()
buf = (C.c_ulonglong * (16 * 24))()
lib.spo_debug_phase_cycles.argtypes = [C.c_void_p, C.c_int]
lib.spo_debug_phase_cycles(buf, 1)
upd.run(data, perms=[perm])
torch.cuda.synchronize()
lib.spo_debug_phase_cycles(buf, 1)
names = {0: "top (slot wait+sync)", 2: "L1 GEMM+tanh", 9: "norm wait", 1: "resolve clip", 19: "h1 push+Adam W2..log_std",
         3: "lsc+adk+h1 wait", 4: "L2+ypartial", 5: "barrier 2", 6: "y pull+loss rows", 7: "dz2", 8: "dh1 partial+push",
         10: "loss sum+dW2+db2", 20: "dW3/db3/dlog_std", 11: "dh1 wait+reduce+dz1", 12: "dW1+db1", 13: "dp exchange",
         14: "reg+sumsq", 17: "norm push", 16: "Adam W1/b1+save"}
for rank in range(12):
    row = [buf[rank * 24 + i] / steps for i in range(24)]
    row_n = [(names[i], row[i]) for i in names]
    net = ("actor", "reward critic", "cost critic")[rank // 4]
    print(f"{net:13s} q{rank % 4} total {sum(row):7.0f} cyc/step | " + " ".join(f"{n}={v:.0f}" for n, v in row_n))
