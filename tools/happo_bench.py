"""Time one HAPPOTrainer.train and one MAPPOTrainer.train at config 5's shape on the device (CUDA events, after a warm-up
call): 1024 envs x 8 steps = 8192 rows, obs 398, act 20, hidden 512, the yaml's learning_iters = 5 whole-batch updates, with
and without the mamujoco mask flags.  Also times the new loss head alone.  Prints the card's name and power limit.

    python tools/happo_bench.py [--reps 5]"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "safe-policy-optimization_b200"), os.path.join(ROOT, "tools")]

import torch  # noqa: E402
from macpo_bench import power_limit, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    from safepo import _lib as L
    from safepo.common.buffer import SeparatedReplayBuffer
    from safepo.common.ma_model import HAPPOTrainer, MAPPOTrainer, MultiAgentNets
    from safepo.multi_agent import happo, mappo
    from safepo.multi_agent.mappolag import init_state
    dev = torch.device("cuda:0")
    T, E, D, A, H = 8, 1024, 398, 20, 512
    n = T * E
    res = {"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit(), "rows": n, "obs": D, "act": A, "hidden": H}
    for name, mod, cls in (("happo", happo, HAPPOTrainer), ("mappo", mappo, MAPPOTrainer)):
        for masks in (False, True):
            cfg = dict(mod.DEFAULT_CONFIG, n_rollout_threads=E, episode_length=T, use_policy_active_masks=masks, use_value_active_masks=masks)
            g = torch.Generator().manual_seed(0)
            nets = MultiAgentNets(init_state(D, H, 2, "actor", A, 1.0, 0.01, g), init_state(D, H, 2, "critic", generator=g), None, dev)
            tr = cls(nets, cfg)
            buf = SeparatedReplayBuffer(cfg, D, D, A, dev)
            buf.obs.normal_(), buf.share_obs.normal_(), buf.actions.normal_(), buf.returns.normal_()
            buf.action_log_probs.copy_(-1.0 + 0.1 * torch.randn_like(buf.action_log_probs))
            buf.active_masks.copy_((torch.rand_like(buf.active_masks) > 0.1).float())
            res[f"{name}_train_ms{'_masks' if masks else ''}"] = round(timed(lambda: tr.train(buf), args.reps), 3)
    # the loss head alone (product mode, masks): one spo_ma_ppo_actor_loss + finalize on 8192 rows
    feat, W, b, ls = torch.randn(n, H, device=dev), 0.05 * torch.randn(A, H, device=dev), torch.zeros(A, device=dev), torch.zeros(A, device=dev)
    act, old, adv, fac = torch.randn(n, A, device=dev), -torch.ones(n, A, device=dev), torch.randn(n, device=dev), torch.ones(n, device=dev)
    m = torch.ones(n, device=dev)
    ms = m.sum().reshape(1)
    dmean, imp, part = torch.empty(n, A, device=dev), torch.empty(n, device=dev), torch.empty((n + 31) // 32 * 66, device=dev)
    gb, gls, sc = torch.empty(A, device=dev), torch.empty(A, device=dev), torch.empty(3, device=dev)

    def head():
        L.check(L.lib().spo_ma_ppo_actor_loss(L.ptr(feat), n, H, L.ptr(W), L.ptr(b), L.ptr(ls), A, L.ptr(act), L.ptr(old), L.ptr(adv), None, None,
                                              L.ptr(fac), L.ptr(m), L.ptr(ms), L.MA_RATIO_PRODUCT, 0.8, 1.2, 1.0, 0.5, L.ptr(dmean), L.ptr(imp),
                                              L.ptr(part), L.stream()), "spo_ma_ppo_actor_loss")
        L.check(L.lib().spo_ma_ppo_actor_finalize(L.ptr(part), (n + 31) // 32, n, L.ptr(ms), L.MA_RATIO_PRODUCT, L.ptr(ls), A, 1.0, 0.5, 0.01,
                                                  L.ptr(gb), L.ptr(gls), L.ptr(sc), L.stream()), "spo_ma_ppo_actor_finalize")
    res["loss_head_ms"] = round(timed(head, 20), 4)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
