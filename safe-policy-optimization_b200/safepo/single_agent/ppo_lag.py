"""PPO-Lagrangian on the libspo kernels.

CLI-compatible with the reference's safepo/single_agent/ppo_lag.py (same flags, same
``default_cfg``, same ``main(args, cfg_env)`` entry, same progress.csv columns); the
rollout -> dual GAE -> clipped-surrogate update path runs as hand-written sm_90a
kernels (see safepo/single_agent/_engine.py).

    python -m safepo.single_agent.ppo_lag --task SafetyPointGoal1-v0 --num-envs 1024 \
        --steps-per-epoch 1024000 --total-steps 10240000
"""
from __future__ import annotations

from safepo.single_agent._engine import run_policy_gradient

default_cfg = {
    "hidden_sizes": [64, 64],
    "gamma": 0.99,
    "target_kl": 0.02,
    "batch_size": 64,
    "learning_iters": 40,
    "max_grad_norm": 40.0,
}


def main(args, cfg_env=None, env=None, max_epochs=None, quiet=False):
    return run_policy_gradient(args, dict(default_cfg), "ppo_lag", env=env, max_epochs=max_epochs, quiet=quiet)


if __name__ == "__main__":
    from safepo.single_agent._cli import launch

    launch(main, __file__)
