"""TEST INFRASTRUCTURE ONLY: the evaluation block of the single-agent scripts' main() (``--use-eval``) on top of
oracle/trainers.py, checked bit for bit against the reference's own main() (tests/golden/make_eval_golden.py ->
tests/golden/sa_eval.pt, tests/test_sa_eval.py).

``train(algo, args, env, eval_env)`` is ``oracle.trainers.train`` with the block inserted where the reference runs it: right
after the rollout, before the multiplier update (ppo_lag.py:237-269; cpo.py:315-347, focops.py:241-273 and
trpo_lag.py:325-355 are the same block), and with the three eval columns logged right after ``Metrics/EpLen``."""
from __future__ import annotations

import numpy as np
import torch

from oracle import spo_oracle as O
from oracle import trainers as TR


def episode_count(epoch, epochs):
    """ppo_lag.py:239: one episode per epoch, ten in the last epoch of the run."""
    return 1 if epoch < epochs - 1 else 10


def evaluate(pol, env, eval_env, episodes, log):
    """ppo_lag.py:241-267, quirks kept: only the reset observation comes from ``eval_env``; every step goes to the *training*
    ``env`` (ppo_lag.py:249), so the sums are per-env arrays and the episode ends on ``terminated[0] or truncated[0]``; what is
    stored is np.mean of the LAST episode's sums, not of the 50-deep deques (which nothing reads).  Returns those sums."""
    eval_rew = eval_cost = eval_len = 0.0
    for _ in range(episodes):
        eval_done = False
        eval_obs, _ = eval_env.reset()
        eval_obs = torch.as_tensor(eval_obs, dtype=torch.float32)
        eval_rew, eval_cost, eval_len = 0.0, 0.0, 0.0
        while not eval_done:
            with torch.no_grad():
                act, _, _, _ = O.policy_step(pol, eval_obs, deterministic=True)
            next_obs, reward, cost, terminated, truncated, info = env.step(act.detach().squeeze().cpu().numpy())
            eval_rew += reward
            eval_cost += cost
            eval_len += 1
            eval_done = terminated[0] or truncated[0]
            eval_obs = torch.as_tensor(next_obs, dtype=torch.float32)
    log.store(**{"Metrics/EvalEpRet": np.mean(eval_rew), "Metrics/EvalEpCost": np.mean(eval_cost),
                 "Metrics/EvalEpLen": np.mean(eval_len)})
    return eval_rew, eval_cost, eval_len


EVAL_KEYS = ("Metrics/EvalEpRet", "Metrics/EvalEpCost", "Metrics/EvalEpLen")


class _EvalStatLog(TR.StatLog):
    """StatLog that logs the eval columns where the reference does: after Metrics/EpLen (ppo_lag.py:353-359)."""

    def log_tabular(self, key, val=None):
        super().log_tabular(key, val)
        if key == "Metrics/EpLen":
            for k in EVAL_KEYS:
                super().log_tabular(k)


def train(algo, args, env, eval_env, max_epochs=None):
    """oracle.trainers.train with ``args.use_eval`` honoured.  Returns what it returns."""
    epochs = args.total_steps // args.steps_per_epoch
    inner, base_log = TR.rollout, TR.StatLog
    state = {"epoch": 0}

    def rollout_then_eval(pol, env_, buf, obs, ep, deques, log, T, epoch_T=None):
        obs = inner(pol, env_, buf, obs, ep, deques, log, T, epoch_T)
        evaluate(pol, env_, eval_env, episode_count(state["epoch"], epochs), log)
        state["epoch"] += 1
        return obs

    TR.rollout, TR.StatLog = rollout_then_eval, _EvalStatLog
    try:
        return TR.train(algo, args, env, max_epochs=max_epochs)
    finally:
        TR.rollout, TR.StatLog = inner, base_log
