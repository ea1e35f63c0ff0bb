"""Where the minibatch update kernel runs each part of its Adam step.

W1 / b1 get their Adam step at the end of a minibatch step, speculatively with clip = 1, and are undone and redone at the
top of the next step when the joint norm turns out above max_grad_norm.  W2, b2, W3, b3 and log_std get theirs in the first
tile of the next step, with the actual clip; the last step of a launch does both in the launch's epilogue.  These tests pin
those paths against the oracle, with the clip pattern of every step chosen by the data: the rows of the "hot" steps carry
reward targets 100x the others, which puts their joint norm far above max_grad_norm while the other steps stay below it.
Every case runs two launches (two passes), so that the Adam moments the first launch writes back are used by the second."""
import pytest
import torch

from oracle import spo_oracle as O

pytestmark = pytest.mark.gpu


def _cuda():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    return torch.device("cuda:0")


def _policy_state(pol):
    return {n: {k: v.detach().cpu().clone() for k, v in getattr(pol, n).state_dict().items()}
            for n in ("actor", "reward_critic", "cost_critic")}


def _close(got, want, rtol, atol):
    got, want = torch.as_tensor(got).double(), torch.as_tensor(want).double()
    err = (got - want).abs()
    return bool((err <= atol + rtol * want.abs()).all()), float(err.max())


def _data(D, A, S, opol, hot_rows, seed):
    g = torch.Generator().manual_seed(seed)
    obs = torch.randn(S, D, generator=g)
    with torch.no_grad():
        mean, std = O.actor_mean_std(opol, obs)
        act = mean + std * torch.randn(S, A, generator=g)
        logp = O.normal_log_prob(act, mean, std).sum(-1) + 0.05 * torch.randn(S, generator=g)
    tr = torch.randn(S, generator=g)
    tr[hot_rows] *= 100.0
    data = {"obs": obs, "act": act, "log_prob": logp, "target_value_r": tr,
            "target_value_c": torch.randn(S, generator=g).abs(), "adv": torch.randn(S, generator=g)}
    return data, g


def _check(D, A, batch, n_steps, last_rows, max_norm, hot, seed):
    """Two passes of n_steps minibatch steps (the last one of last_rows rows); `hot` is the set of steps (of either pass,
    numbered 0 .. n_steps - 1) whose rows carry the large targets, or None for all steps clipped by a tiny max_norm."""
    from safepo import _lib as L
    from safepo.common.model import ActorVCritic
    from safepo.single_agent._engine import PolicyGradientUpdate
    dev = _cuda()
    torch.manual_seed(seed)
    pol = ActorVCritic(D, A, [64, 64]).to(dev)
    opol = O.OraclePolicy(D, A, [64, 64])
    opol.load(_policy_state(pol))
    S = (n_steps - 1) * batch + last_rows
    g0 = torch.Generator().manual_seed(seed + 1)
    perm = torch.randperm(S, generator=g0)
    hot_rows = torch.cat([perm[s * batch:(s + 1) * batch] for s in sorted(hot)]) if hot else torch.zeros(0, dtype=torch.long)
    data_cpu, g = _data(D, A, S, opol, hot_rows, seed)
    # the second pass visits the same minibatches in the same order, so the clip pattern repeats
    perms = [perm, perm.clone()]
    cfg = dict(hidden_sizes=[64, 64], gamma=0.99, target_kl=1e9, batch_size=batch, learning_iters=2, max_grad_norm=max_norm)
    upd = PolicyGradientUpdate(pol, cfg, L.LOSS_PPO_CLIP, epochs=10**9, host_rng=False, device=dev)
    data = {k: v.to(dev).contiguous() for k, v in data_cpu.items()}
    res = upd.run(data, perms=perms, refresh_old=True)

    opt = O.OracleOptim(opol)
    losses, clipped = [], []
    for p in perms:
        for s0 in range(0, S, batch):
            idx = p[s0:s0 + batch]
            losses.append(O.minibatch_step(opol, opt, {k: v[idx] for k, v in data_cpu.items()}, "ppo", max_grad_norm=max_norm))
            norm = torch.sqrt(sum((q.grad ** 2).sum() for q in opol.all_params() if q.grad is not None))
            clipped.append(float(norm) >= max_norm * 0.999)   # grads are the clipped ones here: norm == max_norm when clipped
    want_clip = [True] * n_steps if hot is None else [s in hot for s in range(n_steps)]
    assert clipped == want_clip * 2, (clipped, want_clip)
    assert res["steps"] == 2 * n_steps

    want = torch.tensor(losses, dtype=torch.float64).mean(0)
    for name, got, w in (("loss_r", res["loss_r"], want[0]), ("loss_c", res["loss_c"], want[1]), ("loss_pi", res["loss_pi"], want[2])):
        ok, err = _close(got, w, rtol=5e-5, atol=5e-6)
        assert ok, (name, got, float(w), err)
    final, ofinal = _policy_state(pol), opol.state()
    for net in O.NET_ORDER:
        for k, v in ofinal[net].items():
            err = float((final[net][k] - v).abs().max())
            assert err < 1e-4, (net, k, err)


@pytest.mark.parametrize("hot", [
    {2, 3, 7, 11},        # the last step clipped: the epilogue undoes W1 / b1 and runs the rest with the clip
    set(range(11)),       # every step but the last clipped: the epilogue's step is the unclipped one
])
def test_last_step_of_launch(hot):
    _check(D=60, A=2, batch=64, n_steps=12, last_rows=29, max_norm=20.0, hot=hot, seed=11)


@pytest.mark.parametrize("max_norm,hot", [
    (0.05, None),          # every step clipped
    (20.0, {0, 1, 2, 5}),  # runs of clipped steps between unclipped ones
])
def test_two_tiles_per_step(max_norm, hot):
    """batch 128: two 64-row tiles per step; the deferred half of the Adam step runs in the first tile only."""
    _check(D=60, A=2, batch=128, n_steps=8, last_rows=100, max_norm=max_norm, hot=hot, seed=12)


@pytest.mark.parametrize("max_norm,hot", [
    (0.05, None),
    (20.0, {1, 2, 7, 11}),
])
def test_wide_action(max_norm, hot):
    """act_dim 12 runs the AC = 16 kernel, where threads 0-63 own a second small parameter (w3 rows, b3, log_std)."""
    _check(D=104, A=12, batch=64, n_steps=12, last_rows=64, max_norm=max_norm, hot=hot, seed=13)
