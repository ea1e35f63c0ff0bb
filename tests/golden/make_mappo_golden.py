"""Generate tests/golden/mappo.pt from the REAL reference's MAPPO and HAPPO (safepo/multi_agent/mappo.py, happo.py).

Runs only where the reference is checked out (make_golden.REF, read-only); it reuses make_golden.py's import of the reference
(environment packages stubbed).  It writes mappo.pt and nothing else, so the other fixtures stay byte-identical.

    python tests/golden/make_mappo_golden.py [OUT]        # default: tests/golden/mappo.pt
"""
from __future__ import annotations

import importlib
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as MG  # noqa: E402

ALGOS = {"mappo": ("MAPPO_Policy", "MAPPO_Trainer"), "happo": ("HAPPO_Policy", "HAPPO_Trainer")}
# the yaml's mamujoco flags with its entropy coefficient: both active-mask flags on
FLAGS = {"defaults": {}, "mamujoco": dict(use_policy_active_masks=True, use_value_active_masks=True, entropy_coef=0.01)}
KEEP = ("actor_lr", "critic_lr", "opti_eps", "weight_decay", "clip_param", "huber_delta", "entropy_coef", "max_grad_norm", "gamma",
        "gae_lambda", "value_loss_coef", "layer_N", "std_x_coef", "std_y_coef", "learning_iters", "use_policy_active_masks",
        "use_value_active_masks")


class Sp:
    def __init__(self, d):
        self.shape = (d,)


def _config(algo, **changes):
    import yaml
    cfg = yaml.safe_load(open(os.path.join(MG.REF, "safepo", "multi_agent", "marl_cfg", algo, "config.yaml")))
    cfg.update(device="cpu", algorithm_name=algo, env_name="synthetic", **changes)
    return cfg


def _perturb(pol):
    """Move the LayerNorm affine parameters and biases off their trivial initial values."""
    with torch.no_grad():
        for net in (pol.actor, pol.critic):
            for k, v in net.state_dict().items():
                if k.endswith("bias") or ".2.weight" in k or "feature_norm" in k or k.endswith("log_std"):
                    v.add_(0.1 * torch.randn_like(v))


def _states(pol):
    return {n: {k: v.clone() for k, v in getattr(pol, n).state_dict().items()} for n in ("actor", "critic")}


def gen_updates(out):
    """For each trainer, two consecutive ppo_update calls at the yaml's defaults and two with the mamujoco flags: obs 10,
    share_obs 14, act 3, hidden 32, 48 rows of which about a quarter inactive, ratios spread so that every clip branch occurs
    in some dimension (and the product falls on both sides).  Stored per call: the returned values, the PopArt state and both
    state dicts; per case the initial state dicts and the sample."""
    D, DS, A, N = 10, 14, 3, 48
    cases = {}
    for algo, (pcls, tcls) in ALGOS.items():
        m = importlib.import_module(f"safepo.multi_agent.{algo}")
        for flag_name, flags in FLAGS.items():
            cfg = _config(algo, n_rollout_threads=4, hidden_size=32, **flags)
            torch.manual_seed(31)
            pol = getattr(m, pcls)(cfg, Sp(D), Sp(DS), Sp(A))
            _perturb(pol)
            tr = getattr(m, tcls)(cfg, pol)
            g = torch.Generator().manual_seed(32)
            obs, share = torch.randn(N, D, generator=g) * 2 + 0.5, torch.randn(N, DS, generator=g) * 3
            rnn, masks = np.zeros((N, 1, 32), dtype=np.float32), np.ones((N, 1), dtype=np.float32)
            init = _states(pol)
            with torch.no_grad():
                mu = pol.actor(obs, rnn, masks, deterministic=True)[0]
                std = torch.sigmoid(pol.actor.state_dict()["act.action_out.log_std"] / cfg["std_x_coef"]) * cfg["std_y_coef"]
                actions = mu + std * torch.randn(N, A, generator=g)
                logp = pol.actor.evaluate_actions(obs, rnn, actions, masks, None, None)[0]
            active = (torch.rand(N, 1, generator=g) >= 0.25).float()
            sample = dict(share_obs=share, obs=obs, actions=actions, value_preds=0.1 * torch.randn(N, 1, generator=g),
                          returns=torch.randn(N, 1, generator=g) * 4 + 1, old_action_log_probs=logp + 0.3 * torch.randn(N, A, generator=g),
                          adv_targ=torch.randn(N, 1, generator=g), factor=torch.rand(N, 1, generator=g) + 0.5, active_masks=active)
            calls = []
            for _ in range(2):
                tup = (share.numpy(), obs.numpy(), rnn, rnn, actions.numpy(), sample["value_preds"], sample["returns"], masks,
                       sample["active_masks"], sample["old_action_log_probs"], sample["adv_targ"], None, sample["factor"])
                r = tr.ppo_update(tup)
                names = ("value_loss", "critic_grad_norm", "policy_loss", "dist_entropy", "actor_grad_norm", "imp_weights")
                vn = tr.value_normalizer
                calls.append(dict(out={k: v.detach().clone() for k, v in zip(names, r)},
                                  popart=(vn.running_mean.clone(), vn.running_mean_sq.clone(), vn.debiasing_term.clone()), state=_states(pol)))
            cases[(algo, flag_name)] = dict(cfg={k: cfg[k] for k in KEEP}, init=init, sample=sample, calls=calls)
    out["updates"] = dict(dims=(D, DS, A, N), cases=cases)


def gen_epochs(out):
    """Two whole iterations of TWO agents through each reference Runner's own methods (collect / insert / compute / train of
    mappo.py:347-437,518-526 / happo.py's, called on a stand-in ``self`` carrying the real policies, trainers and buffers -- the
    Runner's constructor needs environments that are not installable here), mamujoco flags on: T = 4 steps, 6 envs, hidden 32,
    learning_iters 2.  Agent 1 of env 0 finishes alone at step 1 of every iteration (active mask 0), every agent of env 1 at
    step 2.  Stored: the initial state dicts, the env stream, the global-RNG seed and after every iteration the buffers' returns,
    masks and factor, the PopArt state and every state dict."""
    T, N, D, DS, A, H, NA = 4, 6, 10, 14, 3, 32, 2
    epochs = {}

    class Log:
        def store(self, **kw):
            pass
    for algo, (pcls, tcls) in ALGOS.items():
        m = importlib.import_module(f"safepo.multi_agent.{algo}")
        cfg = _config(algo, n_rollout_threads=N, hidden_size=H, episode_length=T, learning_iters=2, **FLAGS["mamujoco"])
        torch.manual_seed(41)
        policy = [getattr(m, pcls)(cfg, Sp(D), Sp(DS), Sp(A)) for _ in range(NA)]
        for pol in policy:
            _perturb(pol)
        init = [_states(pol) for pol in policy]
        fake = types.SimpleNamespace(config=cfg, num_agents=NA, logger=Log(), policy=policy,
                                     trainer=[getattr(m, tcls)(cfg, pol) for pol in policy],
                                     buffer=[m.SeparatedReplayBuffer(cfg, Sp(D), Sp(DS), Sp(A)) for _ in range(NA)])
        g = torch.Generator().manual_seed(42)
        obs0, share0 = torch.randn(N, NA, D, generator=g) * 2 + 0.5, torch.randn(N, NA, DS, generator=g) * 3
        for a in range(NA):                                    # Runner.warmup
            fake.buffer[a].share_obs[0].copy_(share0[:, a])
            fake.buffer[a].obs[0].copy_(obs0[:, a])
        stream, iters, seed = [], [], 78
        torch.manual_seed(seed)
        for it in range(2):
            steps = []
            for step in range(T):
                values, actions, action_log_probs, rnn_states, rnn_states_critic = m.Runner.collect(fake, step)
                obs, share_obs = torch.randn(N, NA, D, generator=g) * 2 + 0.5, torch.randn(N, NA, DS, generator=g) * 3
                rewards = torch.randn(N, NA, 1, generator=g)
                dones = torch.zeros(N, NA, dtype=torch.bool)
                if step == 1:
                    dones[0, 1] = True
                if step == 2:
                    dones[1, :] = True
                m.Runner.insert(fake, (obs, share_obs, rewards, dones, None, values, actions, action_log_probs, rnn_states, rnn_states_critic))
                steps.append(dict(obs=obs, share_obs=share_obs, rewards=rewards, dones=dones, values=values.clone(),
                                  actions=[x.clone() for x in actions], action_log_probs=[x.clone() for x in action_log_probs]))
            m.Runner.compute(fake)
            after_compute = [dict(returns=b.returns.clone(), value_preds=b.value_preds.clone(), masks=b.masks.clone(),
                                  active_masks=b.active_masks.clone()) for b in fake.buffer]
            m.Runner.train(fake)
            res = []
            for a in range(NA):
                vn = fake.trainer[a].value_normalizer
                res.append(dict(factor=fake.buffer[a].factor.clone(), popart=(vn.running_mean.clone(), vn.running_mean_sq.clone(),
                                                                              vn.debiasing_term.clone()), state=_states(policy[a])))
            stream.append(steps)
            iters.append(dict(after_compute=after_compute, agents=res))
        epochs[algo] = dict(cfg={k: cfg[k] for k in KEEP}, init=init, obs0=obs0, share_obs0=share0, seed=seed, stream=stream, iters=iters)
    out["epochs"] = dict(dims=(T, N, D, DS, A, H, NA), runs=epochs)


def main():
    path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "mappo.pt")
    sys.path.insert(0, MG.ROOT)
    MG.import_reference()
    threads = torch.get_num_threads()
    torch.set_num_threads(1)       # LayerNorm's backward reductions depend on the intra-op thread count (see make_golden.gen_ma_update)
    out = {}
    gen_updates(out)
    gen_epochs(out)
    torch.set_num_threads(threads)
    torch.save(out, path)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
