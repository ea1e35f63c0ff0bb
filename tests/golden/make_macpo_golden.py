"""Generate tests/golden/macpo.pt from the REAL reference's MACPO_Trainer (safepo/multi_agent/macpo.py:96-415).

Runs only where the reference is checked out (make_golden.REF, read-only); it reuses make_golden.py's import of the reference
(environment packages stubbed) and stubs joblib as well, which macpo.py imports.  It writes macpo.pt and nothing else, so the
other fixtures stay byte-identical.

    python tests/golden/make_macpo_golden.py [OUT]        # default: tests/golden/macpo.pt
"""
from __future__ import annotations

import importlib
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as MG  # noqa: E402

# (aver_episode_costs, cost advantages, target_kl, searching_steps): the cases 1, 2, 3, 4 and 0, then "shrink" -- zero cost
# advantages (case 4) and reward advantages -sum_j (z_j^2 - 1), z = (action - mean) / std, which shrink every std, so the
# reference's KL grows linearly with the step: target_kl 1e-5 rejects the first trials, 1e-6 with one trial rejects it (revert)
SCENARIOS = [(30.0, 1.0, 0.016, 10), (20.0, 1.0, 0.016, 10), (0.0, 1.0, 0.016, 10), (20.0, 0.0, 0.016, 10), (100.0, 1.0, 0.016, 10),
             (20.0, "shrink", 1e-5, 10), (20.0, "shrink", 1e-6, 1)]


def gen_macpo(out):
    """Consecutive trpo_update calls of one MACPO_Trainer at small dimensions (obs 10, share_obs 14, act 3, hidden 32, the yaml's
    layer_N = 2, one intra-op thread), one per scenario.  Stored per call: the sample and the search settings, g and b (the two
    right-hand sides of the conjugate gradient, recorded from its calls), both CG solutions, q / r / s, the case, lambda, nu,
    the final x, the accepted trial (-1: reverted), the returned scalars, the PopArt state and all state dicts after the call."""
    import yaml
    sys.modules.setdefault("joblib", MG._Anything("joblib"))
    MG.import_reference()
    m = importlib.import_module("safepo.multi_agent.macpo")
    cfg = yaml.safe_load(open(os.path.join(MG.REF, "safepo", "multi_agent", "marl_cfg", "macpo", "config.yaml")))
    cfg.update(device="cpu", algorithm_name="macpo", n_rollout_threads=4, hidden_size=32)

    class Sp:
        def __init__(self, d):
            self.shape = (d,)

    threads = torch.get_num_threads()
    torch.set_num_threads(1)       # LayerNorm's backward reductions depend on the intra-op thread count (see gen_ma_update)
    torch.manual_seed(41)
    D, DS, A, N = 10, 14, 3, 48
    pol = m.MACPO_Policy(cfg, Sp(D), Sp(DS), Sp(A))
    with torch.no_grad():          # move the LayerNorm affine parameters and biases off their trivial initial values
        for net in (pol.actor, pol.critic, pol.cost_critic):
            for k, v in net.state_dict().items():
                if k.endswith("bias") or ".2.weight" in k or "feature_norm" in k or k.endswith("log_std"):
                    v.add_(0.1 * torch.randn_like(v))
    tr = m.MACPO_Trainer(cfg, pol)
    rec = {"cg": [], "actor_updates": 0}
    real_cg, real_update = tr.conjugate_gradient, tr.update_model

    def cg(*args, **kw):
        x = real_cg(*args, **kw)
        rec["cg"].append((args[7].clone(), x.clone()))        # (b, solution)
        return x

    def update_model(model, new_params):
        if model is pol.actor:
            rec["actor_updates"] += 1
        return real_update(model, new_params)
    tr.conjugate_gradient, tr.update_model = cg, update_model

    g = torch.Generator().manual_seed(42)
    obs, share = torch.randn(N, D, generator=g) * 2 + 0.5, torch.randn(N, DS, generator=g) * 3
    rnn, masks = np.zeros((N, 1, 32), dtype=np.float32), np.ones((N, 1), dtype=np.float32)
    init = {n: {k: v.clone() for k, v in getattr(pol, n).state_dict().items()} for n in ("actor", "critic", "cost_critic")}
    with torch.no_grad():
        dist = pol.actor.evaluate_actions(obs, rnn, torch.zeros(N, A), masks, None, masks)
        actions = dist[2] + dist[3] * torch.randn(N, A, generator=g)
        logp = pol.actor.evaluate_actions(obs, rnn, actions, masks, None, masks)[0]
    calls = []
    for aver, cadv, tkl, steps in SCENARIOS:
        cfg["target_kl"], cfg["searching_steps"] = tkl, steps
        sample = dict(share_obs=share, obs=obs, actions=actions, value_preds=0.1 * torch.randn(N, 1, generator=g),
                      returns=torch.randn(N, 1, generator=g) * 4 + 1, old_action_log_probs=logp + 0.05 * torch.randn(N, A, generator=g) / A ** 0.5,
                      adv_targ=torch.randn(N, 1, generator=g), factor=torch.rand(N, 1, generator=g) + 0.5,
                      cost_preds=0.1 * torch.randn(N, 1, generator=g), cost_returns=torch.randn(N, 1, generator=g).abs() * 30,
                      cost_adv_targ=(0.0 if cadv == "shrink" else cadv) * torch.randn(N, 1, generator=g),
                      aver_episode_costs=torch.full((N, 1), float(aver)))
        if cadv == "shrink":
            with torch.no_grad():
                _, _, mu, std = pol.actor.evaluate_actions(obs, rnn, actions, masks, None, masks)
                sample["adv_targ"] = -(((actions - mu) / std) ** 2 - 1).sum(-1, keepdim=True)
        tup = (share.numpy(), obs.numpy(), rnn, rnn, actions.numpy(), sample["value_preds"], sample["returns"], masks, masks,
               sample["old_action_log_probs"], sample["adv_targ"], None, sample["factor"], sample["cost_preds"], sample["cost_returns"], rnn,
               sample["cost_adv_targ"], sample["aver_episode_costs"])
        rec["cg"], rec["actor_updates"] = [], 0
        r = tr.trpo_update(tup)
        (value_loss, critic_grad_norm, kl, loss_improve, expected_improve, dist_entropy, ratio, cost_loss, cost_grad_norm, recover,
         _, _, _, lam, nu, _, _, x, _, _, bb) = r
        (gv, xg), (bv, xb) = rec["cg"]
        rescale = (sample["aver_episode_costs"].mean() - cfg["cost_limit"]) * (1 - cfg["gamma"])
        # the case, from the same tests as macpo.py:272-298 on the values it used
        if bb <= 1e-8 and rescale < 0:
            case = 4
        else:
            rec_v = float(recover)
            case = 3 if rescale < 0 and rec_v < 0 else 2 if rescale < 0 else 1 if rec_v >= 0 else 0
        n_upd = rec["actor_updates"]          # one per trial, plus one when the old weights come back
        accepted = -1 if n_upd == steps + 1 else n_upd - 1
        vn = tr.value_normalizer
        calls.append(dict(sample=sample, target_kl=tkl, searching_steps=steps, g=gv, b=bv, xg=xg, xb=xb,
                          q=(gv * xg).sum(0, keepdim=True), r=(gv * xb).sum(0, keepdim=True), s=(bv * xb).sum(0, keepdim=True), bb=bb.clone(),
                          optim_case=case, lam=torch.as_tensor(lam).clone(), nu=torch.as_tensor(nu).clone(), x=x.detach().clone(), accepted=accepted,
                          out=dict(value_loss=value_loss.detach(), critic_grad_norm=critic_grad_norm, kl=kl.detach(), loss_improve=loss_improve.detach(),
                                   expected_improve=expected_improve.detach(), dist_entropy=dist_entropy.detach(), cost_loss=cost_loss.detach(),
                                   cost_grad_norm=cost_grad_norm),
                          popart=(vn.running_mean.clone(), vn.running_mean_sq.clone(), vn.debiasing_term.clone()),
                          state={n: {k: v.clone() for k, v in getattr(pol, n).state_dict().items()} for n in ("actor", "critic", "cost_critic")}))
    keep = ("actor_lr", "critic_lr", "opti_eps", "weight_decay", "clip_param", "huber_delta", "max_grad_norm", "cost_limit", "gamma",
            "value_loss_coef", "layer_N", "std_x_coef", "std_y_coef", "step_fraction", "fraction_coef", "conjugate_gradient_iters")
    torch.set_num_threads(threads)
    out["macpo"] = dict(cfg={k: cfg[k] for k in keep}, dims=(D, DS, A, N), init=init, calls=calls)


def main():
    path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "macpo.pt")
    sys.path.insert(0, MG.ROOT)
    out = {}
    gen_macpo(out)
    torch.save(out, path)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB",
          [(c["optim_case"], c["accepted"]) for c in out["macpo"]["calls"]])


if __name__ == "__main__":
    main()
