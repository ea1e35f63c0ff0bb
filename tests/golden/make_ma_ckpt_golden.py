"""Generate tests/golden/ma_ckpt.pt from the REAL reference's multi-agent Runner.save / restore / eval
(safepo/multi_agent/mappolag.py:506-581; mappo.py, happo.py and macpo.py have the same three methods).

Runs only where the reference is checked out (make_golden.REF, read-only); it reuses make_golden.py's import of the reference
(environment packages stubbed) and writes ma_ckpt.pt and nothing else, so the other fixtures stay byte-identical.  The
methods are called on a stand-in ``self`` carrying the real MAPPO_L_Policy / MAPPO_L_Trainer objects (the Runner's constructor
needs environments that are not installable here) and tests/ma_ckpt_oracle.py's deterministic StubMAEnv.

    python tests/golden/make_ma_ckpt_golden.py [OUT]        # default: tests/golden/ma_ckpt.pt
"""
from __future__ import annotations

import importlib
import os
import sys
import tempfile
import types

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
for _p in (HERE, os.path.dirname(HERE), os.path.dirname(os.path.dirname(HERE))):     # make_golden, ma_ckpt_oracle, oracle
    sys.path.insert(0, _p)
import make_golden as MG  # noqa: E402
from ma_ckpt_oracle import StubMAEnv  # noqa: E402

D, DS, A, H, NA = 10, 14, 3, 128, 2          # the device kernels take even input widths and H in {128, .., 512}
PERIODS = (5, 3, 5, 6)             # environment 1 finishes first, environment 1 twice before environment 3 once
ALONE = (0, 1, 2)                  # agent 1 of environment 0 finishes alone at step 2 of its episodes
ENV_SEED = 61
EVAL_EPISODES = (1, 4)             # one step with one finished episode; three steps ending with two environments at once


class Sp:
    def __init__(self, d):
        self.shape = (d,)


def _perturb(pol, g):
    """Move every tensor off its initial value (the fc_mean weights of gain 0.01 included), so that the actions matter."""
    with torch.no_grad():
        for net in (pol.actor, pol.critic, pol.cost_critic):
            for k, v in net.state_dict().items():
                v.add_((0.3 if k.endswith("fc_mean.weight") else 0.1) * torch.randn(v.shape, generator=g))


def gen(out):
    import yaml
    m = importlib.import_module("safepo.multi_agent.mappolag")
    cfg = yaml.safe_load(open(os.path.join(MG.REF, "safepo", "multi_agent", "marl_cfg", "mappolag", "config.yaml")))
    cfg.update(device="cpu", algorithm_name="mappolag", env_name="synthetic", hidden_size=H, n_rollout_threads=len(PERIODS),
               n_eval_rollout_threads=len(PERIODS))
    g = torch.Generator().manual_seed(60)
    torch.manual_seed(62)
    saved_pol = [m.MAPPO_L_Policy(cfg, Sp(D), Sp(DS), Sp(A)) for _ in range(NA)]
    for pol in saved_pol:
        _perturb(pol, g)
    torch.manual_seed(63)
    fresh_pol = [m.MAPPO_L_Policy(cfg, Sp(D), Sp(DS), Sp(A)) for _ in range(NA)]
    with tempfile.TemporaryDirectory() as tmp:
        src = types.SimpleNamespace(config=cfg, num_agents=NA, save_dir=tmp, policy=saved_pol,
                                    trainer=[m.MAPPO_L_Trainer(cfg, pol) for pol in saved_pol])
        m.Runner.save(src)
        saved = [{n: dict(torch.load(os.path.join(tmp, f"{n}_agent{a}.pt"))) for n in ("actor", "critic")} for a in range(NA)]
        env = StubMAEnv(NA, D, DS, PERIODS, ENV_SEED, alone=ALONE)
        dst = types.SimpleNamespace(config=cfg, num_agents=NA, model_dir=tmp, policy=fresh_pol, eval_envs=env,
                                    trainer=[m.MAPPO_L_Trainer(cfg, pol) for pol in fresh_pol])
        m.Runner.restore(dst)
        for a in range(NA):
            for n in ("actor", "critic"):
                for k, v in getattr(fresh_pol[a], n).state_dict().items():
                    assert torch.equal(v, saved[a][n][k]), (a, n, k)
        evals = {k: tuple(float(x) for x in m.Runner.eval(dst, k)) for k in EVAL_EPISODES}
    out["ckpt"] = dict(dims=(D, DS, A, H, NA), std=(cfg["std_x_coef"], cfg["std_y_coef"], cfg["layer_N"]),
                       env=dict(periods=PERIODS, alone=ALONE, seed=ENV_SEED), saved=saved, evals=evals)


def main():
    path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "ma_ckpt.pt")
    sys.path.insert(0, MG.ROOT)
    MG.import_reference()
    threads = torch.get_num_threads()
    torch.set_num_threads(1)       # as the other multi-agent fixtures: one intra-op thread
    out = {}
    gen(out)
    torch.set_num_threads(threads)
    torch.save(out, path)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
