"""HAPPO on the device: the reference's ``Runner`` (safepo/multi_agent/happo.py:205-534) is MAPPO's line for line
(safepo/multi_agent/mappo.py here) with ``HAPPO_Trainer``: the product ratio times the cross-agent factor, both active-mask
flags honoured.  There is no CPU path."""
from __future__ import annotations

from safepo.common.ma_model import HAPPOTrainer, MultiAgentNets
from safepo.multi_agent import mappo, mappolag


class Runner(mappo.Runner):
    trainer_class = HAPPOTrainer


# the yaml's values (safepo/multi_agent/marl_cfg/happo/config.yaml) that this path reads, and its mamujoco section (which,
# unlike MAPPO's, leaves both active-mask flags off)
DEFAULT_CONFIG = dict(mappo.DEFAULT_CONFIG, episode_length=75, n_rollout_threads=1, actor_lr=5e-4, critic_lr=5e-4)
MAMUJOCO = dict(episode_length=1000, n_rollout_threads=10, hidden_size=128, gamma=0.99, entropy_coef=0.01,
                n_eval_rollout_threads=10)


def main(argv=None):
    """`python -m safepo.multi_agent.happo --env synthetic [--mamujoco]`: HAPPO on the synthetic multi-agent stream."""
    return mappolag.run_cli(argv, Runner, DEFAULT_CONFIG, "happo", mamujoco=MAMUJOCO)


__all__ = ["Runner", "MultiAgentNets", "HAPPOTrainer", "DEFAULT_CONFIG", "MAMUJOCO", "main"]


if __name__ == "__main__":
    main()
