"""MACPO on the device: the reference's ``Runner`` of safepo/multi_agent/macpo.py:427-859, which is MAPPO-Lag's runner
(collect / insert / compute / the cross-agent factor, safepo/multi_agent/mappolag.py here) with ``MACPO_Trainer`` -- one
constrained trust-region step of the actor per iteration and agent (safepo/common/ma_model.py: MACPOTrainer) -- and its own
logged values: ``Loss_actor_improve``, ``Loss_actor_expected_improve`` and ``Misc/KL`` in place of ``Loss_actor`` and the
Lagrange multiplier.  There is no CPU path."""
from __future__ import annotations

from safepo.common.ma_model import MACPOTrainer, MultiAgentNets
from safepo.multi_agent import mappolag


class Runner(mappolag.Runner):
    trainer_class = MACPOTrainer

    def log_agent(self, a, out):
        """MACPO_Trainer.train's logged values (macpo.py:402-414) of agent a.  As in the reference, "Loss_cost_critic" is the
        actor's cost surrogate."""
        return {f"Loss/Loss_reward_critic/agent{a}": float(out["value_loss"]), f"Loss/Loss_cost_critic/agent{a}": float(out["cost_loss"]),
                f"Loss/Loss_actor_improve/agent{a}": float(out["loss_improve"]),
                f"Loss/Loss_actor_expected_improve/agent{a}": float(out["expected_improve"]),
                f"Misc/Reward_critic_norm/agent{a}": float(out["critic_grad_norm"]), f"Misc/Cost_critic_norm/agent{a}": float(out["cost_grad_norm"]),
                f"Misc/Entropy/agent{a}": float(out["dist_entropy"]), f"Misc/Ratio/agent{a}": float(out["ratio"]), f"Misc/KL/agent{a}": float(out["kl"])}


# the yaml's values (safepo/multi_agent/marl_cfg/macpo/config.yaml) that this path reads
DEFAULT_CONFIG = dict(episode_length=8, n_rollout_threads=1024, hidden_size=512, layer_N=2, gamma=0.96, gae_lambda=0.95, learning_iters=5,
                      num_mini_batch=1, actor_lr=9e-5, critic_lr=5e-3, opti_eps=1e-5, weight_decay=0.0, clip_param=0.2, huber_delta=10.0,
                      entropy_coef=0.0, max_grad_norm=10.0, cost_limit=25.0, value_loss_coef=1.0, std_x_coef=1.0, std_y_coef=0.5, actor_gain=0.01,
                      target_kl=0.016, searching_steps=10, step_fraction=0.5, fraction_coef=0.1, conjugate_gradient_iters=10)


def main(argv=None):
    """`python -m safepo.multi_agent.macpo --env synthetic`: MACPO on a synthetic multi-agent stream of config 5's shape, with
    the flags of `python -m safepo.multi_agent.mappolag`."""
    return mappolag.run_cli(argv, Runner, DEFAULT_CONFIG, "macpo")


__all__ = ["Runner", "MultiAgentNets", "MACPOTrainer", "DEFAULT_CONFIG", "main"]


if __name__ == "__main__":
    main()
