"""MAPPO on the device: the per-iteration part of the reference's ``Runner`` (safepo/multi_agent/mappo.py:197-526: ``collect`` /
``insert`` / ``compute`` / ``train`` / ``run``) for agents of an actor and a reward critic, around ``MultiAgentNets`` (two nets)
/ ``MAPPOTrainer`` (safepo/common/ma_model.py) and ``SeparatedReplayBuffer``.  It is MAPPO-Lag's runner with
``cost_critic = False``, which skips the cost side: no costs or cost predictions go into the buffers, compute() builds the
reward returns only, and the cross-agent factor loop of train() is the same (mappo.py:408-437, identical in
happo.py:416-445).  There is no CPU path."""
from __future__ import annotations

from safepo.common.ma_model import MAPPOTrainer, MultiAgentNets
from safepo.multi_agent import mappolag


class Runner(mappolag.Runner):
    trainer_class = MAPPOTrainer
    cost_critic = False

    def log_agent(self, a, out):
        """The logged values of agent a's last update (mappo.py:178-186)."""
        value_loss, critic_norm, policy_loss, entropy, actor_norm, imp = out
        return {f"Loss/Loss_reward_critic/agent{a}": float(value_loss), f"Loss/Loss_actor/agent{a}": float(policy_loss),
                f"Misc/Reward_critic_norm/agent{a}": float(critic_norm), f"Misc/Entropy/agent{a}": float(entropy),
                f"Misc/Ratio/agent{a}": float(imp.mean())}


# the yaml's values (safepo/multi_agent/marl_cfg/mappo/config.yaml) that this path reads, and its mamujoco section
DEFAULT_CONFIG = dict(episode_length=8, n_rollout_threads=80, hidden_size=512, layer_N=2, gamma=0.96, gae_lambda=0.95, learning_iters=5,
                      num_mini_batch=1, actor_lr=9e-5, critic_lr=5e-3, opti_eps=1e-5, weight_decay=0.0, clip_param=0.2, huber_delta=10.0,
                      entropy_coef=0.0, max_grad_norm=10.0, value_loss_coef=1.0, use_policy_active_masks=False,
                      use_value_active_masks=False, std_x_coef=1.0, std_y_coef=0.5, actor_gain=0.01, save_interval=1, use_eval=False,
                      eval_interval=25, n_eval_rollout_threads=1)
MAMUJOCO = dict(episode_length=1000, n_rollout_threads=10, hidden_size=128, gamma=0.99, entropy_coef=0.01, max_grad_norm=10.0,
                use_value_active_masks=True, use_policy_active_masks=True, n_eval_rollout_threads=10)


def main(argv=None):
    """`python -m safepo.multi_agent.mappo --env synthetic [--mamujoco]`: MAPPO on a synthetic multi-agent stream of config 5's
    shape (the reference's Isaac-Gym / multi-agent MuJoCo environments are not installable offline)."""
    return mappolag.run_cli(argv, Runner, DEFAULT_CONFIG, "mappo", mamujoco=MAMUJOCO)


__all__ = ["Runner", "MultiAgentNets", "MAPPOTrainer", "DEFAULT_CONFIG", "MAMUJOCO", "main"]


if __name__ == "__main__":
    main()
