"""Every Anakin system end to end through its hydra_entry_point, at a tiny size: two evaluations (the second learn() call captures and
replays the update step), the absolute metric of the best parameters and a checkpoint, written under a temporary working directory."""
import importlib

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

_BOX = ["env=synthetic/box", "env.kwargs.obs_dim=8", "env.kwargs.num_actions=3", "env.kwargs.p_term=0.05"]
_CONT = ["env.kwargs.obs_dim=8", "env.kwargs.act_dim=2", "env.kwargs.p_term=0.05"]
_MLP = ["network.actor_network.pre_torso.layer_sizes=[32,32]", "network.critic_network.pre_torso.layer_sizes=[32,32]"]
_PPO = ["arch.total_num_envs=16", "system.rollout_length=8", "system.num_minibatches=2", "arch.total_timesteps=512"] + _MLP
_DQN = _BOX + ["arch.total_num_envs=16", "system.rollout_length=2", "system.epochs=2", "system.total_batch_size=32", "system.total_buffer_size=400",
               "system.warmup_steps=3", "arch.total_timesteps=128", "network.actor_network.pre_torso.layer_sizes=[32,32]"]

SYSTEMS = {   # module: (default config, overrides)
    "ppo.anakin.ff_ppo": ("default_ff_ppo", _BOX + _PPO + ["system.normalize_observations=True", "system.obs_norm_warmup_steps=4"]),
    "ppo.anakin.ff_ppo_continuous": ("default_ff_ppo_continuous", _CONT + _PPO),
    "ppo.anakin.ff_ppo_penalty": ("default_ff_ppo", _BOX + _PPO),
    "ppo.anakin.ff_ppo_penalty_continuous": ("default_ff_ppo_continuous", _CONT + _PPO),
    "ppo.anakin.ff_dpo_continuous": ("default_ff_dpo_continuous", _CONT + _PPO),
    "ppo.anakin.rec_ppo": ("default_rec_ppo", _BOX + ["arch.total_num_envs=16", "system.rollout_length=8", "system.num_minibatches=2", "system.epochs=2",
                                                      "arch.total_timesteps=512", "network.actor_network.pre_torso.layer_sizes=[24]",
                                                      "network.actor_network.post_torso.layer_sizes=[20]", "network.critic_network.pre_torso.layer_sizes=[24]",
                                                      "network.critic_network.post_torso.layer_sizes=[20]",
                                                      "network.actor_network.rnn_layer.hidden_state_dim=16",
                                                      "network.critic_network.rnn_layer.hidden_state_dim=16"]),
    "sac.ff_sac": ("default_ff_sac", _CONT + ["arch.total_num_envs=16", "system.total_batch_size=32", "system.total_buffer_size=1024", "system.warmup_steps=2",
                                              "arch.total_timesteps=256", "network.actor_network.pre_torso.layer_sizes=[32,32]",
                                              "network.q_network.pre_torso.layer_sizes=[32,32]"]),
    "q_learning.ff_pqn": ("default_ff_pqn", _BOX + ["arch.total_num_envs=16", "system.rollout_length=4", "system.num_minibatches=2", "system.epochs=2",
                                                    "arch.total_timesteps=256", "network.actor_network.pre_torso.layer_sizes=[32,32]"]),
    "q_learning.ff_dqn": ("default_ff_dqn", _DQN),
    "q_learning.ff_ddqn": ("default_ff_ddqn", _DQN),
    "q_learning.ff_mdqn": ("default_ff_mdqn", _DQN),
    "q_learning.ff_dqn_reg": ("default_ff_dqn_reg", _DQN),
}


@pytest.mark.parametrize("system", list(SYSTEMS))
def test_entry_point_runs_evaluates_and_checkpoints(system, tmp_path, monkeypatch):
    from stoix_b200.config import compose

    torch.cuda.set_device(0)
    monkeypatch.chdir(tmp_path)
    name, overrides = SYSTEMS[system]
    cfg = compose(name, overrides + ["arch.num_evaluation=2", "arch.absolute_metric=True", "logger.checkpointing.save_model=True",
                                     "arch.num_eval_episodes=4", "arch.max_eval_steps=50", "logger.use_console=False"], config_dir="default/anakin")
    mod = importlib.import_module(f"stoix_b200.systems.{system}")
    assert np.isfinite(mod.hydra_entry_point(cfg))
    saved = sorted(tmp_path.glob(f"checkpoints/{cfg.system.system_name}/*/*.pt"))
    assert saved, "no checkpoint written"
    blob = torch.load(saved[-1], map_location="cpu")
    assert set(blob) >= {"params", "mu", "nu", "counts"} and torch.isfinite(blob["params"]).all()
    assert int(blob["counts"][0]) > 0   # the optimiser stepped before the parameters were saved
