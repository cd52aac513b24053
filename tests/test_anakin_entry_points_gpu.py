"""Every Anakin system end to end through its hydra_entry_point, at a tiny size: two evaluations (the second learn() call captures and
replays the update step), the absolute metric of the best parameters and a checkpoint, written under a temporary working directory;
and the warm start from such a checkpoint (logger.checkpointing.load_model), for every Anakin system and for Sebulba."""
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


_RUN = ["arch.num_evaluation=2", "arch.absolute_metric=True", "logger.checkpointing.save_model=True", "arch.num_eval_episodes=4",
        "arch.max_eval_steps=50", "logger.use_console=False"]


@pytest.mark.parametrize("system", list(SYSTEMS))
def test_entry_point_runs_evaluates_and_checkpoints(system, tmp_path, monkeypatch):
    from stoix_b200.config import compose

    torch.cuda.set_device(0)
    monkeypatch.chdir(tmp_path)
    name, overrides = SYSTEMS[system]
    cfg = compose(name, overrides + _RUN, config_dir="default/anakin")
    mod = importlib.import_module(f"stoix_b200.systems.{system}")
    assert np.isfinite(mod.hydra_entry_point(cfg))
    saved = sorted(tmp_path.glob(f"checkpoints/{cfg.system.system_name}/*/*.pt"))
    assert saved, "no checkpoint written"
    blob = torch.load(saved[-1], map_location="cpu")
    assert set(blob) >= {"params", "mu", "nu", "counts"} and torch.isfinite(blob["params"]).all()
    assert int(blob["counts"][0]) > 0   # the optimiser stepped before the parameters were saved


_UID = ["logger.checkpointing.save_args.checkpoint_uid=warm", "logger.checkpointing.load_args.checkpoint_uid=warm"]
# the bf16 tensor-core PPO path (relu 2 x 256 Categorical) keeps a bf16 shadow of the arena that a restore must refresh
_WARM = {**SYSTEMS, "ppo.anakin.ff_ppo@bf16": ("default_ff_ppo", _BOX + ["arch.total_num_envs=128", "system.rollout_length=8", "system.num_minibatches=2",
                                                                         "arch.total_timesteps=4096", "arch.precision=bf16"])}


def _latest(tmp_path) -> torch.Tensor:
    """The parameters of the latest step saved under uid "warm" (what a restore without a step loads)."""
    steps = [q for q in tmp_path.glob("checkpoints/*/warm/*.pt") if q.stem.isdigit()]
    return torch.load(max(steps, key=lambda q: int(q.stem)), map_location="cpu")["params"]


def _check_restored(tree, saved: torch.Tensor, fresh: torch.Tensor) -> None:
    """The restored arena is the saved one (which training moved away from the initial parameters), the bf16 shadow follows it and
    the optimiser starts from zero moments and counts."""
    from stoix_b200 import ops

    assert not torch.equal(saved, fresh)
    assert torch.equal(tree.arena.cpu(), saved)
    if getattr(tree, "arena_bf16", None) is not None:
        assert torch.equal(tree.arena_bf16, ops.cast_bf16(tree.arena))
    assert not tree.arena_mu.any() and not tree.arena_nu.any() and not tree.arena_counts.any()


@pytest.mark.parametrize("system", list(_WARM))
def test_warm_start_restores_the_checkpointed_parameters(system, tmp_path, monkeypatch):
    from stoix_b200 import random as srandom
    from stoix_b200.config import compose
    from stoix_b200.utils import make_env
    from stoix_b200.utils.total_timestep_checker import check_total_timesteps

    torch.cuda.set_device(0)
    monkeypatch.chdir(tmp_path)
    name, overrides = _WARM[system]
    mod = importlib.import_module(f"stoix_b200.systems.{system.split('@')[0]}")
    assert np.isfinite(mod.hydra_entry_point(compose(name, overrides + _RUN + _UID, config_dir="default/anakin")))
    saved = _latest(tmp_path)

    def setup(load: bool):
        cfg = compose(name, overrides + _UID + [f"logger.checkpointing.load_model={load}", "logger.use_console=False"], config_dir="default/anakin")
        cfg.num_devices, cfg.rank = 1, 0
        cfg = check_total_timesteps(cfg, quiet=True)
        env, _ = make_env.make(cfg)
        net_keys = 1 if system.startswith("q_learning.") else 2
        key, _, *net = srandom.split(srandom.PRNGKey(cfg.arch.seed), 2 + net_keys)
        return mod.learner_setup(env, (key, *net), cfg)[2].params

    fresh, params = setup(False), setup(True)
    policy = lambda p: p.online if hasattr(p, "online") else getattr(p, "actor_params", p)   # the checkpointed tree
    _check_restored(policy(params), saved, policy(fresh).arena.cpu())
    if system == "sac.ff_sac":   # the target Q networks start as copies of the restored online ones
        a = params.actor_params
        lay = mod.sac_arena_layout(a.spec, params.q_params.online[0].spec)
        assert torch.equal(a.target_arena, a.arena[lay["q1"]: lay["alpha"]])
    if hasattr(params, "target"):
        assert torch.equal(params.target.arena, params.online.arena)


def test_sebulba_warm_start_restores_the_checkpointed_parameters(tmp_path, monkeypatch):
    from stoix_b200 import random as srandom
    from stoix_b200.config import compose
    from stoix_b200.envs import cpu as cpu_envs
    from stoix_b200.systems.ppo.sebulba import ff_ppo as seb
    from stoix_b200.utils.total_timestep_checker import check_total_timesteps

    torch.cuda.set_device(0)
    monkeypatch.chdir(tmp_path)
    overrides = ["arch.total_num_envs=256", "system.rollout_length=8", "system.num_minibatches=2", "arch.total_timesteps=24576",
                 "arch.actor.actor_per_device=2", "arch.num_evaluation=2", "arch.num_eval_episodes=8", "logger.use_console=False",
                 "arch.precision=bf16", "arch.max_eval_steps=300", "logger.checkpointing.save_model=True"] + _UID
    assert np.isfinite(seb.run_experiment(compose("default_ff_ppo", overrides, config_dir="default/sebulba")))
    saved = _latest(tmp_path)

    def setup(load: bool):
        cfg = compose("default_ff_ppo", overrides + [f"logger.checkpointing.load_model={load}"], config_dir="default/sebulba")
        cfg.num_actor_devices, cfg.num_learner_devices, cfg.arch.world_size = 1, 1, 1
        cfg.arch.total_num_actor_threads = 2
        cfg = check_total_timesteps(cfg, quiet=True)
        keys = srandom.split(srandom.PRNGKey(cfg.arch.seed), 4)
        return seb.learner_setup(cpu_envs.make_factory(cfg), (keys[0], keys[2], keys[3]), [torch.device("cuda", 0)], cfg)[2].params

    fresh, params = setup(False), setup(True)
    _check_restored(params.actor_params, saved, fresh.actor_params.arena.cpu())
