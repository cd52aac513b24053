"""Host-side logic that mirrors the reference's Python faces, checked on CPU against the oracle's restatement of the
same reference lines: shape derivation (total_timestep_checker.py), the learning-rate schedule (utils/training.py),
the config layer (Hydra-style composition, `_target_` resolution) and the leading-dim helpers (utils/jax_utils.py)."""
import itertools

import numpy as np
import pytest
import torch

from oracle import ppo_oracle as O
from stoix_b200.config import _locate, compose, instantiate
from stoix_b200.utils import jax_utils
from stoix_b200.utils.total_timestep_checker import check_total_timesteps
from stoix_b200.utils.training import make_learning_rate, make_learning_rate_schedule


@pytest.mark.parametrize("devices,ubs", [(1, 1), (2, 1), (8, 1), (4, 2), (1, 4)])
def test_shape_derivation_matches_the_successive_floor_divisions(devices, ubs):
    """total_timestep_checker.py:57-61, 88-96, 107: num_envs, num_updates (floor divisions IN THAT ORDER), updates per eval."""
    for total_envs, T, steps, n_eval in itertools.product((64, 4096 * 8, 1024), (8, 128), (1e6, 41943040, 3e7), (1, 5, 20)):
        if total_envs % (devices * ubs):
            continue
        cfg = compose("default_ff_ppo", ["env=synthetic/box", f"arch.total_num_envs={total_envs}", f"arch.update_batch_size={ubs}",
                                         f"system.rollout_length={T}", f"arch.total_timesteps={steps}", f"arch.num_evaluation={n_eval}"])
        cfg.num_devices = devices
        want = O.derive_shapes(total_envs, devices, ubs, steps, T, n_eval)
        if want[1] < n_eval:  # fewer updates than evaluations: nothing to derive (the reference asserts on this configuration)
            continue
        cfg = check_total_timesteps(cfg, quiet=True)
        assert (cfg.arch.num_envs, cfg.arch.num_updates, cfg.arch.num_updates_per_eval) == want


def test_shape_derivation_from_num_updates_and_divisibility_error():
    cfg = compose("default_ff_ppo", ["env=synthetic/box", "arch.total_num_envs=512", "arch.total_timesteps=null", "arch.num_updates=7",
                                     "system.rollout_length=16", "arch.num_evaluation=1"])
    cfg.num_devices = 2
    cfg = check_total_timesteps(cfg, quiet=True)
    assert cfg.arch.num_envs == 256 and cfg.arch.total_timesteps == 2 * 7 * 16 * 256  # :72-85
    cfg.arch.total_num_envs = 511
    with pytest.raises(AssertionError, match="must be divisible"):
        check_total_timesteps(cfg, quiet=True)


def test_learning_rate_schedule_floor_division_and_constants():
    """training.py:24-26: lr(count) = init * (1 - (count // (epochs*minibatches)) / num_updates); constant when decay is off."""
    sched = make_learning_rate_schedule(3e-4, num_updates=10, num_epochs=4, num_minibatches=16)
    for count in (0, 1, 63, 64, 65, 127, 128, 639, 640):
        assert sched(count) == pytest.approx(O.linear_schedule(3e-4, count, 10, 4, 16), rel=0, abs=0)
    assert sched(63) == sched(0) and sched(64) < sched(63)  # steps down once per update, not per optimiser step
    assert (sched.init_lr, sched.num_updates, sched.steps_per_update) == (3e-4, 10, 64)  # what the device-side schedule reads
    cfg = compose("default_ff_ppo", ["env=synthetic/box", "system.decay_learning_rates=False"])
    assert make_learning_rate(1e-3, cfg, 4, 16) == 1e-3
    cfg = compose("default_ff_ppo", ["env=synthetic/box", "system.decay_learning_rates=True", "arch.num_updates=5"])
    assert make_learning_rate(1e-3, cfg, 4, 16)(64 * 5 - 1) == pytest.approx(1e-3 * (1 - 4 / 5))


def test_config_composition_overrides_and_target_resolution():
    cfg = compose("default_ff_ppo", ["env=gymnax/cartpole", "system.clip_eps=0.3", "network.actor_network.pre_torso.layer_sizes=[32,32]",
                                     "arch.precision=bf16", "arch.seed=7"])
    assert cfg.env.scenario.name == "CartPole-v1" and cfg.system.clip_eps == 0.3 and cfg.arch.seed == 7
    assert cfg.network.actor_network.pre_torso.layer_sizes == [32, 32]
    assert cfg.network.critic_network.pre_torso.layer_sizes == [256, 256]  # the other network keeps the default
    # the reference's `_target_` strings resolve to this package's classes (same constructor arguments)
    assert cfg.network.actor_network.pre_torso._target_ == "stoix.networks.torso.MLPTorso"
    torso = instantiate(cfg.network.actor_network.pre_torso)
    assert type(torso) is _locate("stoix.networks.torso.MLPTorso") and type(torso).__module__ == "stoix_b200.networks.torso"
    assert tuple(torso.layer_sizes) == (32, 32)
    with pytest.raises(FileNotFoundError):
        compose("default_ff_ppo", ["env=does/not_exist"])
    # system defaults of configs/system/ppo/ff_ppo.yaml:6-22
    d = compose("default_ff_ppo", ["env=synthetic/box"]).system
    assert (d.rollout_length, d.epochs, d.num_minibatches, d.gamma, d.gae_lambda, d.clip_eps, d.ent_coef, d.vf_coef, d.max_grad_norm) == \
        (128, 4, 16, 0.99, 0.95, 0.2, 0.01, 0.5, 0.5)


def test_merge_leading_dims_is_time_major_flat_index():
    """jax_utils.py:29-43: the flat batch index of (T, E) is t*E + e -- the index space of the shuffle permutation."""
    T, E, D = 3, 5, 2
    x = torch.arange(T * E * D).reshape(T, E, D)
    flat = jax_utils.merge_leading_dims(x, 2)
    assert flat.shape == (T * E, D)
    assert torch.equal(flat[2 * E + 4], x[2, 4])
    assert jax_utils.merge_leading_dims(torch.zeros(4), 2).shape == (4,)  # fewer dims than requested: unchanged
    tree = {"a": torch.ones(2, 3, 4), "b": (torch.zeros(2, 3), 5)}
    out = jax_utils.unreplicate_n_dims(tree, 2)
    assert out["a"].shape == (4,) and out["b"][0].ndim == 0 and out["b"][1] == 5
    assert jax_utils.unreplicate_batch_dim({"m": torch.ones(6, 2, 3)})["m"].shape == (6, 3)


def test_oracle_update_is_invariant_to_the_shard_axis_layout():
    """The learner flattens (T, E) time-major; the oracle must agree with an explicit loop over the flat index."""
    rng = np.random.default_rng(3)
    T, E = 6, 4
    r, d = rng.standard_normal((T, E)), (rng.random((T, E)) < 0.2)
    v, bv = rng.standard_normal((T, E)), rng.standard_normal((T, E))
    r_t, d_t, trunc = O.ppo_gae_inputs(r, d, np.zeros_like(d), 0.99, 1.0)
    adv, tgt = O.gae(r_t, d_t, 0.95, v_tm1=v, v_t=bv, truncation_t=trunc, time_major=True, standardize_advantages=False)
    for e in range(E):  # column by column: the scan runs over time only, environments are independent
        a1, t1 = O.gae(r_t[:, e : e + 1], d_t[:, e : e + 1], 0.95, v_tm1=v[:, e : e + 1], v_t=bv[:, e : e + 1],
                       truncation_t=trunc[:, e : e + 1], time_major=True, standardize_advantages=False)
        np.testing.assert_allclose(adv[:, e], a1[:, 0], rtol=1e-12)
        np.testing.assert_allclose(tgt[:, e], t1[:, 0], rtol=1e-12)


def test_next_row_configs_compose_and_resolve_targets():
    """default_rec_ppo / default_ff_sac / sebulba default_ff_ppo: the reference's group names, `_target_: stoix.*` strings resolve to the
    stoix_b200 classes (also through the `stoix` alias package), shape derivation fills the derived fields."""
    import stoix.networks.base as ref_base
    from stoix_b200.config import compose, instantiate
    from stoix_b200.networks import recurrent
    from stoix_b200.utils.total_timestep_checker import check_total_timesteps

    assert ref_base.ScannedRNN is recurrent.ScannedRNN and ref_base.RecurrentActor is recurrent.RecurrentActor
    c = compose("default_rec_ppo", ["arch.total_num_envs=64", "system.rollout_length=16", "arch.total_timesteps=4096"], config_dir="default/anakin")
    assert c.system.system_name == "rec_ppo" and c.system.recurrent_chunk_size is None and c.network.actor_network.rnn_layer.cell_type == "gru"
    rnn = instantiate(c.network.critic_network.rnn_layer)
    assert isinstance(rnn, recurrent.ScannedRNN) and rnn.hidden_state_dim == 128 and rnn.state_dim == 128
    assert recurrent.ScannedRNN(32, "lstm").state_dim == 64 and recurrent.ScannedRNN(32, "optimised_lstm").cell_type == "lstm"
    with pytest.raises(NotImplementedError):
        recurrent.ScannedRNN(32, "mgu")
    c.num_devices = 1
    c = check_total_timesteps(c, quiet=True)
    assert c.arch.num_envs == 64 and c.arch.num_updates == 4
    s = compose("default_ff_sac", ["arch.total_num_envs=128"], config_dir="default/anakin")
    assert s.system.tau == 0.005 and s.system.actor_lr == 3e-4 and s.network.q_network.pre_torso.use_layer_norm is True
    head = instantiate(s.network.actor_network.action_head, action_dim=6, minimum=-1.0, maximum=1.0)
    assert head.out_dim == 12 and head.kernel_blocks == (6, 6)
    b = compose("default_ff_ppo", ["arch.total_num_envs=512"], config_dir="default/sebulba")
    assert b.arch.architecture_name == "sebulba"


def test_recurrent_and_sac_arena_layouts_match_the_oracle_flat_order():
    """RecLayout (pre-torso | W_i | b_i | W_h | b_hn | post-torso | head) == oracle RecNet.flat(); SAC arena blocks are 8-float aligned."""
    from oracle import ppo_oracle as O
    from oracle import rec_oracle as R
    from stoix_b200.networks.recurrent import RecLayout
    from stoix_b200 import ops

    rng = np.random.default_rng(0)
    for cell, G in (("gru", 3), ("lstm", 4)):
        D, P, H, Q, A = 12, 24, 16, 20, 5
        lay = RecLayout(D, (P,), H, (Q,), A, "silu", False, "silu", False, cell)
        pre = O.MLPParams([rng.standard_normal((D, P)), rng.standard_normal((P, G * H))], [rng.standard_normal(P), rng.standard_normal(G * H)], "silu")
        post = O.MLPParams([rng.standard_normal((H, Q)), rng.standard_normal((Q, A))], [rng.standard_normal(Q), rng.standard_normal(A)], "silu")
        net = R.RecNet(pre, rng.standard_normal((H, G * H)), rng.standard_normal(H if cell == "gru" else 0), post)
        flat = net.flat()
        assert flat.size == lay.param_count and lay.S == (H if cell == "gru" else 2 * H) and lay.G == G
        np.testing.assert_array_equal(flat[lay.off_wh:lay.off_bhn].reshape(H, G * H), net.Wh)
        np.testing.assert_array_equal(flat[lay.off_post:lay.off_post + H * Q].reshape(H, Q), post.W[0])
        back = R.RecNet.from_flat(flat, lay.spec_pre.sizes, H, lay.spec_post.sizes, "silu")
        np.testing.assert_array_equal(back.flat(), flat)
        assert back.is_lstm == (cell == "lstm")
    from stoix_b200.systems.sac.ff_sac import sac_arena_layout

    sa = ops.MlpSpec((17, 256, 256, 256, 256, 12), activation="silu")
    sq = ops.MlpSpec((23, 256, 256, 256, 256, 1), activation="silu", use_layer_norm=True)
    lay = sac_arena_layout(sa, sq)
    assert all(lay[k] % 8 == 0 for k in ("actor", "q1", "q2", "alpha", "total")) and lay["q1"] >= sa.param_count
    assert lay["q2"] - lay["q1"] >= sq.param_count == 204801 and lay["q_block"] == lay["alpha"] - lay["q1"] and lay["total"] == lay["alpha"] + 8


def test_adam_plan_refuses_bad_segment_tables(monkeypatch):
    """include/stx.h: a segment offset is a float4 index (multiple of 4), counts >= 1, segments disjoint, 1..8 of them.  The table
    is refused before anything is allocated or the library is called (a misaligned plan would fault on the device instead)."""
    from stoix_b200 import _lib, ops

    def boom(*a, **k):
        raise AssertionError("AdamPlan allocated or called the library before checking its segment table")

    ok = ops.AdamPlan([(0, 10, 1e-3, 0.5), (12, 1, 1e-3, 0.5)], "cpu")   # adjacent after padding: accepted
    assert ok.end == 13 and ok.nseg == 2
    monkeypatch.setattr(_lib, "load", boom)
    monkeypatch.setattr(torch, "zeros", boom)
    monkeypatch.setattr(torch, "from_numpy", boom)
    bad = {
        "not a non-negative multiple of 4": [[(2, 10, 1e-3, 0.5)], [(0, 8, 1e-3, 0.5), (10, 4, 1e-3, 0.5)], [(-4, 8, 1e-3, 0.5)]],
        "has count": [[(0, 0, 1e-3, 0.5)], [(0, 8, 1e-3, 0.5), (8, -3, 1e-3, 0.5)]],
        "overlap": [[(0, 9, 1e-3, 0.5), (8, 4, 1e-3, 0.5)], [(16, 4, 1e-3, 0.5), (0, 20, 1e-3, 0.5)], [(0, 4, 1e-3, 0.5), (0, 4, 1e-3, 0.5)]],
        "segments": [[], [(8 * i, 4, 1e-3, 0.5) for i in range(9)]],
    }
    for msg, tables in bad.items():
        for segs in tables:
            with pytest.raises(_lib.StxError, match=msg):
                ops.AdamPlan(segs, "cpu")


def test_clip_adam_step_refuses_arenas_that_do_not_fit_the_plan(monkeypatch):
    """clip_adam_step checks dtype, contiguity and length of every arena against the plan before it calls the library."""
    from stoix_b200 import _lib, ops

    plan = ops.AdamPlan([(0, 10, 1e-3, 0.5), (16, 5, 1e-3, 0.5)], "cpu")   # last segment ends at 21

    def boom(*a, **k):
        raise AssertionError("clip_adam_step called the library before checking its arenas")

    monkeypatch.setattr(_lib, "load", boom)
    f = lambda n=24, dt=torch.float32: torch.zeros(n, dtype=dt)
    good = dict(params=f(), grads=f(), mu=f(), nu=f())
    cases = [
        (dict(params=f(dt=torch.float64)), "params must be a contiguous torch.float32"),
        (dict(grads=f(dt=torch.bfloat16)), "grads must be a contiguous torch.float32"),
        (dict(mu=f(48)[::2]), "mu must be a contiguous"),
        (dict(nu=f(20)), "nu holds 20 elements"),
        (dict(grads=f(21 - 1)), "grads holds 20 elements"),
        (dict(params_bf16=f()), "params_bf16 must be a contiguous torch.bfloat16"),
        (dict(params_bf16=f(16, torch.bfloat16)), "params_bf16 holds 16 elements"),
    ]
    for override, msg in cases:
        kw = dict(good, **override)
        with pytest.raises(_lib.StxError, match=msg):
            ops.clip_adam_step(plan, kw["params"], kw["grads"], kw["mu"], kw["nu"], params_bf16=kw.get("params_bf16"))
    # arenas that fit reach the next check: CPU tensors have no kernel
    with pytest.raises(_lib.StxError, match="only on CUDA"):
        ops.clip_adam_step(plan, f(21), f(21), f(21), f(21), params_bf16=f(21, torch.bfloat16))
