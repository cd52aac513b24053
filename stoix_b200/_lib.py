"""ctypes binding of libstoixb200.so (the C ABI declared in include/stx.h).

There is NO CPU fallback: importing the ops without the built library raises, and calling them
without a CUDA device raises.  `python -m stoix_b200.build` (or `__graft_entry__.build()`) builds
the library in-tree.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

STX_MAX_LAYERS = 7
STX_PREC_F32 = 0
STX_PREC_BF16 = 1

_LIB_PATH = Path(__file__).resolve().parent / "lib" / "libstoixb200.so"


class StxMlp(C.Structure):
    _fields_ = [
        ("n_layers", C.c_int32),
        ("sizes", C.c_int32 * (STX_MAX_LAYERS + 1)),
        ("params", C.c_void_p),
        ("params_bf16", C.c_void_p),
        ("activation", C.c_int32),
        ("use_layer_norm", C.c_int32),
    ]


STX_ACTIVATIONS = {"relu": 0, "tanh": 1, "silu": 2, "swish": 2, "elu": 3, "gelu": 4, "sigmoid": 5, "softplus": 6, "identity": 7, "none": 7}


class StxPpoHyper(C.Structure):
    _fields_ = [
        ("clip_eps", C.c_float),
        ("ent_coef", C.c_float),
        ("vf_coef", C.c_float),
        ("standardize_advantages", C.c_int32),
        ("overwrite_grads", C.c_int32),
        ("reserved", C.c_int32),
        ("adam_scratch", C.c_void_p),
    ]


class StxAdamSeg(C.Structure):
    _fields_ = [
        ("offset", C.c_int64),
        ("count", C.c_int64),
        ("init_lr", C.c_float),
        ("max_grad_norm", C.c_float),
    ]


class StxAdamHyper(C.Structure):
    _fields_ = [
        ("b1", C.c_float),
        ("b2", C.c_float),
        ("eps", C.c_float),
        ("grad_scale", C.c_float),
        ("decay", C.c_int32),
        ("steps_per_update", C.c_int32),
        ("num_updates", C.c_int32),
        ("prenorm", C.c_int32),
    ]


class StxRadamHyper(C.Structure):
    _fields_ = [
        ("adam", StxAdamHyper),
        ("eps_root", C.c_float),
        ("threshold", C.c_float),
    ]


class StxVtraceLoss(C.Structure):
    _fields_ = [
        ("logits", C.c_void_p),
        ("values", C.c_void_p),
        ("action", C.c_void_p),
        ("log_prob_b", C.c_void_p),
        ("reward", C.c_void_p),
        ("done", C.c_void_p),
        ("reward_stats", C.c_void_p),
        ("d_logits", C.c_void_p),
        ("d_value", C.c_void_p),
        ("metrics", C.c_void_p),
        ("ld", C.c_int64),
        ("T", C.c_int32),
        ("Em", C.c_int32),
        ("A", C.c_int32),
        ("gamma", C.c_float),
        ("lambda_", C.c_float),
        ("clip_rho", C.c_float),
        ("clip_pg_rho", C.c_float),
        ("ent_coef", C.c_float),
        ("vf_coef", C.c_float),
        ("reward_scale", C.c_float),
        ("reward_eps", C.c_float),
    ]


class StxEpsilonSchedule(C.Structure):
    _fields_ = [
        ("init_value", C.c_float),
        ("end_value", C.c_float),
        ("transition_steps", C.c_float),
        ("steps_per_update", C.c_int32),
        ("decay", C.c_int32),
        ("reserved", C.c_int32),
    ]


class StxReplay(C.Structure):
    _fields_ = [
        ("obs", C.c_void_p),
        ("action", C.c_void_p),
        ("reward", C.c_void_p),
        ("done", C.c_void_p),
        ("next_obs", C.c_void_p),
        ("state", C.c_void_p),
        ("capacity", C.c_int64),
        ("obs_dim", C.c_int32),
        ("act_dim", C.c_int32),
    ]


class StxReplayDiscrete(C.Structure):
    _fields_ = [
        ("obs", C.c_void_p),
        ("action", C.c_void_p),
        ("reward", C.c_void_p),
        ("done", C.c_void_p),
        ("next_obs", C.c_void_p),
        ("state", C.c_void_p),
        ("capacity", C.c_int64),
        ("obs_dim", C.c_int32),
        ("reserved", C.c_int32),
    ]


class StxQTdHyper(C.Structure):
    _fields_ = [
        ("gamma", C.c_float),
        ("max_abs_reward", C.c_float),
        ("huber_delta", C.c_float),
        ("entropy_temperature", C.c_float),
        ("munchausen_coefficient", C.c_float),
        ("clip_value_min", C.c_float),
        ("regularizer_coeff", C.c_float),
        ("reserved", C.c_int32),
    ]


class StxDistQHyper(C.Structure):
    _fields_ = [
        ("gamma", C.c_float),
        ("max_abs_reward", C.c_float),
        ("huber_delta", C.c_float),
        ("reserved", C.c_int32),
    ]


STX_NOISY_MAX_LAYERS = 8
STX_PRIO_FANOUT = 32


class StxNoisyLayer(C.Structure):
    _fields_ = [
        ("param", C.c_int64),
        ("eff_w", C.c_int64),
        ("eff_b", C.c_int64),
        ("noise", C.c_int64),
        ("in_", C.c_int32),
        ("out", C.c_int32),
        ("ld", C.c_int32),
        ("reserved", C.c_int32),
    ]


class StxNoisyNet(C.Structure):
    _fields_ = [
        ("layers", StxNoisyLayer * STX_NOISY_MAX_LAYERS),
        ("n_layers", C.c_int32),
        ("reserved", C.c_int32),
    ]


class StxReplayPrioritised(C.Structure):
    _fields_ = [
        ("obs", C.c_void_p),
        ("action", C.c_void_p),
        ("reward", C.c_void_p),
        ("done", C.c_void_p),
        ("next_obs", C.c_void_p),
        ("tree", C.c_void_p),
        ("state", C.c_void_p),
        ("max_priority", C.c_void_p),
        ("length", C.c_int64),
        ("envs", C.c_int32),
        ("obs_dim", C.c_int32),
        ("n_step", C.c_int32),
        ("priority_exponent", C.c_float),
        ("owner", C.c_void_p),
    ]


class StxPpoBatch(C.Structure):
    _fields_ = [
        ("obs", C.c_void_p),
        ("action", C.c_void_p),
        ("log_prob", C.c_void_p),
        ("value", C.c_void_p),
        ("advantages", C.c_void_p),
        ("targets", C.c_void_p),
        ("adv_stats", C.c_void_p),
        ("perm", C.c_void_p),
        ("B", C.c_int64),
    ]


class StxTanhNormalPpo(C.Structure):
    _fields_ = [
        ("action", C.c_void_p),
        ("eps_in", C.c_void_p),
        ("eps_out", C.c_void_p),
        ("dev_counter", C.c_void_p),
        ("seed", C.c_uint64),
        ("offset", C.c_uint64),
        ("minimum", C.c_float),
        ("maximum", C.c_float),
        ("min_scale", C.c_float),
        ("reserved", C.c_int32),
    ]


STX_PPO_KL_PENALTY = 1
STX_PPO_DPO = 2


class StxPpoVariant(C.Structure):
    _fields_ = [
        ("behaviour", C.c_void_p),
        ("kind", C.c_int32),
        ("kl_coef", C.c_float),
        ("dpo_alpha", C.c_float),
        ("dpo_beta", C.c_float),
    ]



STX_VMPO_CATEGORICAL = 0
STX_VMPO_TANH_NORMAL = 1
STX_VMPO_MAX_A = 32
STX_VMPO_METRICS = 9


class StxVmpoLoss(C.Structure):
    _fields_ = [
        ("kind", C.c_int32),
        ("A", C.c_int32),
        ("per_dim", C.c_int32),
        ("overwrite", C.c_int32),
        ("N", C.c_int64),
        ("value_rows", C.c_int64),
        ("head", C.c_void_p),
        ("head_target", C.c_void_p),
        ("action", C.c_void_p),
        ("action_cont", C.c_void_p),
        ("adv", C.c_void_p),
        ("mask", C.c_void_p),
        ("count", C.c_void_p),
        ("value", C.c_void_p),
        ("targets", C.c_void_p),
        ("duals", C.c_void_p),
        ("d_head", C.c_void_p),
        ("d_value", C.c_void_p),
        ("dual_grad", C.c_void_p),
        ("metrics", C.c_void_p),
        ("epsilon", C.c_float),
        ("epsilon_alpha", C.c_float),
        ("epsilon_stddev", C.c_float),
        ("weight", C.c_float),
        ("minimum", C.c_float),
        ("maximum", C.c_float),
        ("min_scale", C.c_float),
        ("reserved", C.c_int32),
    ]


STX_MPO_CATEGORICAL = 0
STX_MPO_TANH_NORMAL = 1
STX_MPO_MAX_A = 32
STX_MPO_METRICS = 14


class StxSeqRing(C.Structure):
    _fields_ = [("obs", C.c_void_p), ("action", C.c_void_p), ("reward", C.c_void_p), ("done", C.c_void_p), ("truncated", C.c_void_p),
                ("log_prob", C.c_void_p), ("state", C.c_void_p), ("length", C.c_int64), ("envs", C.c_int32), ("obs_dim", C.c_int32),
                ("act_words", C.c_int32), ("reserved", C.c_int32)]


class StxMpoRows(C.Structure):
    _fields_ = [("kind", C.c_int32), ("A", C.c_int32), ("N", C.c_int32), ("D", C.c_int32), ("M", C.c_int64), ("NL", C.c_int32),
                ("stochastic", C.c_int32), ("seed", C.c_uint64), ("obs", C.c_void_p), ("logits_t", C.c_void_p), ("logits_b", C.c_void_p),
                ("action", C.c_void_p), ("log_prob", C.c_void_p), ("reward", C.c_void_p), ("done", C.c_void_p), ("act_in", C.c_void_p),
                ("act_out", C.c_void_p), ("eps_in", C.c_void_p), ("act_cont_out", C.c_void_p), ("xq", C.c_void_p), ("log_rho", C.c_void_p),
                ("r", C.c_void_p), ("d", C.c_void_p), ("gamma", C.c_float), ("max_abs_reward", C.c_float), ("minimum", C.c_float),
                ("maximum", C.c_float), ("min_scale", C.c_float), ("reserved", C.c_int32)]


class StxMpoLoss(C.Structure):
    _fields_ = [("kind", C.c_int32), ("A", C.c_int32), ("N", C.c_int32), ("overwrite", C.c_int32), ("M", C.c_int64), ("NL", C.c_int32),
                ("per_dim", C.c_int32), ("head", C.c_void_p), ("head_target", C.c_void_p), ("q", C.c_void_p), ("actions", C.c_void_p),
                ("q_boot", C.c_void_p), ("duals", C.c_void_p), ("v", C.c_void_p), ("d_head", C.c_void_p), ("dual_grad", C.c_void_p),
                ("metrics", C.c_void_p), ("epsilon", C.c_float), ("epsilon_policy", C.c_float), ("epsilon_stddev", C.c_float),
                ("weight", C.c_float), ("minimum", C.c_float), ("maximum", C.c_float), ("min_scale", C.c_float), ("reserved", C.c_int32)]


STX_LN_TORSO = 1
STX_LN_FINAL = 2
STX_R2D2_METRICS = 6
STX_VTRACE_METRICS = 5


class StxR2d2Ring(C.Structure):
    _fields_ = [("obs", C.c_void_p), ("action", C.c_void_p), ("reward", C.c_void_p), ("done", C.c_void_p), ("truncated", C.c_void_p),
                ("reset", C.c_void_p), ("carry", C.c_void_p), ("tree", C.c_void_p), ("state", C.c_void_p), ("max_priority", C.c_void_p),
                ("owner", C.c_void_p), ("length", C.c_int64), ("envs", C.c_int32), ("obs_dim", C.c_int32), ("carry_dim", C.c_int32),
                ("seq_len", C.c_int32), ("period", C.c_int32), ("priority_exponent", C.c_float)]


class StxR2d2Loss(C.Structure):
    _fields_ = [("T", C.c_int32), ("B", C.c_int32), ("A", C.c_int32), ("n", C.c_int32), ("q", C.c_void_p), ("q_target", C.c_void_p),
                ("action", C.c_void_p), ("reward", C.c_void_p), ("done", C.c_void_p), ("prob", C.c_void_p), ("count", C.c_void_p),
                ("d_q", C.c_void_p), ("priorities", C.c_void_p), ("metrics", C.c_void_p), ("td", C.c_void_p), ("gamma", C.c_float),
                ("max_abs_reward", C.c_float), ("eta", C.c_float), ("tx_eps", C.c_float), ("beta0", C.c_float), ("beta_steps", C.c_float),
                ("weight", C.c_float), ("reserved", C.c_int32)]


_P = C.c_void_p
_SIGNATURES = {
    # name: (restype, argtypes)
    "stx_version": (C.c_int, []),
    "stx_last_error_string": (C.c_char_p, []),
    "stx_launch_count": (C.c_ulonglong, []),
    "stx_tc_trap_message": (C.c_char_p, []),
    "stx_debug_callfree_math": (C.c_int, [C.c_int, C.c_uint32, C.c_uint32, _P, _P]),
    "stx_mlp_param_count": (C.c_int64, [C.POINTER(StxMlp)]),
    "stx_gae_scratch_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "stx_gae_set_tuning": (C.c_int, [C.c_int]),
    "stx_gae_ppo_f32": (C.c_int, [_P, _P, _P, _P, _P, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.c_int, _P, _P, _P, _P, _P]),
    "stx_gae_generic_f32": (C.c_int, [_P, _P, _P, C.c_float, _P, _P, _P, C.c_int, C.c_int, C.c_int, _P, _P, _P, _P, _P]),
    "stx_mlp_forward_workspace_bytes": (C.c_size_t, [C.POINTER(StxMlp), C.c_int64, C.c_int]),
    "stx_mlp_forward": (C.c_int, [C.POINTER(StxMlp), _P, C.c_int64, _P, C.c_int64, _P, C.c_int, _P, C.c_size_t, _P]),
    "stx_tc_debug_forward": (C.c_int, [C.POINTER(StxMlp), _P, C.c_int64, C.c_int64, _P, _P, _P, _P]),
    "stx_tc_debug_set_prof_buffer": (C.c_int, [_P]),
    "stx_tc_set_forward_ctas": (None, [C.c_int]),
    "stx_categorical": (C.c_int, [_P, C.c_int64, C.c_int, C.c_int, C.c_uint64, C.c_uint64, _P, _P, _P, _P, _P]),
    "stx_ppo_arena_offsets": (None, [C.POINTER(StxMlp), C.POINTER(StxMlp), C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "stx_ppo_workspace_bytes": (C.c_size_t, [C.POINTER(StxMlp), C.POINTER(StxMlp), C.c_int64, C.c_int]),
    "stx_ppo_minibatch_grads": (C.c_int, [C.POINTER(StxMlp), C.POINTER(StxMlp), C.POINTER(StxPpoBatch), C.c_int64, C.c_int64, C.POINTER(StxPpoHyper), C.c_float, _P, _P, C.c_int, _P, C.c_size_t, _P]),
    "stx_loss_scratch_bytes": (C.c_size_t, []),
    "stx_ppo_clip_loss": (C.c_int, [_P, _P, _P, C.c_int64, C.c_float, _P, _P, _P]),
    "stx_clipped_value_loss": (C.c_int, [_P, _P, _P, C.c_int64, C.c_float, _P, _P, _P]),
    "stx_adam_scratch_bytes": (C.c_size_t, [C.c_int]),
    "stx_clip_adam_step": (C.c_int, [_P, _P, _P, _P, _P, _P, C.c_int, C.POINTER(StxAdamHyper), _P, _P, _P, _P]),
    "stx_allreduce_clip_adam_step": (C.c_int, [_P, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.c_int, C.c_int, C.c_int, _P, _P, _P, _P, _P,
                                                C.c_int, C.POINTER(StxAdamHyper), _P, _P, _P, _P]),
    "stx_make_permutation": (C.c_int, [_P, C.c_int64, C.c_uint64, C.c_uint64, _P, _P]),
    "stx_counter_add": (C.c_int, [_P, C.c_uint64, _P]),
    "stx_synth_env_step": (C.c_int, [C.c_int64, C.c_int, C.c_uint64, C.c_uint64, _P, C.c_float, C.c_float, _P, _P, _P, C.c_int, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "stx_synth_env_trajectory": (C.c_int, [C.c_int64, C.c_int, C.c_int, C.c_uint64, C.c_uint64, _P, C.c_float, C.c_float] + [_P] * 11),
    "stx_tc_rollout_policy": (C.c_int, [C.POINTER(StxMlp), _P, _P, _P, C.c_int, C.c_int64, C.c_uint64, C.c_uint64, _P, C.c_int, _P]),
    "stx_tc_rollout_values_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int64, C.c_int]),
    "stx_tc_rollout_values": (C.c_int, [C.POINTER(StxMlp), _P, _P, _P, C.c_int, C.c_int64, _P, _P, _P, C.c_size_t, _P]),
    "stx_tc_rollout_synth": (C.c_int, [C.POINTER(StxMlp)] + [_P] * 12 + [C.c_int, C.c_int64, C.c_uint64, C.c_uint64, _P, C.c_float, C.c_float,
                                        C.c_uint64, C.c_uint64, _P, _P]),
    "stx_cast_f32_to_bf16": (C.c_int, [_P, _P, C.c_int64, _P]),
    "stx_mlp_train_workspace_bytes": (C.c_size_t, [C.POINTER(StxMlp), C.c_int64]),
    "stx_mlp_forward_train": (C.c_int, [C.POINTER(StxMlp), _P, C.c_int64, _P, C.c_int64, _P, _P, C.c_size_t, _P]),
    "stx_mlp_backward": (C.c_int, [C.POINTER(StxMlp), _P, C.c_int64, _P, C.c_int64, _P, _P, C.c_size_t, C.c_float, _P, C.c_int, _P, _P]),
    "stx_tanh_normal_sample": (C.c_int, [_P, C.c_int64, C.c_int, _P, C.c_uint64, C.c_uint64, _P, C.c_float, C.c_float, C.c_float, _P, C.c_int64,
                                         _P, _P, _P]),
    "stx_tanh_normal_backward": (C.c_int, [_P, _P, C.c_int64, C.c_int, C.c_float, C.c_float, C.c_float, _P, C.c_float, _P, C.c_int64, _P, _P]),
    "stx_sac_actor_seed": (C.c_int, [_P, _P, _P, _P, C.c_int64, _P, _P, _P, C.c_float, _P]),
    "stx_sac_q_loss": (C.c_int, [_P] * 8 + [C.c_float, C.c_int64, _P, _P, _P, C.c_float, _P]),
    "stx_sac_alpha_grad": (C.c_int, [_P, _P, C.c_float, C.c_int64, C.c_int, _P, C.c_float, C.c_int, _P, C.c_float, _P]),
    "stx_polyak_update": (C.c_int, [_P, _P, C.c_int64, C.c_float, _P]),
    "stx_uniform_indices": (C.c_int, [_P, C.c_int64, C.c_uint64, C.c_uint64, _P, _P, _P]),
    "stx_gather_rows_f32": (C.c_int, [_P, _P, C.c_int64, C.c_int, _P, C.c_int64, _P]),
    "stx_gather_u8": (C.c_int, [_P, _P, C.c_int64, _P, _P]),
    "stx_gru_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int64, C.c_int]),
    "stx_gru_sequence_forward": (C.c_int, [_P, _P, _P, _P, _P, C.c_int, C.c_int64, C.c_int, _P, _P, C.c_size_t, _P]),
    "stx_gru_sequence_backward": (C.c_int, [_P, _P, _P, C.c_int, C.c_int64, C.c_int, _P, C.c_size_t, _P, _P, _P, C.c_float, C.c_int, _P, _P]),
    "stx_lstm_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int64, C.c_int]),
    "stx_lstm_sequence_forward": (C.c_int, [_P, _P, _P, _P, C.c_int, C.c_int64, C.c_int, _P, _P, _P, C.c_size_t, _P]),
    "stx_lstm_sequence_backward": (C.c_int, [_P, _P, _P, C.c_int, C.c_int64, C.c_int, _P, C.c_size_t, _P, _P, C.c_float, C.c_int, _P, _P]),
    "stx_ppo_head_scratch_bytes": (C.c_size_t, [C.c_int64]),
    "stx_ppo_head_grads": (C.c_int, [_P, _P, _P, C.c_int64, _P, _P, _P, _P, _P, _P, C.c_int64, C.c_int, C.c_float, C.c_float, C.c_float, _P, _P, _P,
                                     C.c_float, _P, _P]),
    "stx_replay_add": (C.c_int, [_P, _P, _P, _P, _P, _P, C.c_int64, _P]),
    "stx_replay_sample": (C.c_int, [_P, C.c_int64, C.c_uint64, C.c_uint64, _P, _P, _P, _P, _P, C.c_int64, _P, _P, _P, _P]),
    "stx_running_stats_scratch_bytes": (C.c_size_t, [C.c_int]),
    "stx_running_stats_accumulate": (C.c_int, [_P, _P, C.c_int64, C.c_int, _P, _P, _P, _P]),
    "stx_running_stats_finalize": (C.c_int, [_P, C.c_int, _P, _P, _P, _P, C.c_float, C.c_float, _P]),
    "stx_obs_normalize": (C.c_int, [_P, C.c_int64, C.c_int, _P, _P, C.c_float, _P, C.c_int, _P]),
    "stx_tanh_normal_log_prob": (C.c_int, [_P, C.c_int64, C.c_int, _P, C.c_int64, C.c_float, C.c_float, C.c_float, _P, _P]),
    "stx_tanh_normal_entropy": (C.c_int, [_P, C.c_int64, C.c_int, _P, C.c_uint64, C.c_uint64, _P, C.c_float, C.c_float, C.c_float, _P, _P, _P]),
    "stx_ppo_tanh_normal_head_grads": (C.c_int, [_P, _P, C.c_int64, C.POINTER(StxTanhNormalPpo), _P, _P, _P, C.c_int64, C.c_int, C.c_float,
                                                 C.c_float, _P, _P, C.c_float, _P, _P]),
    "stx_ppo_continuous_minibatch_grads": (C.c_int, [C.POINTER(StxMlp), C.POINTER(StxMlp), C.POINTER(StxPpoBatch), C.POINTER(StxTanhNormalPpo),
                                                     C.c_int64, C.c_int64, C.POINTER(StxPpoHyper), C.c_float, _P, _P, C.c_int, _P, C.c_size_t, _P]),
    "stx_categorical_kl": (C.c_int, [_P, _P, C.c_int64, C.c_int, _P, _P]),
    "stx_tanh_normal_kl": (C.c_int, [_P, _P, C.c_int64, C.c_int, C.c_float, _P, _P]),
    "stx_ppo_penalty_loss": (C.c_int, [_P, _P, _P, _P, C.c_int64, C.c_float, _P, _P, _P]),
    "stx_dpo_loss": (C.c_int, [_P, _P, _P, C.c_int64, C.c_float, C.c_float, _P, _P, _P]),
    "stx_ppo_penalty_head_grads": (C.c_int, [_P, _P, C.c_int64, C.POINTER(StxPpoVariant), _P, _P, _P, _P, C.c_int64, C.c_int, C.c_float, _P, _P,
                                             C.c_float, _P, _P]),
    "stx_ppo_variant_tanh_normal_head_grads": (C.c_int, [_P, _P, C.c_int64, C.POINTER(StxTanhNormalPpo), C.POINTER(StxPpoVariant), _P, _P, _P,
                                                         C.c_int64, C.c_int, C.c_float, _P, _P, C.c_float, _P, _P]),
    "stx_ppo_penalty_minibatch_grads": (C.c_int, [C.POINTER(StxMlp), C.POINTER(StxMlp), C.POINTER(StxPpoBatch), C.POINTER(StxPpoVariant),
                                                  C.c_int64, C.c_int64, C.POINTER(StxPpoHyper), C.c_float, _P, _P, C.c_int, _P, C.c_size_t, _P]),
    "stx_ppo_variant_continuous_minibatch_grads": (C.c_int, [C.POINTER(StxMlp), C.POINTER(StxMlp), C.POINTER(StxPpoBatch),
                                                             C.POINTER(StxTanhNormalPpo), C.POINTER(StxPpoVariant), C.c_int64, C.c_int64,
                                                             C.POINTER(StxPpoHyper), C.c_float, _P, _P, C.c_int, _P, C.c_size_t, _P]),
    "stx_epsilon_greedy": (C.c_int, [_P, C.c_int64, C.c_int, C.c_int, C.c_uint64, C.c_uint64, _P, _P, C.POINTER(StxEpsilonSchedule), _P, _P, _P,
                                     _P]),
    "stx_q_lambda_f32": (C.c_int, [_P, C.c_int, _P, _P, _P, C.c_int, C.c_int, C.c_float, C.c_float, _P, _P]),
    "stx_lambda_returns_f32": (C.c_int, [_P, _P, _P, C.c_int, _P, C.c_float, C.c_int, C.c_int, _P, _P]),
    "stx_q_loss_grads": (C.c_int, [_P, _P, C.c_int64, _P, _P, C.c_int64, C.c_int, C.c_float, _P, _P, C.c_float, _P, _P]),
    "stx_clip_radam_step": (C.c_int, [_P, _P, _P, _P, _P, _P, C.c_int, C.POINTER(StxRadamHyper), _P, _P, _P, _P]),
    "stx_replay_add_discrete": (C.c_int, [C.POINTER(StxReplayDiscrete), _P, _P, _P, _P, _P, C.c_int64, _P]),
    "stx_replay_sample_discrete": (C.c_int, [C.POINTER(StxReplayDiscrete), C.c_int64, C.c_uint64, C.c_uint64, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "stx_q_td_loss_grads": (C.c_int, [C.c_int, _P, _P, _P, _P, _P, _P, _P, C.c_int64, C.c_int, C.POINTER(StxQTdHyper), _P, _P, C.c_float, _P, _P]),
    "stx_dist_q_scratch_bytes": (C.c_size_t, [C.c_int64]),
    "stx_dist_q_values": (C.c_int, [C.c_int, _P, C.c_int64, C.c_int, C.c_int, _P, _P, _P]),
    "stx_categorical_q_loss_grads": (C.c_int, [_P, _P, _P, _P, C.c_int64, _P, C.c_int64, _P, _P, _P, _P, C.c_int64, C.c_int, C.c_int,
                                               C.POINTER(StxDistQHyper), _P, _P, _P, C.c_float, _P, _P]),
    "stx_quantile_q_loss_grads": (C.c_int, [_P, _P, _P, _P, C.c_int64, _P, _P, _P, _P, C.c_int64, C.c_int, C.c_int, C.POINTER(StxDistQHyper), _P,
                                            _P, _P, C.c_float, _P, _P]),
    "stx_categorical_q_loss_grads_weighted": (C.c_int, [_P, _P, _P, _P, C.c_int64, _P, C.c_int64, _P, _P, _P, _P, _P, C.c_int64, C.c_int, C.c_int,
                                                        C.POINTER(StxDistQHyper), _P, _P, _P, C.c_float, _P, _P]),
    "stx_noisy_weights": (C.c_int, [C.POINTER(StxNoisyNet), _P, _P, _P, C.c_int, C.c_uint64, C.c_uint64, _P, _P]),
    "stx_noisy_fold": (C.c_int, [C.POINTER(StxNoisyNet), _P, _P, _P, C.c_int, _P]),
    "stx_dueling_combine": (C.c_int, [_P, C.c_int64, C.c_int, C.c_int, _P, _P]),
    "stx_dueling_backward": (C.c_int, [_P, C.c_int64, C.c_int, C.c_int, _P, _P]),
    "stx_prio_tree_floats": (C.c_int64, [C.c_int64]),
    "stx_prio_scratch_bytes": (C.c_size_t, []),
    "stx_replay_add_prioritised": (C.c_int, [C.POINTER(StxReplayPrioritised), _P, _P, _P, _P, _P, C.c_int, _P]),
    "stx_replay_sample_prioritised": (C.c_int, [C.POINTER(StxReplayPrioritised), C.c_int64, C.c_uint64, C.c_uint64, _P, _P, _P, C.c_float, C.c_float,
                                                C.c_float, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "stx_replay_set_priorities": (C.c_int, [C.POINTER(StxReplayPrioritised), _P, _P, C.c_int64, _P]),
    "stx_vmpo_topk_scratch_bytes": (C.c_size_t, []),
    "stx_vmpo_topk": (C.c_int, [_P, C.c_int64, C.c_int64, _P, _P, _P, _P, _P]),
    "stx_vmpo_loss_scratch_bytes": (C.c_size_t, []),
    "stx_vmpo_loss_grads": (C.c_int, [C.POINTER(StxVmpoLoss), _P, _P]),
    "stx_vmpo_after_step": (C.c_int, [_P, C.c_int, _P, _P, C.c_int64, _P, C.c_int, _P]),
    "stx_n_step_returns_f32": (C.c_int, [_P, _P, _P, _P, C.c_int, C.c_int, C.c_int, C.c_float, _P, _P, _P]),
    "stx_replay_add_sequence": (C.c_int, [C.POINTER(StxSeqRing), _P, _P, _P, _P, _P, _P, C.c_int, _P]),
    "stx_replay_sample_sequence": (C.c_int, [C.POINTER(StxSeqRing), C.c_int, C.c_int, C.c_int, C.c_uint64, C.c_uint64, _P, _P, _P, _P, _P, _P, _P,
                                             _P, _P]),
    "stx_mpo_sample_actions": (C.c_int, [C.POINTER(StxMpoRows), C.c_uint64, _P, _P]),
    "stx_mpo_loss_scratch_bytes": (C.c_size_t, []),
    "stx_mpo_loss_grads": (C.c_int, [C.POINTER(StxMpoLoss), _P, _P]),
    "stx_retrace_f32": (C.c_int, [_P, _P, _P, _P, _P, _P, C.c_float, C.c_int, C.c_int, _P, _P]),
    "stx_mpo_q_grad": (C.c_int, [_P, _P, C.c_int, C.c_int, _P, _P, C.c_float, _P]),
    "stx_r2d2_tree_floats": (C.c_int64, [C.POINTER(StxR2d2Ring)]),
    "stx_r2d2_ring_add": (C.c_int, [C.POINTER(StxR2d2Ring), _P, _P, _P, _P, _P, _P, _P, C.c_int, _P]),
    "stx_r2d2_ring_sample": (C.c_int, [C.POINTER(StxR2d2Ring), C.c_int, C.c_uint64, C.c_uint64, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "stx_r2d2_ring_set_priorities": (C.c_int, [C.POINTER(StxR2d2Ring), _P, _P, C.c_int64, _P]),
    "stx_r2d2_value_transform": (C.c_int, [_P, C.c_int64, C.c_int, C.c_float, _P, _P]),
    "stx_r2d2_loss_scratch_bytes": (C.c_size_t, [C.c_int]),
    "stx_r2d2_loss_grads": (C.c_int, [C.POINTER(StxR2d2Loss), _P, _P]),
    "stx_dueling_q": (C.c_int, [_P, _P, C.c_int64, C.c_int, _P, _P]),
    "stx_dueling_q_backward": (C.c_int, [_P, C.c_int64, C.c_int, _P, _P, C.c_float, C.c_int, _P]),
    "stx_reward_stats": (C.c_int, [_P, C.c_int, C.c_int, C.c_int64, _P, _P]),
    "stx_clip_rmsprop_step": (C.c_int, [_P, _P, _P, _P, _P, C.c_int, C.POINTER(StxAdamHyper), _P, _P, _P, _P]),
    "stx_vtrace_loss_scratch_bytes": (C.c_size_t, []),
    "stx_vtrace_loss_grads": (C.c_int, [C.POINTER(StxVtraceLoss), _P, _P]),
}

_lib = None


class StxError(RuntimeError):
    pass


def library_path() -> Path:
    return _LIB_PATH


def declared_symbols():
    """Names this binding expects; tests cross-check them against include/stx.h."""
    return sorted(_SIGNATURES)


def load():
    """Load the shared library (once).  Raises StxError if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not _LIB_PATH.exists():
        raise StxError(
            f"{_LIB_PATH} is missing: build it with `python -m stoix_b200.build` "
            "(there is no CPU or PyTorch fallback for the stoix_b200 kernels)"
        )
    lib = C.CDLL(os.fspath(_LIB_PATH))
    for name, (res, args) in _SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = load().stx_last_error_string()
        trap = load().stx_tc_trap_message()
        raise StxError(f"{what} failed (rc={rc}): {msg.decode() if msg else ''}" + (f" [{trap.decode()}]" if trap else ""))
