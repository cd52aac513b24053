"""CPU oracle for continuous-action PPO (stoix/systems/ppo/anakin/ff_ppo_continuous.py)  --  TEST INFRASTRUCTURE, NOT PRODUCT.

fp64 NumPy restatement of `_actor_loss_fn` for the tanh-Normal head (:191-213): log_prob of a GIVEN action
(stoix/networks/distributions.py:56-80, the inverse path with the clipped tails), the clipped surrogate, the seeded entropy
estimate `entropy(seed)` (distributions.py:85-88) with its noise injected, and hand-derived d(loss)/d(head output); plus
the update step and the network part of the rollout with float actions.  The tanh-Normal formulas come from
oracle/sac_oracle.py (head_sample, head_log_prob_grad); the networks, GAE, critic loss and optimiser from oracle/ppo_oracle.py.
The gradients are checked against torch.autograd in tests/test_oracle_ppo_continuous.py.

`entropy_noise` regenerates the kernels' Philox draws of the entropy noise (counter layout in include/stx.h)."""
from __future__ import annotations

from typing import Dict, Tuple

import numpy as np

from oracle import ppo_oracle as O
from oracle import sac_oracle as S
from oracle.synth_env import normal2, philox4x32

TAG_PPO_ENTROPY = 0x50504F45
EPSILON = 1e-3


def entropy_noise(seed: int, rows: int, A: int, call: int) -> np.ndarray:
    """(rows, A) float32 noise eps' of stx_ppo_continuous_minibatch_grads / stx_tanh_normal_entropy for row index 0..rows-1."""
    groups = (A + 3) // 4
    m = np.arange(rows, dtype=np.uint64)[:, None]
    g = np.arange(groups, dtype=np.uint64)[None, :]
    c2 = (np.uint64(call >> 32) ^ (g << np.uint64(20)) ^ ((m >> np.uint64(32)) << np.uint64(8))) & np.uint64(0xFFFFFFFF)
    r = philox4x32(m, np.uint64(call & 0xFFFFFFFF), c2, np.uint64(TAG_PPO_ENTROPY), seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    a0, a1 = normal2(r[0], r[1])
    b0, b1 = normal2(r[2], r[3])
    return np.stack([a0, a1, b0, b1], axis=-1).reshape(rows, groups * 4)[:, :A]


def _geometry(minimum: float, maximum: float):
    s, sh = (maximum - minimum) / 2.0, (minimum + maximum) / 2.0
    return s, sh, minimum + EPSILON, maximum - EPSILON


def log_prob_given(head_out: np.ndarray, action: np.ndarray, minimum: float, maximum: float, min_scale: float = 1e-3):
    """log_prob(action) per row and d log_prob / d(head output) (rows, 2A) with the action held fixed.

    The event is handed to sac_oracle.head_sample as the noise that reproduces it (tails: a sample well beyond the clip band),
    so the value comes from the very formulas of the SAC oracle.  Derivative inside the band: z = (atanh(..) - loc)/sigma,
    d/dloc = z/sigma, d/dsigma = (z^2 - 1)/sigma; in the tails the event is a constant in both paths, so the Mills-ratio terms
    of head_log_prob_grad apply unchanged."""
    A = head_out.shape[-1] // 2
    loc, raw = head_out[..., :A], head_out[..., A:]
    sigma = S.softplus(raw) + min_scale
    s, sh, lo, hi = _geometry(minimum, maximum)
    ev = np.clip(action, lo, hi)
    band = (ev > lo) & (ev < hi)
    u_lo, u_hi = np.arctanh((lo - sh) / s), np.arctanh((hi - sh) / s)
    u = np.where(band, np.arctanh(np.clip((ev - sh) / s, -1 + 1e-15, 1 - 1e-15)), np.where(ev <= lo, u_lo - 10.0, u_hi + 10.0))
    t = S.head_sample(head_out, (u - loc) / sigma, minimum, maximum, min_scale, EPSILON)
    assert np.array_equal(t.branch == 0, band)
    ones = np.ones(head_out.shape[:-1])
    tails = S.head_log_prob_grad(t, ones, np.zeros_like(loc), minimum, maximum, EPSILON)
    z = np.where(band, (u - loc) / sigma, 0.0)
    d_loc = np.where(band, z / sigma, tails[..., :A])
    d_raw = np.where(band, (z * z - 1.0) / sigma * S.sigmoid(raw), tails[..., A:])
    return t.log_prob, np.concatenate([d_loc, d_raw], axis=-1)


def fldj_tanh(x):
    return 2.0 * (np.log(2.0) - x - S.softplus(-2.0 * x))


def entropy_estimate(head_out: np.ndarray, eps: np.ndarray, minimum: float, maximum: float, min_scale: float = 1e-3):
    """entropy(seed) per row = sum_j [Normal entropy + log s + fldj_tanh(loc + sigma eps')] and its gradient (eps' fixed):
    dH/dloc = -2 tanh(u'), dH/dsigma = 1/sigma - 2 tanh(u') eps'."""
    A = head_out.shape[-1] // 2
    loc, raw = head_out[..., :A], head_out[..., A:]
    sigma = S.softplus(raw) + min_scale
    s = (maximum - minimum) / 2.0
    u = loc + sigma * eps
    H = (0.5 + S.LOG_SQRT_2PI + np.log(sigma) + np.log(s) + fldj_tanh(u)).sum(-1)
    th = np.tanh(u)
    dH = np.concatenate([-2.0 * th, (1.0 / sigma - 2.0 * th * eps) * S.sigmoid(raw)], axis=-1)
    return H, dH


def actor_loss_and_dhead(head_out, action, logp_old, adv, clip_eps, ent_coef, eps, minimum, maximum, min_scale=1e-3):
    """_actor_loss_fn (ff_ppo_continuous.py:191-213): ppo_clip_loss - ent_coef * mean(entropy(seed)), and d/d(head output).
    Branch / tie rule of the surrogate as in ppo_oracle.actor_loss_and_dlogits."""
    m = head_out.shape[0]
    lp, dlp = log_prob_given(head_out, action, minimum, maximum, min_scale)
    ratio = np.exp(lp - logp_old)
    l1 = ratio * adv
    l2 = np.clip(ratio, 1.0 - clip_eps, 1.0 + clip_eps) * adv
    loss_actor = (-np.minimum(l1, l2)).mean()
    H, dH = entropy_estimate(head_out, eps, minimum, maximum, min_scale)
    in_band = (ratio >= 1.0 - clip_eps) & (ratio <= 1.0 + clip_eps)
    dlogp = np.where((l1 < l2) | in_band, -adv * ratio, 0.0) / m
    dhead = dlogp[:, None] * dlp - (ent_coef / m) * dH
    info = {"actor_loss": loss_actor, "entropy": H.mean(), "advantages": adv.mean()}
    return loss_actor - ent_coef * H.mean(), dhead, info


def evaluate_rollout(actor: O.MLPParams, critic: O.MLPParams, traj: O.Trajectory, minimum: float, maximum: float, min_scale: float = 1e-3):
    """The network part of _env_step (ff_ppo_continuous.py:98-101, 113-116) on recorded obs / float actions (T, E, A)."""
    T, E, D = traj.obs.shape
    head, _ = O.mlp_forward(actor, traj.obs.reshape(T * E, D))
    traj.log_prob = log_prob_given(head, traj.action.reshape(T * E, -1), minimum, maximum, min_scale)[0].reshape(T, E)
    v, _ = O.mlp_forward(critic, traj.obs.reshape(T * E, D))
    traj.value = v[:, 0].reshape(T, E)
    bv, _ = O.mlp_forward(critic, traj.next_obs.reshape(T * E, D))
    traj.bootstrap_value = bv[:, 0].reshape(T, E)
    return traj


def ppo_update(actor: O.MLPParams, critic: O.MLPParams, a_state: O.AdamState, c_state: O.AdamState, traj: O.Trajectory, perms: np.ndarray,
               h: O.PPOHyper, eps: np.ndarray, minimum: float, maximum: float,
               min_scale: float = 1e-3) -> Tuple[O.MLPParams, O.MLPParams, Dict[str, np.ndarray], np.ndarray, np.ndarray]:
    """ppo_oracle.ppo_update with the tanh-Normal actor: float actions (T, E, A) and the entropy noise of every minibatch
    injected as eps (epochs, num_minibatches, mb, A)."""
    dt = traj.reward.dtype
    T, E, D = traj.obs.shape
    r_t, d_t, trunc = O.ppo_gae_inputs(traj.reward, traj.done, traj.truncated, h.gamma, h.reward_scale, dt.type)
    adv, targets = O.gae(r_t, d_t, h.gae_lambda, v_tm1=traj.value, v_t=traj.bootstrap_value, truncation_t=trunc, time_major=True,
                         standardize_advantages=h.standardize_advantages, dtype=dt.type)
    B = T * E
    mb = B // h.num_minibatches
    obs, act = traj.obs.reshape(B, D), traj.action.reshape(B, -1)
    lp_old, v_old, adv_f, tgt_f = (x.reshape(B) for x in (traj.log_prob, traj.value, adv, targets))
    sizes_a = [actor.W[0].shape[0]] + [w.shape[1] for w in actor.W]
    sizes_c = [critic.W[0].shape[0]] + [w.shape[1] for w in critic.W]
    names = ("actor_loss", "entropy", "value_loss", "advantages")
    metrics = {k: np.zeros((h.epochs, h.num_minibatches), dt) for k in names}
    for ep in range(h.epochs):
        for i in range(h.num_minibatches):
            idx = perms[ep][i * mb:(i + 1) * mb]
            head, a_acts = O.mlp_forward(actor, obs[idx])
            _, dhead, a_info = actor_loss_and_dhead(head, act[idx], lp_old[idx], adv_f[idx], h.clip_eps, h.ent_coef, eps[ep, i], minimum, maximum,
                                                    min_scale)
            a_g = O.mlp_backward(actor, a_acts, dhead).flat()
            v, c_acts = O.mlp_forward(critic, obs[idx])
            _, dvalue, c_info = O.critic_loss_and_dvalue(v[:, 0], v_old[idx], tgt_f[idx], h.clip_eps, h.vf_coef)
            c_g = O.mlp_backward(critic, c_acts, dvalue[:, None]).flat()
            a_lr = O.linear_schedule(h.actor_lr, a_state.sched_count, h.num_updates, h.epochs, h.num_minibatches, h.decay_learning_rates)
            c_lr = O.linear_schedule(h.critic_lr, c_state.sched_count, h.num_updates, h.epochs, h.num_minibatches, h.decay_learning_rates)
            a_new, _ = O.clip_adam_step(actor.flat(), a_g.astype(dt), a_state, a_lr, h.max_grad_norm)
            c_new, _ = O.clip_adam_step(critic.flat(), c_g.astype(dt), c_state, c_lr, h.max_grad_norm)
            actor = O.MLPParams.from_flat(a_new, sizes_a, actor.activation, actor.ln_bias is not None)
            critic = O.MLPParams.from_flat(c_new, sizes_c, critic.activation, critic.ln_bias is not None)
            info = {**a_info, **c_info}
            for k in names:
                metrics[k][ep, i] = info[k]
    return actor, critic, metrics, adv, targets
