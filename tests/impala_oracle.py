"""fp64 NumPy restatement of IMPALA's learner step (stoix/systems/impala/sebulba/ff_impala.py:358-566).

  - ⚠ rlax.vtrace_td_error_and_advantage and rlax.vtrace: rlax is not vendored in the reference; the rules below are restated from its
    published definitions (as SURVEY.md Appendix A restates the other rlax functions):
      c = lambda min(1, rho);  delta = min(clip_rho, rho) (r + d v_t - v_tm1);  acc_t = delta_t + d_t c_t acc_{t+1}, acc_T = 0
      vs = acc + v_tm1;  errors = stop_gradient(vs) - v_tm1
      q_t = r_t + d_t (lambda vs_{t+1} + (1 - lambda) v_tm1_{t+1}) for t < T - 1, r + d v_t at T - 1
      pg_adv = min(clip_pg_rho, rho) (q - v_tm1)
  - ⚠ optax.rmsprop at the pinned commit's defaults (decay 0.9, eps 1e-8, initial_scale 0, eps_in_sqrt, no centring / momentum / bias
    correction), from upstream knowledge: nu = (1 - decay) g^2 + decay nu;  u = g / sqrt(nu + eps).
  - the losses are sums: critic vf_coef 0.5 sum errors^2, actor -sum pg_adv logp(a) - ent_coef sum H.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import numpy as np

from oracle import ppo_oracle as O


def vtrace(v_tm1, v_t, r_t, discount_t, rho_tm1, lambda_=1.0, clip_rho=1.0, clip_pg_rho=1.0):
    """vtrace_td_error_and_advantage on time-major (T, ...) arrays.  Returns (errors, pg_advantage, q_estimate)."""
    v_tm1, v_t, r_t, d, rho = (np.asarray(x, np.float64) for x in (v_tm1, v_t, r_t, discount_t, rho_tm1))
    T = r_t.shape[0]
    c = lambda_ * np.minimum(1.0, rho)
    delta = np.minimum(clip_rho, rho) * (r_t + d * v_t - v_tm1)
    acc = np.zeros_like(r_t)
    run = np.zeros_like(r_t[0])
    for t in range(T - 1, -1, -1):
        run = delta[t] + d[t] * c[t] * run
        acc[t] = run
    vs = acc + v_tm1
    errors = vs - v_tm1
    boot = np.concatenate([lambda_ * vs[1:] + (1.0 - lambda_) * v_tm1[1:], v_t[-1:]], axis=0)
    q = r_t + d * boot
    return errors, np.minimum(clip_pg_rho, rho) * (q - v_tm1), q


def normalize_rewards(r, scale=1.0, eps=1e-8):
    """r_t = reward_scale (r_t - mean) / (std + reward_eps) over the whole (T, E) batch, population std (ff_impala.py:389-392)."""
    r = np.asarray(r, np.float64)
    return scale * (r - r.mean()) / (r.std() + eps)


@dataclass
class VtraceHyper:
    gamma: float = 0.99
    lambda_: float = 1.0
    clip_rho: float = 1.0
    clip_pg_rho: float = 1.0
    ent_coef: float = 0.01
    vf_coef: float = 0.5


def loss_and_head_grads(logits, values, action, log_prob_b, r_t, done, h: VtraceHyper):
    """One minibatch: logits (T, Em, A), values (T + 1, Em), action / log_prob_b / r_t (already normalised) / done (T, Em).
    Returns (d_logits (T, Em, A), d_value (T + 1, Em), metrics dict) of the summed losses as the reference writes them."""
    logits, values = np.asarray(logits, np.float64), np.asarray(values, np.float64)
    lp = O.log_softmax(logits)
    p = np.exp(lp)
    a = np.asarray(action).astype(np.int64)
    logp_a = np.take_along_axis(lp, a[..., None], axis=-1)[..., 0]
    H = -(p * lp).sum(-1)
    rho = np.exp(logp_a - np.asarray(log_prob_b, np.float64))
    d = h.gamma * (1.0 - np.asarray(done, np.float64))
    err, pg, q = vtrace(values[:-1], values[1:], r_t, d, rho, h.lambda_, h.clip_rho, h.clip_pg_rho)
    onehot = np.eye(logits.shape[-1])[a]
    d_logits = -pg[..., None] * (onehot - p) + h.ent_coef * p * (lp + H[..., None])
    d_value = np.zeros_like(values)
    d_value[:-1] = -h.vf_coef * err
    metrics = {"actor_loss": float(-(pg * logp_a).sum()), "entropy": float(H.sum()), "value_loss": float(0.5 * (err ** 2).sum()),
               "q_estimate": float(q.mean()), "pg_advantage": float(pg.mean())}
    return d_logits, d_value, metrics


@dataclass
class RmspropState:
    nu: np.ndarray
    count: int = 0        # the fused kernel's per-segment counter (scale_by_rms itself keeps none)
    sched_count: int = 0  # ScaleByScheduleState.count


def clip_rmsprop_step(p, g, st: RmspropState, lr, max_grad_norm, decay=0.9, eps=1e-8):
    """optax.chain(clip_by_global_norm(max_grad_norm), rmsprop(lr)).update + apply_updates on one network's flat vector, in place on st."""
    g = np.asarray(g, np.float64)
    g_norm = np.sqrt((g ** 2).sum())
    if g_norm >= max_grad_norm:
        g = g / g_norm * max_grad_norm
    st.nu = (1.0 - decay) * g * g + decay * st.nu
    st.count += 1
    st.sched_count += 1
    return p - lr * g / np.sqrt(st.nu + eps)


@dataclass
class ImpalaHyper(VtraceHyper):
    num_minibatches: int = 4
    actor_lr: float = 6e-4
    critic_lr: float = 6e-4
    max_grad_norm: float = 40.0
    num_updates: int = 1
    decay_learning_rates: bool = True
    normalize_rewards: bool = False
    reward_scale: float = 1.0
    reward_eps: float = 1e-8


def update(actor: O.MLPParams, critic: O.MLPParams, a_st: RmspropState, c_st: RmspropState, obs, action, log_prob, reward, done,
           h: ImpalaHyper) -> Tuple[O.MLPParams, O.MLPParams, List[Dict[str, float]], Tuple[float, float]]:
    """One learner step on a (T + 1, E) batch: reward statistics, then the env-column blocks in order, each one clip + RMSProp step
    per network on the parameters the previous block left.  Returns (actor, critic, per-minibatch metrics, (reward mean, std))."""
    T1, E = action.shape
    T, nmb = T1 - 1, h.num_minibatches
    Em = E // nmb
    r = np.asarray(reward[:T], np.float64)
    stats = (float(r.mean()), float(r.std()))
    if h.normalize_rewards:
        r = normalize_rewards(r, h.reward_scale, h.reward_eps)
    metrics = []
    for i in range(nmb):
        cols = slice(i * Em, (i + 1) * Em)
        x = np.asarray(obs[:, cols], np.float64)
        D = x.shape[-1]
        logits, acts_a = O.mlp_forward(actor, x[:T].reshape(T * Em, D))
        v, acts_c = O.mlp_forward(critic, x.reshape((T + 1) * Em, D))
        d_logits, d_value, m = loss_and_head_grads(logits.reshape(T, Em, -1), v.reshape(T + 1, Em), action[:T, cols], log_prob[:T, cols],
                                                   r[:, cols], done[:T, cols], h)
        ga = O.mlp_backward(actor, acts_a, d_logits.reshape(T * Em, -1)).flat()
        gc = O.mlp_backward(critic, acts_c, d_value.reshape(-1, 1)).flat()
        lr_a = O.linear_schedule(h.actor_lr, a_st.sched_count, h.num_updates, 1, nmb, h.decay_learning_rates)
        lr_c = O.linear_schedule(h.critic_lr, c_st.sched_count, h.num_updates, 1, nmb, h.decay_learning_rates)
        sizes_a, sizes_c = [actor.W[0].shape[0]] + [w.shape[1] for w in actor.W], [critic.W[0].shape[0]] + [w.shape[1] for w in critic.W]
        actor = O.MLPParams.from_flat(clip_rmsprop_step(actor.flat(), ga, a_st, lr_a, h.max_grad_norm), sizes_a, actor.activation)
        critic = O.MLPParams.from_flat(clip_rmsprop_step(critic.flat(), gc, c_st, lr_c, h.max_grad_norm), sizes_c, critic.activation)
        metrics.append(m)
    return actor, critic, metrics, stats
