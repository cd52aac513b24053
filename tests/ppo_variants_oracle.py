"""CPU oracle for the PPO variants: KL-penalty PPO (stoix/systems/ppo/anakin/ff_ppo_penalty.py, ff_ppo_penalty_continuous.py)
and DPO (ff_dpo_continuous.py)  --  TEST INFRASTRUCTURE, NOT PRODUCT.

fp64 NumPy restatement of the variants' `_actor_loss_fn` with hand-derived d(loss)/d(head output):
  ppo_penalty_loss (stoix/utils/loss.py:35-47): -mean(ratio A) + beta mean KL(behaviour || current), no ratio clipping;
  dpo_loss (loss.py:50-65): -mean(ratio A - drift).
The Categorical pieces reuse oracle/ppo_oracle.py, the tanh-Normal log-prob and entropy estimate tests/ppo_continuous_oracle.py.

The tanh-Normal KL is restated FROM UPSTREAM KNOWLEDGE (TFP is not vendored): tfp registers the KL of two
TransformedDistributions with the same bijector as the KL of their base distributions, and the KL of two Independent
distributions as the sum over the reinterpreted dimension, so KL = sum_j KL(Normal(mb_j, sb_j) || Normal(m_j, s_j)).

`variant_update` is the update step with the behaviour policy RECOMPUTED from the behaviour parameters (the actor at the start of
the update, ff_ppo_penalty.py:137,158), as the reference does.  The gradients are checked against torch.autograd in
tests/test_oracle_ppo_variants.py."""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import numpy as np

from oracle import ppo_oracle as O
from oracle import sac_oracle as S
from tests import ppo_continuous_oracle as PC

KL_PENALTY, DPO = "kl_penalty", "dpo"


# ------------------------------------------------------------------------------------------------ Categorical KL penalty


def categorical_kl(logits_p: np.ndarray, logits_q: np.ndarray) -> np.ndarray:
    """KL(Categorical(p) || Categorical(q)) per row = sum_j p_j (log p_j - log q_j)."""
    lp, lq = O.log_softmax(logits_p), O.log_softmax(logits_q)
    return (np.exp(lp) * (lp - lq)).sum(-1)


def penalty_actor_loss_and_dlogits(logits, b_logits, action, logp_old, adv, beta, ent_coef):
    """ff_ppo_penalty.py:150-178: ppo_penalty_loss - ent_coef * mean(entropy), and d/dlogits (the behaviour logits constant):
    -(1/m) A ratio (1[j=a] - p_j) + (beta/m)(p_j - pb_j) + (ent_coef/m) p_j (log p_j + H)."""
    m = logits.shape[0]
    lp = O.log_softmax(logits)
    p = np.exp(lp)
    pb = np.exp(O.log_softmax(b_logits))
    onehot = np.zeros_like(lp)
    onehot[np.arange(m), np.asarray(action, np.int64)] = 1.0
    ratio = np.exp((lp * onehot).sum(-1) - logp_old)
    kl = categorical_kl(b_logits, logits)
    loss_actor = -(ratio * adv).mean() + beta * kl.mean()
    H = -(p * lp).sum(-1)
    dlogits = (-(adv * ratio) / m)[:, None] * (onehot - p) + (beta / m) * (p - pb) + (ent_coef / m) * p * (lp + H[:, None])
    info = {"actor_loss": loss_actor, "entropy": H.mean(), "kl_divergence": kl.mean()}
    return loss_actor - ent_coef * H.mean(), dlogits, info


# ------------------------------------------------------------------------------------------------ tanh-Normal pieces


def tanh_normal_kl(head_p: np.ndarray, head_q: np.ndarray, min_scale: float = 1e-3):
    """KL(p || q) per row of two tanh-Normal heads (upstream knowledge, see the module doc) and d KL / d head_q (rows, 2A):
    dKL/dm = (m - mp) / s^2, dKL/ds = 1/s - (sp^2 + (mp - m)^2) / s^3, times sigmoid(raw) for the scale column."""
    A = head_p.shape[-1] // 2
    mp, sp = head_p[..., :A], S.softplus(head_p[..., A:]) + min_scale
    mq, raw = head_q[..., :A], head_q[..., A:]
    sq = S.softplus(raw) + min_scale
    d = mp - mq
    kl = (np.log(sq / sp) + (sp ** 2 + d ** 2) / (2.0 * sq ** 2) - 0.5).sum(-1)
    grad = np.concatenate([-d / sq ** 2, (1.0 / sq - (sp ** 2 + d ** 2) / sq ** 3) * S.sigmoid(raw)], axis=-1)
    return kl, grad


def dpo_rows(ld: np.ndarray, adv: np.ndarray, alpha: float, beta: float):
    """Per-row -(ratio A - drift) of dpo_loss (loss.py:50-65) and its derivative with respect to ld = logp - logp_old;
    relu'(0) = 0 (jax.nn.relu)."""
    ratio = np.exp(ld)
    x1, x2 = (ratio - 1.0) * adv, ld * adv
    t1, t2 = np.tanh(x1 / alpha), np.tanh(x2 / beta)
    y1, y2 = x1 - alpha * t1, x2 - beta * t2
    pos = adv >= 0.0
    drift = np.where(pos, np.maximum(y1, 0.0), np.maximum(y2, 0.0))
    d = -ratio * adv + np.where(pos & (y1 > 0), t1 * t1 * adv * ratio, 0.0) + np.where(~pos & (y2 > 0), t2 * t2 * adv, 0.0)
    return -(ratio * adv - drift), d


def tanh_variant_actor_loss_and_dhead(kind, head, action, logp_old, adv, ent_coef, eps, minimum, maximum, b_head=None, kl_coef=0.0,
                                      alpha=2.0, beta=0.6, min_scale=1e-3):
    """_actor_loss_fn of ff_ppo_penalty_continuous.py:150-179 (kind KL_PENALTY, behaviour head b_head) or ff_dpo_continuous.py:148-170
    (kind DPO), with the seeded entropy estimate's noise injected as eps; returns (total, d total / d head, info)."""
    m = head.shape[0]
    lp, dlp = PC.log_prob_given(head, action, minimum, maximum, min_scale)
    H, dH = PC.entropy_estimate(head, eps, minimum, maximum, min_scale)
    ld = lp - logp_old
    ratio = np.exp(ld)
    info = {"entropy": H.mean()}
    if kind == KL_PENALTY:
        kl, dkl = tanh_normal_kl(b_head, head, min_scale)
        loss_actor = -(ratio * adv).mean() + kl_coef * kl.mean()
        dhead = (-(adv * ratio) / m)[:, None] * dlp + (kl_coef / m) * dkl
        info["kl_divergence"] = kl.mean()
    else:
        rows, dld = dpo_rows(ld, adv, alpha, beta)
        loss_actor = rows.mean()
        dhead = (dld / m)[:, None] * dlp
    dhead = dhead - (ent_coef / m) * dH
    info["actor_loss"] = loss_actor
    return loss_actor - ent_coef * H.mean(), dhead, info


# ------------------------------------------------------------------------------------------------ the update step


def variant_update(kind: str, actor: O.MLPParams, critic: O.MLPParams, a_state: O.AdamState, c_state: O.AdamState, traj: O.Trajectory,
                   perms: np.ndarray, h: O.PPOHyper, kl_coef: float = 0.0, alpha: float = 2.0, beta: float = 0.6,
                   eps: Optional[np.ndarray] = None, minimum: Optional[float] = None, maximum: Optional[float] = None,
                   min_scale: float = 1e-3) -> Tuple[O.MLPParams, O.MLPParams, Dict[str, np.ndarray], np.ndarray, np.ndarray]:
    """GAE + epochs x minibatches of the variant's _update_minibatch.  Categorical actor when eps is None (integer actions (T, E)),
    tanh-Normal otherwise (float actions (T, E, A), entropy noise (epochs, num_minibatches, mb, A)).  The behaviour policy of the
    KL penalty is recomputed per minibatch from the actor parameters at the start of the update."""
    dt = traj.reward.dtype
    T, E, D = traj.obs.shape
    r_t, d_t, trunc = O.ppo_gae_inputs(traj.reward, traj.done, traj.truncated, h.gamma, h.reward_scale, dt.type)
    adv, targets = O.gae(r_t, d_t, h.gae_lambda, v_tm1=traj.value, v_t=traj.bootstrap_value, truncation_t=trunc, time_major=True,
                         standardize_advantages=h.standardize_advantages, dtype=dt.type)
    B = T * E
    mb = B // h.num_minibatches
    obs = traj.obs.reshape(B, D)
    act = traj.action.reshape(B, -1) if eps is not None else traj.action.reshape(B)
    lp_old, v_old, adv_f, tgt_f = (x.reshape(B) for x in (traj.log_prob, traj.value, adv, targets))
    sizes_a = [actor.W[0].shape[0]] + [w.shape[1] for w in actor.W]
    sizes_c = [critic.W[0].shape[0]] + [w.shape[1] for w in critic.W]
    behaviour_actor = actor  # behaviour_actor_params = params.actor_params (ff_ppo_penalty.py:137)
    names = ("actor_loss", "entropy", "value_loss") + (("kl_divergence",) if kind == KL_PENALTY else ())
    metrics = {k: np.zeros((h.epochs, h.num_minibatches), dt) for k in names}
    for ep in range(h.epochs):
        for i in range(h.num_minibatches):
            idx = perms[ep][i * mb:(i + 1) * mb]
            head, a_acts = O.mlp_forward(actor, obs[idx])
            b_head = O.mlp_forward(behaviour_actor, obs[idx])[0] if kind == KL_PENALTY else None
            if eps is None:
                assert kind == KL_PENALTY, "the reference has no discrete DPO"
                _, dhead, a_info = penalty_actor_loss_and_dlogits(head, b_head, act[idx], lp_old[idx], adv_f[idx], kl_coef, h.ent_coef)
            else:
                _, dhead, a_info = tanh_variant_actor_loss_and_dhead(kind, head, act[idx], lp_old[idx], adv_f[idx], h.ent_coef, eps[ep, i],
                                                                     minimum, maximum, b_head, kl_coef, alpha, beta, min_scale)
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
