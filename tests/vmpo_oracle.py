"""CPU oracle for V-MPO (stoix/systems/mpo/ff_vmpo.py, ff_vmpo_continuous.py)  --  TEST INFRASTRUCTURE, NOT PRODUCT.

fp64 NumPy restatement of the update step: the full-batch epochs, their critic targets (GAE, or batch_n_step_bootstrapped_returns
of stoix/utils/multistep.py:148-210), rlax.vmpo_loss with the reference's KL constraints, the l2 value loss, three
chain(clip_by_global_norm, adam) steps, the dual clamp at -18 and optax.periodic_update of the target actor.  The networks, GAE and
Adam come from oracle/ppo_oracle.py; the tanh-Normal log-prob of a given action from tests/ppo_continuous_oracle.py.

rlax is not vendored with the reference.  The rules below are restated from rlax's published mpo_ops.py (vmpo_loss and
vmpo_compute_weights_and_temperature_loss) and are marked (!) where they are upstream knowledge rather than reference code:
  (!) k = int(top_k_fraction N) with top_k_fraction = 0.5; tau = the k-th largest advantage; the selection is advantages >= tau
      compared as floats, so every tie at tau is selected and -0 == +0; K = the number selected.
  (!) temperature eta = the projected Lagrange multiplier softplus(log_temperature) + 1e-8 (rlax's projection clip at 1e-10 is a
      no-op in value and gradient for these values); m = max over the selection of A / eta, Z = sum exp(A / eta - m) over it.
  (!) weights w = exp(A / eta - m) / Z on the selection, 0 elsewhere, stop-gradient.
  (!) policy loss L_pi = -sum w log pi(a | s): a SUM over the rows, no 1/N.
  (!) temperature loss L_eta = eta (epsilon + log Z + m - log K).
  (!) per KL constraint (kl, alpha, epsilon_alpha): mean_kl = mean over rows (a vector over action dims when per-dimension);
      L_kl = sum sg(alpha) mean_kl, L_alpha = sum alpha (epsilon_alpha - sg(mean_kl)).
  (!) loss = L_pi + L_kl + L_alpha + L_eta; its extras are reported as loss_policy, loss_kl, loss_alpha, loss_temperature.
The gradients are hand-derived and checked against torch.autograd of these rules in tests/test_oracle_vmpo.py.

`mask`: the whole-update oracle can take the device's selection of every epoch, so that fp32-vs-fp64 rounding of an advantage at
tau does not decide a comparison (the tests assert it agrees with the oracle's own selection away from tau).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence

import numpy as np

from oracle import ppo_oracle as O
from tests import ppo_continuous_oracle as PC

MPO_FLOAT_EPSILON = 1e-8
MIN_LOG_DUAL = -18.0
METRICS = ("loss_policy", "loss_kl", "loss_alpha", "loss_temperature", "temperature", "alpha", "alpha_stddev", "advantages", "v_loss")


def softplus(x):
    x = np.asarray(x, np.float64)
    return np.maximum(x, 0.0) + np.log1p(np.exp(-np.abs(x)))


def sigmoid(x):
    return 1.0 / (1.0 + np.exp(-np.asarray(x, np.float64)))


def dual_value(x):
    """softplus(x) + 1e-8, the transform of every dual variable (ff_vmpo.py:130-131)."""
    return softplus(x) + MPO_FLOAT_EPSILON


def topk_select(adv: np.ndarray):
    """(tau, mask, K) of the rows of `adv` (float comparison: ties at tau all selected, -0 == +0)."""
    a = np.asarray(adv).reshape(-1)
    k = int(0.5 * a.size)
    tau = np.sort(a)[::-1][k - 1]
    mask = a >= tau
    return tau, mask, int(mask.sum())


def n_step_returns(r_t, discount_t, v_t, n: int, lambda_t: float = 1.0) -> np.ndarray:
    """batch_n_step_bootstrapped_returns (multistep.py:148-210) per element, batch-major [B, T]: the bootstrap value shifted by n and
    padded with v_t[:, -1], then G = r + d ((1 - l) v + l G) from step t + n - 1 down to t, padded steps with r = 0, d = 1, l = 1."""
    r_t, discount_t, v_t = (np.asarray(x, np.float64) for x in (r_t, discount_t, v_t))
    B, T = r_t.shape
    out = np.empty((B, T))
    for t in range(T):
        g = v_t[:, min(t + n - 1, T - 1)].copy()
        for i in reversed(range(n)):
            s = t + i
            if s < T:
                rr, dd, ll, vv = r_t[:, s], discount_t[:, s], lambda_t, v_t[:, s]
            else:
                rr, dd, ll, vv = 0.0, 1.0, 1.0, v_t[:, T - 1]
            g = rr + dd * ((1.0 - ll) * vv + ll * g)
        out[:, t] = g
    return out


def vmpo_loss(kind: str, head, head_t, action, adv, duals, epsilon: float, epsilon_alpha: float, epsilon_stddev: float = 0.0,
              per_dim: bool = True, minimum: float = -1.0, maximum: float = 1.0, min_scale: float = 1e-3,
              mask: Optional[np.ndarray] = None) -> Dict[str, np.ndarray]:
    """rlax.vmpo_loss of one shard (rules in the module docstring) with its analytic gradients: d_head (N, W), d_duals (n_dual),
    the loss terms, the metrics (METRICS order) and the selection."""
    head, head_t, adv, duals = (np.asarray(x, np.float64) for x in (head, head_t, adv, duals))
    N = adv.size
    if mask is None:
        _, mask, _ = topk_select(adv)
    mask = np.asarray(mask, bool).reshape(N)
    K = int(mask.sum())
    eta = dual_value(duals[0])
    x = adv / eta
    m = x[mask].max()
    e = np.where(mask, np.exp(np.where(mask, x - m, 0.0)), 0.0)
    Z = e.sum()
    w = e / Z
    if kind == "categorical":
        A = head.shape[1]
        lp, lq = O.log_softmax(head), O.log_softmax(head_t)
        p, q = np.exp(lp), np.exp(lq)
        act = np.asarray(action).reshape(N).astype(np.int64)
        logp = lp[np.arange(N), act]
        kl_cols = (q * (lq - lp)).sum(-1)[:, None]   # KL(target || online)
        onehot = np.eye(A)[act]
        alpha = dual_value(duals[1:2])
        d_head = -w[:, None] * (onehot - p) + alpha[0] / N * (p - q)
        eps_cols = np.array([epsilon_alpha])
        half = 1
    else:
        A = head.shape[1] // 2
        logp, dlogp = PC.log_prob_given(head, np.asarray(action, np.float64).reshape(N, A), minimum, maximum, min_scale)
        mu, raw = head[:, :A], head[:, A:]
        sig = softplus(raw) + min_scale
        mu_t, sig_t = head_t[:, :A], softplus(head_t[:, A:]) + min_scale
        km = (mu - mu_t) ** 2 / (2.0 * sig_t ** 2)                                   # KL(target || N(mu, sigma_t))
        ks = np.log(sig / sig_t) + sig_t ** 2 / (2.0 * sig ** 2) - 0.5              # KL(target || N(mu_t, sigma))
        d_km_dmu = (mu - mu_t) / sig_t ** 2
        d_ks_dsig = 1.0 / sig - sig_t ** 2 / sig ** 3
        if per_dim:
            kl_cols, half = np.concatenate([km, ks], axis=1), A
            am, a_s = dual_value(duals[1:1 + A]), dual_value(duals[1 + A:1 + 2 * A])
        else:
            kl_cols, half = np.stack([km.sum(1), ks.sum(1)], axis=1), 1
            am, a_s = np.full(A, dual_value(duals[1])), np.full(A, dual_value(duals[2]))
        d_loc = -w[:, None] * dlogp[:, :A] + am / N * d_km_dmu
        d_raw = -w[:, None] * dlogp[:, A:] + a_s / N * d_ks_dsig * sigmoid(raw)
        d_head = np.concatenate([d_loc, d_raw], axis=1)
        alpha = dual_value(duals[1:1 + kl_cols.shape[1]])
        eps_cols = np.array([epsilon_alpha] * half + [epsilon_stddev] * half)
    mean_kl = kl_cols.mean(0)
    lse = np.log(Z) + m
    loss_policy = -(w * logp).sum()
    loss_temperature = eta * (epsilon + lse - np.log(K))
    loss_kl = (alpha * mean_kl).sum()
    loss_alpha = (alpha * (eps_cols - mean_kl)).sum()
    g_eta = epsilon + lse - np.log(K) - (w * adv).sum() / eta
    d_duals = np.concatenate([[g_eta * sigmoid(duals[0])], (eps_cols - mean_kl) * sigmoid(duals[1:1 + kl_cols.shape[1]])])
    alpha_m = alpha[:half].mean()
    alpha_s = alpha[half:].mean() if kind != "categorical" else 0.0
    return {"d_head": d_head, "d_duals": d_duals, "mask": mask, "K": K, "weights": w, "mean_kl": mean_kl,
            "loss": loss_policy + loss_kl + loss_alpha + loss_temperature,
            "metrics": np.array([loss_policy, loss_kl, loss_alpha, loss_temperature, eta, alpha_m, alpha_s, adv.mean(), np.nan])}


def value_loss(value, targets):
    """rlax.l2_loss(targets - v).mean() and its gradient with respect to v."""
    td = np.asarray(targets, np.float64) - np.asarray(value, np.float64)
    return 0.5 * (td ** 2).mean(), -td / td.size


@dataclass
class VmpoHyper:
    kind: str
    gamma: float = 0.99
    gae_lambda: float = 0.95
    max_abs_reward: float = 20000.0
    epochs: int = 16
    actor_lr: float = 3e-4
    critic_lr: float = 3e-4
    dual_lr: float = 1e-2
    max_grad_norm: float = 1.0
    epsilon: float = 0.5
    epsilon_alpha: float = 0.001
    epsilon_stddev: float = 0.0
    per_dim: bool = True
    actor_target_period: int = 50
    n_step: int = 0              # > 0: use_n_step_bootstrap with this n
    minimum: float = -1.0
    maximum: float = 1.0
    min_scale: float = 1e-3


@dataclass
class VmpoState:
    actor: O.MLPParams
    target: O.MLPParams
    critic: O.MLPParams
    duals: np.ndarray
    s_actor: O.AdamState
    s_critic: O.AdamState
    s_duals: O.AdamState


def init_state(actor: O.MLPParams, target: O.MLPParams, critic: O.MLPParams, duals: np.ndarray, counts=(0, 0, 0)) -> VmpoState:
    z = lambda p: np.zeros_like(p)
    st = [O.AdamState(z(actor.flat()), z(actor.flat())), O.AdamState(z(critic.flat()), z(critic.flat())), O.AdamState(z(duals), z(duals))]
    for s, c in zip(st, counts):
        s.count = s.sched_count = int(c)
    return VmpoState(actor, target, critic, np.asarray(duals, np.float64), *st)


def targets(h: VmpoHyper, critic: O.MLPParams, obs, reward, done):
    """Current critic on all T rows, advantages and targets on the first T-1 (ff_vmpo.py:184-208), time-major (T-1, E)."""
    T, E, D = obs.shape
    v = O.mlp_forward(critic, obs.reshape(T * E, D))[0][:, 0].reshape(T, E)
    r = np.clip(np.asarray(reward, np.float64), -h.max_abs_reward, h.max_abs_reward)
    d = (1.0 - np.asarray(done, np.float64)) * h.gamma
    if h.n_step:
        tg = n_step_returns(r[:-1].T, d[:-1].T, v[1:].T, h.n_step).T
        return tg - v[:-1], tg, v
    adv, tg = O.gae(r[:-1], d[:-1], h.gae_lambda, v_tm1=v[:-1], v_t=v[1:], time_major=True)
    return adv, tg, v


def epoch(h: VmpoHyper, st: VmpoState, obs, action, reward, done, mask: Optional[np.ndarray] = None):
    """One _update_epoch (ff_vmpo.py:111-289) of one shard.  Returns (grads {actor, critic, duals}, metrics, oracle mask, adv) and
    steps `st` in place."""
    T, E, D = obs.shape
    N = (T - 1) * E
    adv, tg, v = targets(h, st.critic, obs, reward, done)
    x = obs[:-1].reshape(N, D)
    head_t = O.mlp_forward(st.target, x)[0]
    head, acts = O.mlp_forward(st.actor, x)
    act = action[:-1].reshape(N, -1) if h.kind == "tanh_normal" else action[:-1].reshape(N)
    own_mask = topk_select(adv.reshape(N))[1]
    out = vmpo_loss(h.kind, head, head_t, act, adv.reshape(N), st.duals, h.epsilon, h.epsilon_alpha, h.epsilon_stddev, h.per_dim, h.minimum,
                    h.maximum, h.min_scale, mask=own_mask if mask is None else mask)
    g_a = O.mlp_backward(st.actor, acts, out["d_head"]).flat()
    vl, dv = value_loss(v[:-1].reshape(N), tg.reshape(N))
    c_v, c_acts = O.mlp_forward(st.critic, x)
    g_c = O.mlp_backward(st.critic, c_acts, dv[:, None]).flat()
    metrics = out["metrics"].copy()
    metrics[8] = vl
    sizes = lambda p: [p.W[0].shape[0]] + [w.shape[1] for w in p.W]
    a_new, _ = O.clip_adam_step(st.actor.flat(), g_a, st.s_actor, h.actor_lr, h.max_grad_norm)
    c_new, _ = O.clip_adam_step(st.critic.flat(), g_c, st.s_critic, h.critic_lr, h.max_grad_norm)
    d_new, _ = O.clip_adam_step(st.duals, out["d_duals"], st.s_duals, h.dual_lr, h.max_grad_norm)
    st.actor = O.MLPParams.from_flat(a_new, sizes(st.actor), st.actor.activation)
    st.critic = O.MLPParams.from_flat(c_new, sizes(st.critic), st.critic.activation)
    st.duals = np.maximum(MIN_LOG_DUAL, d_new)
    if st.s_actor.count % h.actor_target_period == 0:   # optax.periodic_update after learner_step_count += 1
        st.target = st.actor.copy()
    return {"actor": g_a, "critic": g_c, "duals": out["d_duals"]}, metrics, own_mask, adv


def update(h: VmpoHyper, st: VmpoState, obs, action, reward, done, masks: Optional[Sequence[np.ndarray]] = None):
    """The update epochs of ff_vmpo.py:291-296 on a recorded rollout (one shard).  Returns (metrics (epochs, 9), own masks)."""
    ms: List[np.ndarray] = []
    own: List[np.ndarray] = []
    advs: List[np.ndarray] = []
    for ep in range(h.epochs):
        _, m, om, adv = epoch(h, st, obs, action, reward, done, None if masks is None else masks[ep])
        ms.append(m), own.append(om), advs.append(adv)
    return np.stack(ms), own, advs
