"""NumPy float64 oracle of the distributional Q-learning systems (stoix/systems/q_learning/ff_c51.py, ff_qr_dqn.py), test
infrastructure only.

It reuses ppo_oracle's MLP and clip + Adam, dqn_oracle's ring, sample and loss hyper-parameters, and pqn_oracle's epsilon-greedy
draw (through the tests), and restates:
  - the expected Q of the two heads (stoix/networks/heads.py:251-253, 288-289);
  - rlax.categorical_l2_project.  rlax is not part of the reference tree; this is its published definition written out: clip the
    source support to [z_q[0], z_q[-1]], inverse spacings d_pos / d_neg to the next / previous target atom (0 where the wrapped
    spacing at either end, or a repeated atom, is not positive), delta_hat = d_sign delta d_pos - (1 - d_sign) delta d_neg with
    d_sign = (delta >= 0), and sum_j clip(1 - delta_hat, 0, 1) p_j;
  - categorical_double_q_learning (stoix/utils/loss.py:81-103) and its gradient with respect to the taken action's logits:
    (softmax sum_j t_j - t) / M;
  - quantile_q_learning + quantile_regression_loss (:226-314) and their gradient with the tie conventions of the kernels:
    delta_neg = (delta < 0), so delta = 0 weighs tau_i; the Huber slope clip(delta, -kappa, kappa); and in the kappa = 0 branch
    the slope of |x| at 0 is +1, which is what JAX's lax.abs JVP, select(x >= 0, g, -g), gives (taken from JAX's published
    differentiation rule; JAX is not used here).  torch.abs has slope 0 there.
"""
from __future__ import annotations

from typing import Callable, List, Optional, Sequence, Tuple

import numpy as np

from oracle import ppo_oracle as O
from tests.dqn_oracle import LossHyper

LOSSES = ("categorical_double_q_learning", "quantile_q_learning")


def _softmax(z: np.ndarray) -> np.ndarray:
    e = np.exp(z - z.max(axis=-1, keepdims=True))
    return e / e.sum(axis=-1, keepdims=True)


def _log_softmax(z: np.ndarray) -> np.ndarray:
    s = z - z.max(axis=-1, keepdims=True)
    return s - np.log(np.exp(s).sum(axis=-1, keepdims=True))


def categorical_q_values(logits: np.ndarray, atoms: np.ndarray, A: int) -> np.ndarray:
    """sum_i softmax(logits[a])_i atoms_i of head rows (M, A N)."""
    z = np.asarray(logits, np.float64).reshape(len(logits), A, -1)
    return (_softmax(z) * np.asarray(atoms, np.float64)).sum(-1)


def quantile_q_values(q: np.ndarray, A: int) -> np.ndarray:
    """mean_i q[a, i] of head rows (M, A N)."""
    return np.asarray(q, np.float64).reshape(len(q), A, -1).mean(-1)


def l2_project(z_p: np.ndarray, probs: np.ndarray, z_q: np.ndarray) -> np.ndarray:
    """rlax.categorical_l2_project for one row: source support z_p (Np), probabilities probs (Np), target support z_q (Nq)."""
    z_p, probs, z_q = (np.asarray(x, np.float64) for x in (z_p, probs, z_q))
    vmin, vmax = z_q[0], z_q[-1]
    d_pos = np.concatenate([z_q, [vmin]])[1:]
    d_neg = np.concatenate([[vmax], z_q])[:-1]
    z_p = np.clip(z_p, vmin, vmax)[:, None]
    d_pos = (d_pos - z_q)[None, :]
    d_neg = (z_q - d_neg)[None, :]
    with np.errstate(divide="ignore"):
        d_neg = np.where(d_neg > 0, 1.0 / np.where(d_neg > 0, d_neg, 1.0), 0.0)
        d_pos = np.where(d_pos > 0, 1.0 / np.where(d_pos > 0, d_pos, 1.0), 0.0)
    delta_qp = z_p - z_q[None, :]
    d_sign = (delta_qp >= 0.0).astype(np.float64)
    delta_hat = (d_sign * delta_qp * d_pos) - ((1.0 - d_sign) * delta_qp * d_neg)
    return np.sum(np.clip(1.0 - delta_hat, 0.0, 1.0) * probs[:, None], 0)


def _r_d(reward, done, discount, h: LossHyper) -> Tuple[np.ndarray, np.ndarray]:
    r = np.clip(np.asarray(reward, np.float64), -h.max_abs_reward, h.max_abs_reward)
    d = (1.0 - np.asarray(done, np.float64)) * h.gamma if discount is None else np.asarray(discount, np.float64)
    return r, d


def _support(x, M: int, N: int) -> np.ndarray:
    x = np.asarray(x, np.float64)
    return np.broadcast_to(x, (M, N)) if x.ndim == 1 else x


def categorical_loss_and_grad(logits_tm1, logits_t, q_sel, atoms_tm1, atoms_t, a, reward, done, h: LossHyper, discount=None,
                              ) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """Per-row loss (M), d mean(loss) / d logits_tm1 (M, A N) and the projected targets (M, N).  Atoms (N) or (M, N)."""
    q_sel = np.asarray(q_sel, np.float64)
    M, A = q_sel.shape
    lt1 = np.asarray(logits_tm1, np.float64).reshape(M, A, -1)
    N = lt1.shape[-1]
    lt = np.asarray(logits_t, np.float64).reshape(M, A, N)
    z_tm1, z_t = _support(atoms_tm1, M, N), _support(atoms_t, M, N)
    a = np.asarray(a, np.int64)
    r, d = _r_d(reward, done, discount, h)
    rows = np.arange(M)
    p = _softmax(lt[rows, q_sel.argmax(-1)])
    target_z = r[:, None] + d[:, None] * z_t
    t = np.stack([l2_project(target_z[m], p[m], z_tm1[m]) for m in range(M)])
    la = lt1[rows, a]
    loss = -(t * _log_softmax(la)).sum(-1)
    g = np.zeros((M, A, N))
    g[rows, a] = (_softmax(la) * t.sum(-1, keepdims=True) - t) / M
    return loss, g.reshape(M, A * N), t


def quantile_loss_and_grad(q_tm1, q_t, q_sel, tau, a, reward, done, h: LossHyper, A: int, discount=None) -> Tuple[np.ndarray, np.ndarray]:
    """Per-row loss (M) and d mean(loss) / d q_tm1 (M, A N); head rows (M, A N), tau (N) or (M, N), q_sel None -> q_t."""
    q1 = np.asarray(q_tm1, np.float64)
    M = q1.shape[0]
    q1 = q1.reshape(M, A, -1)
    N = q1.shape[-1]
    qt = np.asarray(q_t, np.float64).reshape(M, A, N)
    sel = qt if q_sel is None else np.asarray(q_sel, np.float64).reshape(M, A, N)
    tau = _support(tau, M, N)
    a = np.asarray(a, np.int64)
    r, d = _r_d(reward, done, discount, h)
    rows = np.arange(M)
    target = r[:, None] + d[:, None] * qt[rows, sel.mean(-1).argmax(-1)]
    src = q1[rows, a]
    delta = target[:, None, :] - src[:, :, None]          # (M, i, j)
    w = np.abs(tau[:, :, None] - (delta < 0.0))
    if h.huber > 0:
        ax = np.abs(delta)
        quad = np.minimum(ax, h.huber)
        rho, slope = 0.5 * quad ** 2 + h.huber * (ax - quad), np.clip(delta, -h.huber, h.huber)
    else:
        rho, slope = np.abs(delta), np.where(delta >= 0.0, 1.0, -1.0)
    loss = (w * rho).mean(-1).sum(-1)
    g = np.zeros((M, A, N))
    g[rows, a] = -(w * slope).mean(-1) / M
    return loss, g.reshape(M, A * N)


def batch_grad(loss: str, online: O.MLPParams, target: O.MLPParams, obs, next_obs, a, reward, done, h: LossHyper, support, A: int
               ) -> Tuple[float, np.ndarray]:
    """jax.grad(_q_loss_fn) of one shard's batch (ff_c51.py:159-188, ff_qr_dqn.py:159-202): (mean loss, flat online gradient).
    support: the atoms (C51) or the quantile midpoints tau (QR-DQN), (N)."""
    out_tm1, acts = O.mlp_forward(online, np.asarray(obs, np.float64))
    out_t, _ = O.mlp_forward(target, np.asarray(next_obs, np.float64))
    if loss == "categorical_double_q_learning":
        sel = categorical_q_values(O.mlp_forward(online, np.asarray(next_obs, np.float64))[0], support, A)
        rows, g, _ = categorical_loss_and_grad(out_tm1, out_t, sel, support, support, a, reward, done, h)
    else:
        rows, g = quantile_loss_and_grad(out_tm1, out_t, None, support, a, reward, done, h, A)
    return float(rows.mean()), O.mlp_backward(online, acts, g).flat()


def distq_update(loss: str, online: np.ndarray, target: np.ndarray, st: O.AdamState, epochs: Sequence[Sequence[tuple]], h: LossHyper, support,
                 A: int, lr: float, max_grad_norm: float, tau: float, sizes: List[int], activation: str = "silu", ln: bool = False,
                 grad_sync: Optional[Callable] = None, eps: float = 1e-5) -> Tuple[np.ndarray, np.ndarray]:
    """_update_epoch x len(epochs) as dqn_oracle.dqn_update, with the distributional gradient: per epoch the mean of the shards'
    gradients, grad_sync (the pmean over devices), clip + Adam, then Polyak."""
    b1, b2 = float(np.float32(0.9)), float(np.float32(0.999))
    for batches in epochs:
        on = O.MLPParams.from_flat(online, sizes, activation, ln)
        tg = O.MLPParams.from_flat(target, sizes, activation, ln)
        g = np.mean([batch_grad(loss, on, tg, *b, h, support, A)[1] for b in batches], axis=0)
        if grad_sync is not None:
            g = grad_sync(g)
        online, _ = O.clip_adam_step(online, g, st, lr, max_grad_norm, b1, b2, float(np.float32(eps)))
        target = tau * online + (1.0 - tau) * target
    return online, target
