"""NumPy float64 oracle of PQN (stoix/systems/q_learning/ff_pqn.py), test infrastructure only.

It reuses ppo_oracle's MLP (every torso option) and synth_env's Philox, and restates:
  - the epsilon-greedy draw of stx_epsilon_greedy from its Philox words (integer arithmetic: bit-exact) and the fp32 epsilon
    schedule (optax.linear_schedule / constant_schedule as ff_pqn.py:286-297 builds them);
  - batch_lambda_returns / batch_q_lambda as the literal reverse loop of stoix/utils/multistep.py:384-408 / :559-569;
  - rlax.l2_loss / rlax.huber_loss and their gradient with respect to q[a];
  - optax.clip_by_global_norm + optax.radam (scale_by_radam, no nesterov; from upstream knowledge of optax 0.2.7.dev0, the version
    the reference pins);
  - the update loop (ff_pqn.py:97-207) with injected actions and permutations.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional, Sequence

import numpy as np

from oracle import ppo_oracle as O
from oracle.synth_env import philox4x32

_TAG = 0x45475259  # fourth counter word of the epsilon-greedy draw


def epsilon_at(init_value: float, end_value: float, transition_steps: float, decay: bool, update_no) -> np.ndarray:
    """The schedule in fp32, each operation rounded (optax.polynomial_schedule with power 1; transition_steps <= 0: init_value)."""
    f = np.float32
    u = np.asarray(update_no)
    if not decay:
        return np.full(u.shape, f(end_value), np.float32)
    if not transition_steps > 0:
        return np.full(u.shape, f(init_value), np.float32)
    c = np.minimum(np.maximum(u.astype(np.float32), f(0)), f(transition_steps)).astype(np.float32)
    frac = (f(1) - (c / f(transition_steps)).astype(np.float32)).astype(np.float32)
    return ((f(init_value) - f(end_value)) * frac + f(end_value)).astype(np.float32)


def epsilon_greedy(q: np.ndarray, eps: float, seed: int, call: int, mode: bool = False) -> np.ndarray:
    """Actions of stx_epsilon_greedy for q (E, A) float32 rows: explore if (w0 >> 8) 2^-24 < eps, then (w1 A) >> 32; else the
    ((w1 n_ties) >> 32)-th maximal index; mode: the first maximal index."""
    q = np.asarray(q, np.float32)
    E, A = q.shape
    qmax = q.max(axis=1, keepdims=True)
    is_max = q == qmax
    first = is_max.argmax(axis=1)
    if mode:
        return first.astype(np.int32)
    e = np.arange(E, dtype=np.uint64)
    c2 = (np.uint64(call >> 32) ^ ((e >> np.uint64(32)) << np.uint64(16))) & np.uint64(0xFFFFFFFF)
    w0, w1, _, _ = philox4x32(e, np.uint64(call & 0xFFFFFFFF), c2, np.uint64(_TAG), seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    explore = (w0 >> np.uint64(8)).astype(np.float32) * np.float32(2.0 ** -24) < np.float32(eps)
    uniform = ((w1 * np.uint64(A)) >> np.uint64(32)).astype(np.int64)
    n_ties = is_max.sum(axis=1).astype(np.uint64)
    pick = ((w1 * n_ties) >> np.uint64(32)).astype(np.int64)
    greedy = np.array([np.flatnonzero(is_max[i])[pick[i]] for i in range(E)], dtype=np.int64)
    return np.where(explore, uniform, greedy).astype(np.int32)


def batch_lambda_returns(r_t, discount_t, v_t, lambda_=1.0) -> np.ndarray:
    """multistep.py:384-408, time-major: acc = v_t[-1]; for t = T-1 .. 0: acc = r + d ((1 - lambda) v + lambda acc)."""
    r_t, discount_t, v_t = (np.asarray(x, np.float64) for x in (r_t, discount_t, v_t))
    lam = np.ones_like(discount_t) * np.asarray(lambda_, np.float64)
    acc = v_t[-1].copy()
    out = np.zeros_like(r_t)
    for t in range(r_t.shape[0] - 1, -1, -1):
        acc = r_t[t] + discount_t[t] * ((1 - lam[t]) * v_t[t] + lam[t] * acc)
        out[t] = acc
    return out


def batch_q_lambda(r_t, discount_t, q_t, lambda_) -> np.ndarray:
    """multistep.py:559-569, time-major: v_t = max_a q_t."""
    return batch_lambda_returns(r_t, discount_t, np.asarray(q_t, np.float64).max(axis=-1), lambda_)


def q_loss_and_dq(q: np.ndarray, action: np.ndarray, targets: np.ndarray, delta: float):
    """mean(l2 / Huber loss of td = targets - q[a]) and its gradient with respect to q (ff_pqn.py:139-162)."""
    m = q.shape[0]
    td = targets - q[np.arange(m), action]
    if delta > 0:
        ax = np.abs(td)
        quad = np.minimum(ax, delta)
        loss = 0.5 * quad ** 2 + delta * (ax - quad)
        g = np.clip(td, -delta, delta)
    else:
        loss = 0.5 * td ** 2
        g = td
    dq = np.zeros_like(q)
    dq[np.arange(m), action] = -g / m
    return float(loss.mean()), dq


@dataclass
class RadamState:
    mu: np.ndarray
    nu: np.ndarray
    count: int = 0


def radam_rectifier(b2: float, t: int) -> Optional[float]:
    """r_t of optax.scale_by_radam at step t (count + 1), or None on the un-rectified branch (rho_t < 5)."""
    rho_inf = 2.0 / (1.0 - b2) - 1.0
    b2t = b2 ** t
    rho = rho_inf - 2.0 * t * b2t / (1.0 - b2t)
    if rho < 5.0:
        return None
    return float(np.sqrt((rho - 4.0) * (rho - 2.0) * rho_inf / ((rho_inf - 4.0) * (rho_inf - 2.0) * rho)))


def clip_radam_step(p: np.ndarray, g: np.ndarray, st: RadamState, lr: float, max_grad_norm: float, b1=0.9, b2=0.999, eps=1e-8,
                    eps_root=0.0, threshold=5.0) -> np.ndarray:
    """optax.chain(clip_by_global_norm(max_grad_norm), radam(lr)).update + apply_updates, in place on st; returns the new params."""
    g = np.asarray(g, np.float64)
    g_norm = float(np.sqrt((g * g).sum()))
    if not g_norm < max_grad_norm:
        g = g / g_norm * max_grad_norm
    st.mu = b1 * st.mu + (1 - b1) * g
    st.nu = b2 * st.nu + (1 - b2) * g * g
    t = st.count + 1
    mh, nh = st.mu / (1 - b1 ** t), st.nu / (1 - b2 ** t)
    rho_inf = 2.0 / (1.0 - b2) - 1.0
    rho = rho_inf - 2.0 * t * b2 ** t / (1.0 - b2 ** t)
    if rho >= threshold:
        r = np.sqrt((rho - 4.0) * (rho - 2.0) * rho_inf / ((rho_inf - 4.0) * (rho_inf - 2.0) * rho))
        u = r * mh / (np.sqrt(nh + eps_root) + eps)
    else:
        u = mh
    st.count = t
    return p - lr * u


@dataclass
class PqnHyper:
    epochs: int
    num_minibatches: int
    gamma: float
    q_lambda: float
    huber: float
    lr: float
    max_grad_norm: float
    num_updates: int = 1
    decay: bool = False
    b1: float = float(np.float32(0.9))
    b2: float = float(np.float32(0.999))
    eps: float = float(np.float32(1e-8))


def targets_literal(p: O.MLPParams, obs: np.ndarray, next_obs: np.ndarray, reward, done, truncated, gamma, q_lambda) -> np.ndarray:
    """ff_pqn.py:97-120 time-major: q_t = Q(concat(obs[0..T-1], next_obs[T-1]))[1:], d_t = gamma (1 - (done | truncated))."""
    T, E, D = obs.shape
    observations = np.concatenate([obs, next_obs[T - 1:T]], axis=0)
    q_all, _ = O.mlp_forward(p, observations.reshape(-1, D))
    q_t = q_all.reshape(T + 1, E, -1)[1:]
    d_t = gamma * (1.0 - (np.asarray(done, bool) | np.asarray(truncated, bool)).astype(np.float64))
    return batch_q_lambda(reward, d_t, q_t, q_lambda)


def pqn_update(p: O.MLPParams, st: RadamState, obs: np.ndarray, action: np.ndarray, targets: np.ndarray, perms: Sequence[np.ndarray],
               h: PqnHyper, sizes: List[int], grad_sync=None) -> O.MLPParams:
    """_update_epoch x epochs (ff_pqn.py:122-207) on the flat (T*E) batch with the given permutation per epoch.  grad_sync (optional):
    the pmean over "device" of each minibatch gradient (flat array in, mean over the ranks out)."""
    T, E, D = obs.shape
    B = T * E
    mb = B // h.num_minibatches
    x, a, tg = obs.reshape(B, D), np.asarray(action).reshape(B), targets.reshape(B)
    flat = p.flat()
    for ep in range(h.epochs):
        for i in range(h.num_minibatches):
            idx = np.asarray(perms[ep])[i * mb:(i + 1) * mb]
            net = O.MLPParams.from_flat(flat, sizes, p.activation, p.ln_bias is not None)
            q, acts = O.mlp_forward(net, x[idx])
            _, dq = q_loss_and_dq(q, a[idx], tg[idx], h.huber)
            grad = O.mlp_backward(net, acts, dq).flat()
            if grad_sync is not None:
                grad = grad_sync(grad)
            lr = h.lr
            if h.decay:  # schedule steps per update = epochs (ff_pqn.py:263)
                lr = h.lr * (1.0 - (st.count // h.epochs) / h.num_updates)
            flat = clip_radam_step(flat, grad, st, lr, h.max_grad_norm, h.b1, h.b2, h.eps)
    return O.MLPParams.from_flat(flat, sizes, p.activation, p.ln_bias is not None)
