"""NumPy float64 oracle of the DQN family (stoix/systems/q_learning/ff_dqn.py, ff_ddqn.py, ff_mdqn.py, ff_dqn_reg.py), test
infrastructure only.

It reuses ppo_oracle's MLP and clip + Adam, pqn_oracle's epsilon-greedy draw and synth_env's Philox, and restates:
  - the four losses (stoix/utils/loss.py:106-146, 190-223; ff_dqn_reg.py:165-176) with reward clipping and d_t = (1 - done) gamma
    (ff_dqn.py:156-162), and their gradient with respect to q_tm1;
  - the discrete ring's add (time-major, oldest overwritten, newest `capacity` kept) and its uniform sample from the Philox words
    of stx_uniform_indices;
  - the update loop (ff_dqn.py:144-220) on injected sampled batches: clip + Adam, then Polyak after every optimiser step.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Callable, List, Optional, Sequence, Tuple

import numpy as np

from oracle import ppo_oracle as O
from oracle.synth_env import philox4x32

_TAG = 0x52504C59   # fourth counter word of the replay-index draw


def uniform_indices(M: int, n: int, seed: int, call: int) -> np.ndarray:
    """Index r = floor(w[r & 3] n / 2^32), w = Philox4x32-10 (seed; r / 4, call, call >> 32, tag)."""
    g = np.arange((M + 3) // 4, dtype=np.uint64)
    w = philox4x32(g, np.uint64(call & 0xFFFFFFFF), np.uint64(call >> 32), np.uint64(_TAG), seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    words = np.stack(w, axis=1).reshape(-1)[:M]
    return ((words * np.uint64(n)) >> np.uint64(32)).astype(np.int64)


class Ring:
    """The item buffer: add appends rows in time-major order and overwrites the oldest; sample is uniform with replacement."""

    def __init__(self, capacity: int, obs_dim: int):
        self.capacity = capacity
        self.obs = np.zeros((capacity, obs_dim), np.float32)
        self.next_obs = np.zeros((capacity, obs_dim), np.float32)
        self.action = np.zeros(capacity, np.int32)
        self.reward = np.zeros(capacity, np.float32)
        self.done = np.zeros(capacity, np.uint8)
        self.pos, self.size = 0, 0

    def add(self, obs, action, reward, done, next_obs) -> None:
        n = int(np.asarray(reward).size)
        D = self.obs.shape[1]
        cols = (np.asarray(obs).reshape(n, D), np.asarray(action).reshape(n), np.asarray(reward).reshape(n), np.asarray(done).reshape(n),
                np.asarray(next_obs).reshape(n, D))
        for r in range(max(0, n - self.capacity), n):
            s = (self.pos + r) % self.capacity
            self.obs[s], self.action[s], self.reward[s], self.done[s], self.next_obs[s] = (c[r] for c in cols)
        self.pos = (self.pos + n) % self.capacity
        self.size = min(self.size + n, self.capacity)

    def sample(self, M: int, seed: int, call: int, idx: Optional[np.ndarray] = None):
        j = uniform_indices(M, self.size, seed, call) if idx is None else np.asarray(idx, np.int64)
        return self.obs[j], self.next_obs[j], self.action[j], self.reward[j], self.done[j], j


@dataclass
class LossHyper:
    gamma: float = 0.99
    max_abs_reward: float = np.inf
    huber: float = 0.0
    tau: float = 0.03
    alpha: float = 0.9
    clip_value_min: float = -1e3
    reg: float = 0.0


def _logsumexp(z: np.ndarray) -> np.ndarray:
    m = z.max(axis=-1, keepdims=True)
    return (m + np.log(np.exp(z - m).sum(axis=-1, keepdims=True)))[..., 0]


def targets(rule: str, q_t, q_aux, a, r, d_t, h: LossHyper) -> np.ndarray:
    """target_tm1 of each rule (stop-gradient), d_t given."""
    q_t = np.asarray(q_t, np.float64)
    if rule in ("q_learning", "q_learning_reg"):
        return r + d_t * q_t.max(axis=-1)
    if rule == "double_q_learning":
        return r + d_t * q_t[np.arange(len(a)), np.asarray(q_aux).argmax(-1)]
    z = np.asarray(q_aux, np.float64) / h.tau   # munchausen_q_learning
    log_pi = z - _logsumexp(z)[:, None]
    m_a = np.clip(h.tau * log_pi[np.arange(len(a)), a], h.clip_value_min, 0.0)
    return r + h.alpha * m_a + d_t * h.tau * _logsumexp(q_t / h.tau)


def loss_and_dq(rule: str, q_tm1, q_t, q_aux, a, reward, done, h: LossHyper, discount=None) -> Tuple[float, np.ndarray]:
    """The batch loss (the q_loss metric) and d loss / d q_tm1."""
    q_tm1 = np.asarray(q_tm1, np.float64)
    M = q_tm1.shape[0]
    a = np.asarray(a, np.int64)
    r = np.clip(np.asarray(reward, np.float64), -h.max_abs_reward, h.max_abs_reward)
    d_t = (1.0 - np.asarray(done, np.float64)) * h.gamma if discount is None else np.asarray(discount, np.float64)
    qa = q_tm1[np.arange(M), a]
    td = targets(rule, q_t, q_aux, a, r, d_t, h) - qa
    if h.huber > 0:
        ax = np.abs(td)
        quad = np.minimum(ax, h.huber)
        loss = 0.5 * quad ** 2 + h.huber * (ax - quad)
        g = np.clip(td, -h.huber, h.huber)
    else:
        loss = 0.5 * td ** 2
        g = td
    dq = np.zeros_like(q_tm1)
    dq[np.arange(M), a] = -g / M
    total = float(loss.mean())
    if rule == "q_learning_reg":
        dq[np.arange(M), a] += h.reg / M
        total += h.reg * float(qa.mean())
    return total, dq


def batch_grad(rule: str, online: O.MLPParams, target: O.MLPParams, obs, next_obs, a, reward, done, h: LossHyper) -> Tuple[float, np.ndarray]:
    """jax.grad(_q_loss_fn) of one shard's batch: (loss, flat gradient of the online network)."""
    q_tm1, acts = O.mlp_forward(online, np.asarray(obs, np.float64))
    q_t, _ = O.mlp_forward(target, np.asarray(next_obs, np.float64))
    q_aux = None
    if rule == "double_q_learning":
        q_aux, _ = O.mlp_forward(online, np.asarray(next_obs, np.float64))
    elif rule == "munchausen_q_learning":
        q_aux, _ = O.mlp_forward(target, np.asarray(obs, np.float64))
    loss, dq = loss_and_dq(rule, q_tm1, q_t, q_aux, a, reward, done, h)
    return loss, O.mlp_backward(online, acts, dq).flat()


def dqn_update(rule: str, online: np.ndarray, target: np.ndarray, st: O.AdamState, epochs: Sequence[Sequence[tuple]], h: LossHyper, lr: float,
               max_grad_norm: float, tau: float, sizes: List[int], activation: str, ln: bool, grad_sync: Optional[Callable] = None,
               eps: float = 1e-5) -> Tuple[np.ndarray, np.ndarray]:
    """_update_epoch x len(epochs) (ff_dqn.py:144-220) on flat online / target vectors.  epochs[k] = one sampled batch per shard
    (obs, next_obs, action, reward, done); the shard gradients are averaged (pmean over "batch"), grad_sync (optional) is the
    pmean over "device"; then clip + Adam and Polyak."""
    b1, b2 = float(np.float32(0.9)), float(np.float32(0.999))
    for batches in epochs:
        on = O.MLPParams.from_flat(online, sizes, activation, ln)
        tg = O.MLPParams.from_flat(target, sizes, activation, ln)
        g = np.mean([batch_grad(rule, on, tg, *b, h)[1] for b in batches], axis=0)
        if grad_sync is not None:
            g = grad_sync(g)
        online, _ = O.clip_adam_step(online, g, st, lr, max_grad_norm, b1, b2, float(np.float32(eps)))
        target = tau * online + (1.0 - tau) * target
    return online, target
