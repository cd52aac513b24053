"""NumPy oracle of Rainbow (stoix/systems/q_learning/ff_rainbow.py), test infrastructure only.

It restates:
  - NoisyLinear (stoix/networks/layers.py:71-169): y = x (mu_w + sigma_w o eps_w) + mu_b + sigma_b o eps_b, eps_w = f(eps_in) f(eps_out)^T,
    eps_b = f(eps_out), f(z) = sign(z) sqrt|z|.  The draws themselves are this project's (Philox4x32-10, include/stx.h); JAX's
    threefry stream is not reproduced.  `effective` / `fold` mirror the kernels' fp32 products in order, so they are exact;
    `noisy_forward64` is the float64 formula.
  - the dueling combine (stoix/networks/dueling.py:117): q[a, i] = v[i] + adv[a, i] - mean_a adv[., i].
  - NoisyLinear init (layers.py:120-150): sigma_w = sigma_b = sigma_zero / sqrt(fan_in).  dueling.py:104-109 builds the value and
    advantage branches as NoisyMLPTorso(layer_sizes, activation, use_layer_norm, sigma_zero): the 4th positional argument binds to
    NoisyMLPTorso's 4th field, kernel_init (torso.py:36-44), which NoisyLinear never reads, so the branch layers keep the default
    sigma_zero = 0.5 while the torso and the two output layers use system.sigma_zero.  Restated as written, not fixed.
  - the n-step transition of ff_rainbow.py:222-246: reward = batch_discounted_returns(r, (1 - done) gamma, 0)[:, 0], i.e.
    G = r_{n-1}, G_k = r_k + (1 - done_k) gamma G_{k+1}; done = any(done); obs / action of step 0, next_obs of step n-1.  The loss then
    bootstraps with gamma (d_t = (1 - done) gamma), not gamma^n: the reference does so and it is kept.
  - the importance weights (:196-200): w_i = (1/p_i)^beta / max_j (1/p_j)^beta, beta = optax.linear_schedule(beta0, 1, steps)(count).
  - the prioritised trajectory buffer.  flashbax is not installed here; its rules as fbx.make_prioritised_trajectory_buffer applies them
    with add_batch_size = E, sample_sequence_length = n, period = 1, max_length_time_axis = L (ff_rainbow.py:433-442):
      * time-major ring, one write index for all envs (flashbax trajectory_buffer: `current_index`);
      * item (env e, start row p) is sampleable only if its n rows are written and do not straddle the write head; unsampleable
        items carry priority 0 (prioritised_trajectory_buffer: the invalid items' priorities are zeroed on add);
      * items that become valid get max_recorded_priority, initially 1.0;
      * set_priorities stores priority ** priority_exponent and raises max_recorded_priority to the largest stored value;
      * sampling is stratified: one uniform in each of M equal slices of the total (sum_tree.stratified_sample), p_i = priority_i / total.
    Where flashbax leaves a rule open this project fixes it: an index given twice to one set_priorities keeps the LAST value in
    batch order; item i = e L + p orders the leaves.  Here validity is evaluated from its definition over all items after every add
    (an item keeps its priority unless it changed validity or contains a row the add wrote), independently of the kernel's window.
"""
from __future__ import annotations

from typing import Dict, Sequence

import numpy as np

from oracle.synth_env import normal2, philox4x32

NOISE_TAG, PRIO_TAG = 0x4E4F4953, 0x5052494F


def noise(seed: int, call: int, count: int) -> np.ndarray:
    """f(z) of noise elements 0 .. count-1 of one call (stx_noisy_weights with draw)."""
    j = np.arange(count, dtype=np.uint64)
    r = philox4x32(j, np.uint64(call & 0xFFFFFFFF), np.uint64(call >> 32), np.uint64(NOISE_TAG), seed & 0xFFFFFFFF, seed >> 32)
    z, _ = normal2(r[0], r[1])
    return (np.sign(z) * np.sqrt(np.abs(z))).astype(np.float32)


def prio_uniforms(seed: int, call: int, M: int) -> np.ndarray:
    r = np.arange(M, dtype=np.uint64)
    w = philox4x32(r >> np.uint64(2), np.uint64(call & 0xFFFFFFFF), np.uint64(call >> 32), np.uint64(PRIO_TAG), seed & 0xFFFFFFFF, seed >> 32)
    words = np.stack(w, -1)[np.arange(M), (r & np.uint64(3)).astype(np.int64)]
    return (((words >> np.uint64(9)).astype(np.float32) + np.float32(0.5)) * np.float32(1.0 / 8388608.0)).astype(np.float32)


def _parts(L: Dict, flat: np.ndarray):
    n_in, n_out, o = L["in_"], L["out"], L["param"]
    W = n_in * n_out
    return (flat[o:o + W].reshape(n_in, n_out), flat[o + W:o + W + n_out], flat[o + W + n_out:o + 2 * W + n_out].reshape(n_in, n_out),
            flat[o + 2 * W + n_out:o + 2 * W + 2 * n_out])


def _f(L: Dict, nz: np.ndarray):
    return nz[L["noise"]:L["noise"] + L["in_"]], nz[L["noise"] + L["in_"]:L["noise"] + L["in_"] + L["out"]]


def effective(layers: Sequence[Dict], params: np.ndarray, nz: np.ndarray, eff_count: int, dtype=np.float32) -> np.ndarray:
    """The effective StxMlp arena, products in the kernel's order (zero where no layer writes); fp32 as the kernel, or float64."""
    eff = np.zeros(eff_count, dtype)
    for L in layers:
        mu_w, mu_b, sg_w, sg_b = (x.astype(dtype) for x in _parts(L, params))
        fin, fout = (x.astype(dtype) for x in _f(L, nz))
        W = mu_w + sg_w * (fin[:, None] * fout[None, :]).astype(dtype)
        for r in range(L["in_"]):
            eff[L["eff_w"] + r * L["ld"]: L["eff_w"] + r * L["ld"] + L["out"]] = W[r]
        eff[L["eff_b"]: L["eff_b"] + L["out"]] = mu_b + sg_b * fout
    return eff


def fold(layers: Sequence[Dict], eff_grad: np.ndarray, nz: np.ndarray, param_count: int) -> np.ndarray:
    """(d mu, d sigma) in the parameter layout from the effective gradient, fp32 products in the kernel's order."""
    g = np.zeros(param_count, np.float32)
    for L in layers:
        n_in, n_out, o = L["in_"], L["out"], L["param"]
        W = n_in * n_out
        fin, fout = _f(L, nz)
        gw = np.stack([eff_grad[L["eff_w"] + r * L["ld"]: L["eff_w"] + r * L["ld"] + n_out] for r in range(n_in)]).astype(np.float32)
        gb = eff_grad[L["eff_b"]: L["eff_b"] + n_out].astype(np.float32)
        g[o:o + W] = gw.reshape(-1)
        g[o + W:o + W + n_out] = gb
        g[o + W + n_out:o + 2 * W + n_out] = (gw * (fin[:, None] * fout[None, :]).astype(np.float32)).reshape(-1)
        g[o + 2 * W + n_out:o + 2 * W + 2 * n_out] = gb * fout
    return g


def _silu(x):
    return x / (1.0 + np.exp(-x))


def noisy_forward64(layers: Sequence[Dict], params: np.ndarray, nz: np.ndarray, x: np.ndarray, n_torso: int, n_branch: int) -> np.ndarray:
    """(v | adv) rows of the reference network (dueling.py:103-116) in float64, silu everywhere but the output layers."""
    def lin(L, h):
        mu_w, mu_b, sg_w, sg_b = (np.asarray(p, np.float64) for p in _parts(L, params))
        fin, fout = (np.asarray(f, np.float64) for f in _f(L, nz))
        return h @ (mu_w + sg_w * np.outer(fin, fout)) + mu_b + sg_b * fout

    h = np.asarray(x, np.float64)
    for L in layers[:n_torso]:
        h = _silu(lin(L, h))
    branches = []
    for b in range(2):
        hb = h
        for L in layers[n_torso + b * n_branch: n_torso + (b + 1) * n_branch]:
            hb = _silu(lin(L, hb))
        branches.append(hb)
    return np.concatenate([lin(layers[-2], branches[0]), lin(layers[-1], branches[1])], axis=1)


def dueling_combine(head: np.ndarray, A: int, N: int) -> np.ndarray:
    head = np.asarray(head, np.float64)
    v, adv = head[:, None, :N], head[:, N:].reshape(-1, A, N)
    return (v + adv - adv.mean(1, keepdims=True)).reshape(-1, A * N)


def dueling_backward(dq: np.ndarray, A: int, N: int) -> np.ndarray:
    dq = np.asarray(dq, np.float64).reshape(-1, A, N)
    s = dq.sum(1)
    return np.concatenate([s, (dq - s[:, None, :] / A).reshape(-1, A * N)], axis=1)


def n_step_return(r: np.ndarray, done: np.ndarray, gamma: float) -> float:
    """sum_k (prod_{j<k} (1 - done_j) gamma) r_k, float64."""
    g, disc = 0.0, 1.0
    for k in range(len(r)):
        g += disc * float(r[k])
        disc *= (1.0 - float(done[k])) * gamma
    return g


def n_step_return32(r: np.ndarray, done: np.ndarray, gamma: float) -> np.float32:
    """The kernel's fp32 evaluation: the reference's backward recursion, each product and sum rounded."""
    g = np.float32(r[-1])
    for k in range(len(r) - 2, -1, -1):
        g = np.float32(r[k]) + np.float32((np.float32(1.0) - np.float32(done[k])) * np.float32(gamma)) * g
    return np.float32(g)


def beta_at(count: int, beta0: float, steps: float) -> float:
    if steps <= 0:
        return beta0
    c = min(max(float(count), 0.0), steps)
    return (beta0 - 1.0) * (1.0 - c / steps) + 1.0


def importance_weights(prob: np.ndarray, beta: float) -> np.ndarray:
    iw = (1.0 / np.asarray(prob, np.float64)) ** beta
    return iw / iw.max()


class PrioRing:
    """The prioritised n-step trajectory buffer, rules as in the module docstring."""

    def __init__(self, L: int, E: int, D: int, n: int, alpha: float):
        self.L, self.E, self.D, self.n, self.alpha = L, E, D, n, alpha
        self.obs, self.next_obs = np.zeros((L, E, D), np.float32), np.zeros((L, E, D), np.float32)
        self.action, self.reward, self.done = np.zeros((L, E), np.int32), np.zeros((L, E), np.float32), np.zeros((L, E), np.uint8)
        self.w, self.c = 0, 0
        self.prio = np.zeros(E * L)
        self.maxp = 1.0

    def valid(self, p: int) -> bool:
        age = (self.w - 1 - p) % self.L
        return self.n - 1 <= age < self.c

    def add(self, obs, action, reward, done, next_obs) -> None:
        T = reward.shape[0]
        written = set()
        for t in range(max(0, T - self.L), T):
            row = (self.w + t) % self.L
            self.obs[row], self.next_obs[row], self.action[row] = obs[t], next_obs[t], action[t]
            self.reward[row], self.done[row] = reward[t], done[t]
            written.add(row)
        self.w, self.c = (self.w + T) % self.L, min(self.c + T, self.L)
        for e in range(self.E):
            for p in range(self.L):
                i = e * self.L + p
                if not self.valid(p):
                    self.prio[i] = 0.0
                elif any((p + k) % self.L in written for k in range(self.n)):
                    self.prio[i] = self.maxp

    def sample(self, u: np.ndarray) -> np.ndarray:
        """The first item whose cumulative priority exceeds v = (r + u_r) total / M; at or past the total, the last positive item
        (with no positive item, item 0)."""
        M = len(u)
        cum = np.cumsum(self.prio)
        pos = np.flatnonzero(self.prio > 0)
        if len(pos) == 0:
            return np.zeros(M, np.int64)
        v = (np.arange(M) + np.asarray(u, np.float64)) * cum[-1] / M
        return np.minimum(np.searchsorted(cum, v, side="right"), pos[-1])

    def transition(self, i: int, gamma: float):
        e, p = divmod(int(i), self.L)
        rows = [(p + k) % self.L for k in range(self.n)]
        r, d = self.reward[rows, e], self.done[rows, e]
        return self.obs[p, e], self.action[p, e], n_step_return(r, d, gamma), bool(d.any()), self.next_obs[rows[-1], e], r, d

    def set_priorities(self, idx: Sequence[int], pr: np.ndarray) -> None:
        new = np.asarray(pr, np.float64) ** self.alpha
        for m, i in enumerate(idx):
            self.prio[int(i)] = new[m]
        self.maxp = max(self.maxp, float(new.max()))


def tree_floats(items: int, fanout: int = 32) -> int:
    total, c = 0, items
    while True:
        total += c
        if c <= 1:
            return total
        c = (c + fanout - 1) // fanout
