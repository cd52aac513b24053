"""fp64 restatement of R2D2 (stoix/systems/q_learning/rec_r2d2.py) for the tests.

Upstream rules restated here (flashbax, rlax and flax are not installed):
- The prioritised sequence ring (fbx.make_prioritised_trajectory_buffer with add_batch_size E, sample_sequence_length S, period p):
  L = max_size // E time rows with one write index; item (e, k), k < L // p, is env e's sequence starting at ring row k p; it is
  valid iff S - 1 <= age(k p) < c with age(row) = (w - 1 - row) mod L and c = min(rows written, L).  After an add, the items whose
  start row lies in w0 - S + 1 .. w0 + T - 1 (mod L, at most L rows) get max_priority if valid, else 0.  Sampling is Rainbow's
  stratified descent of the sum tree; set_priorities stores priority ** alpha (the last of duplicate indices wins) and raises the max.
- rlax.transformed_n_step_q_learning with SIGNED_HYPERBOLIC_PAIR and the reference's importance weights and priorities.
- DuelingQNetwork(use_layer_norm=True): MLPTorso branches whose last Dense has no bias and is followed by a LayerNorm (eps 1e-6)
  without activation; q = v + (adv - mean adv).

The ring, the loss and the dueling combine are NumPy; the recurrent network is written in torch float64 on the CPU so that one
optimiser step's gradient comes from autograd through exactly the reference's graph (burn-in and targets under stop_gradient)."""
from __future__ import annotations

from typing import Dict, List, Optional

import numpy as np
import torch

TX_EPS = 1e-3
FANOUT = 32


# ---------------------------------------------------------------------------------------------------------- value transform ----
def h(x, eps: float = TX_EPS):
    """rlax.signed_hyperbolic, published form."""
    x = np.asarray(x, np.float64)
    return np.sign(x) * (np.sqrt(np.abs(x) + 1.0) - 1.0) + eps * x


def h_inv(x, eps: float = TX_EPS):
    """rlax.signed_parabolic, published form."""
    x = np.asarray(x, np.float64)
    z = np.sqrt(1.0 + 4.0 * eps * (eps + 1.0 + np.abs(x))) / 2.0 / eps - 1.0 / 2.0 / eps
    return np.sign(x) * (np.square(z) - 1.0)


def h_stable(x, eps: float = TX_EPS):
    """h without cancellation near 0: sqrt(|x| + 1) - 1 = |x| / (sqrt(|x| + 1) + 1).  In fp64 the published form loses every digit
    for |x| below about 1e-16."""
    x = np.asarray(x, np.float64)
    return np.sign(x) * np.abs(x) / (np.sqrt(np.abs(x) + 1.0) + 1.0) + eps * x


def h_inv_stable(x, eps: float = TX_EPS):
    """h^-1 without cancellation near 0: z = 1 + delta, delta = 2 |x| (1 - 2 eps / (1 + 2 eps + s)) / (s + 1), s = sqrt(1 + 4 eps (eps
    + 1 + |x|)), and z^2 - 1 = delta (2 + delta)."""
    x = np.asarray(x, np.float64)
    ax = np.abs(x)
    s = np.sqrt(1.0 + 4.0 * eps * (eps + 1.0 + ax))
    delta = 2.0 * ax * (1.0 - 2.0 * eps / (1.0 + 2.0 * eps + s)) / (s + 1.0)
    return np.sign(x) * delta * (2.0 + delta)


def transformed_n_step_returns(r_t, d_t, v_t, n: int):
    """rlax.transformed_n_step_returns with lambda 1: r padded with n-1 zeros, d with n-1 ones, v shifted by n-1 and padded with
    its last value; targets = h(r_i + d_i h^-1(targets)) for i = n-1 .. 0."""
    seq = len(r_t)
    r = np.concatenate([r_t, np.zeros(n - 1)])
    d = np.concatenate([d_t, np.ones(n - 1)])
    targets = np.concatenate([v_t[n - 1:], np.full(min(n - 1, seq), v_t[-1])])
    for i in reversed(range(n)):
        targets = h(r[i:i + seq] + d[i:i + seq] * h_inv(targets))
    return targets


def beta_at(count: int, beta0: float, steps: float) -> float:
    if steps <= 0:
        return beta0
    c = min(max(count, 0), steps)
    return (beta0 - 1.0) * (1.0 - c / steps) + 1.0


def loss(q, q_tg, action, reward, done, prob, n: int, gamma: float, max_abs_reward: float, eta: float, beta: float) -> Dict[str, np.ndarray]:
    """_q_loss_fn (rec_r2d2.py:331-384) over a learn window: q, q_tg (T, B, A); returns td (T-1, B), d_q (T, B, A), priorities (B),
    the loss and the metrics in ops.R2D2_METRICS order."""
    q, q_tg = np.asarray(q, np.float64), np.asarray(q_tg, np.float64)
    T, B, A = q.shape
    sel = np.argmax(q, axis=-1)
    r = np.clip(np.asarray(reward, np.float64), -max_abs_reward, max_abs_reward)
    d = (1.0 - np.asarray(done, np.float64)) * gamma
    td = np.zeros((T - 1, B))
    for b in range(B):
        v = q_tg[1:, b][np.arange(T - 1), sel[1:, b]]
        tgt = transformed_n_step_returns(r[:-1, b], d[:-1, b], v, n)
        td[:, b] = tgt - q[:-1, b][np.arange(T - 1), action[:-1, b]]
    per_seq = 0.5 * np.square(td).sum(axis=0)
    iw = (1.0 / (np.asarray(prob, np.float64) + 1e-6)) ** beta
    w = iw / iw.max()
    mean_loss = np.mean(w * per_seq)
    d_q = np.zeros((T, B, A))
    for t in range(T - 1):
        d_q[t, np.arange(B), action[t]] = -w * td[t] / B
    a = np.abs(td)
    pr = eta * a.max(axis=0) + (1 - eta) * a.mean(axis=0)
    metrics = np.array([mean_loss, q.mean(), pr.max(), pr.mean(), a.max(axis=0).mean(), a.mean(axis=0).mean()])
    return {"td": td, "d_q": d_q, "priorities": pr, "loss": mean_loss, "metrics": metrics, "weights": w}


# ---------------------------------------------------------------------------------------------------------- the ring ----
class Ring:
    """The prioritised sequence ring of one shard (rows as numpy arrays, priorities as leaves)."""

    def __init__(self, L: int, E: int, S: int, period: int, alpha: float):
        self.L, self.E, self.S, self.p, self.alpha = L, E, S, period, alpha
        self.K = L // period
        self.w = self.c = 0
        self.max_priority = 1.0
        self.leaves = np.zeros(E * self.K)
        self.rows: Dict[str, np.ndarray] = {}
        self.carry: Optional[np.ndarray] = None

    def add(self, **batch: np.ndarray) -> None:
        """batch: time-major (T, E, ...) arrays, `carry` included (stored at item-start rows only)."""
        T = batch["reward"].shape[0]
        skip = max(T - self.L, 0)
        for name, x in batch.items():
            if name == "carry":
                if self.carry is None:
                    self.carry = np.zeros((self.K, self.E) + x.shape[2:], x.dtype)
            elif name not in self.rows:
                self.rows[name] = np.zeros((self.L,) + x.shape[1:], x.dtype)
        for t in range(skip, T):
            row = (self.w + t) % self.L
            for name, x in batch.items():
                if name == "carry":
                    if row % self.p == 0 and row // self.p < self.K:
                        self.carry[row // self.p] = x[t]
                else:
                    self.rows[name][row] = x[t]
        w0 = self.w
        self.w, self.c = (w0 + T) % self.L, min(self.c + T, self.L)
        win, first = min(T + self.S - 1, self.L), (w0 - (self.S - 1)) % self.L
        for e in range(self.E):
            for k in range(self.K):
                start = k * self.p
                if (start - first) % self.L < win:
                    self.leaves[e * self.K + k] = self.max_priority if self.valid(start) else 0.0

    def valid(self, start: int) -> bool:
        age = (self.w - 1 - start) % self.L
        return self.S - 1 <= age < self.c

    def valid_items(self) -> List[int]:
        return [e * self.K + k for e in range(self.E) for k in range(self.K) if self.valid(k * self.p)]

    def tree(self) -> List[np.ndarray]:
        """Levels leaves-first, each parent the fp32 sum of its children in order (the device's rounding)."""
        levels = [self.leaves.astype(np.float32)]
        while len(levels[-1]) > 1:
            ch = levels[-1]
            levels.append(np.array([_fsum(ch[i:i + FANOUT]) for i in range(0, len(ch), FANOUT)], np.float32))
        return levels

    def sample_items(self, u: np.ndarray) -> np.ndarray:
        """Stratified descent with the uniforms u (B) in fp32, as the device: v = ((b + u_b) total) / B.  A level where no child takes
        v (fp32 rounding left v at or past the node's sum) takes its last positive child, and so does every level below it (v = +inf)."""
        levels = self.tree()
        B = len(u)
        total = levels[-1][0]
        out = np.zeros(B, np.int64)
        for b in range(B):
            v = np.float32(np.float32(np.float32(np.float32(b) + np.float32(u[b])) * total) / np.float32(B))
            node = 0
            for lv in range(len(levels) - 1, 0, -1):
                ch = levels[lv - 1][node * FANOUT: node * FANOUT + FANOUT]
                pick, last_pos = -1, 0
                for c, s in enumerate(ch):
                    if s > 0:
                        last_pos = c
                    if pick < 0:
                        if v < s:
                            pick = c
                        else:
                            v = np.float32(v - s)
                if pick < 0:
                    v = np.float32(np.inf)
                node = node * FANOUT + (last_pos if pick < 0 else pick)
            out[b] = node
        return out

    def probabilities(self, items) -> np.ndarray:
        levels = self.tree()
        total = levels[-1][0]
        return (levels[0][items] / total).astype(np.float32) if total > 0 else np.zeros(len(items), np.float32)

    def sequence(self, item: int) -> Dict[str, np.ndarray]:
        e, k = divmod(int(item), self.K)
        rows = [(k * self.p + t) % self.L for t in range(self.S)]
        out = {name: x[rows, e] for name, x in self.rows.items()}
        out["carry0"] = self.carry[k, e]
        return out

    def set_priorities(self, idx, pr) -> None:
        for i, v in zip(idx, pr):   # the last occurrence wins
            self.leaves[int(i)] = float(np.float32(v) ** np.float32(self.alpha))
        self.max_priority = max(self.max_priority, max(float(np.float32(v) ** np.float32(self.alpha)) for v in pr))


def _fsum(xs) -> np.float32:
    s = np.float32(0)
    for x in xs:
        s = np.float32(s + x)
    return s


# ---------------------------------------------------------------------------------------------------------- the network ----
def _mlp(spec, flat: torch.Tensor, x: torch.Tensor) -> torch.Tensor:
    """An ops.MlpSpec network in float64: Dense (no bias when LayerNorm) -> LayerNorm(eps 1e-6) -> activation on torso layers; the
    last layer Dense + bias, or with ln_final Dense -> LayerNorm, no activation."""
    sl, lb = spec.layer_slices(), spec.ln_bias_slices()
    act = {"relu": torch.relu, "silu": torch.nn.functional.silu, "tanh": torch.tanh}[spec.activation]
    for i in range(spec.n_layers):
        W = flat[sl[i][0]].view(spec.sizes[i], spec.sizes[i + 1])
        y = x @ W
        if spec.has_ln(i):
            y = torch.nn.functional.layer_norm(y, (spec.sizes[i + 1],), flat[sl[i][1]], flat[lb[i]], eps=1e-6)
        else:
            y = y + flat[sl[i][1]]
        x = act(y) if i < spec.n_layers - 1 else y
    return x


def network(lay, flat: torch.Tensor, obs: torch.Tensor, reset: torch.Tensor, carry: torch.Tensor):
    """ScannedRNN + RecurrentActor over (T, B, D) rows from carry (B, carry_dim): returns (q (T, B, A), last carry)."""
    T, B, D = obs.shape
    H = lay.H
    pre, w_h, b_hn, post = lay.blocks(flat)
    gi = _mlp(lay.spec_pre, pre, obs.reshape(T * B, D)).view(T, B, -1)
    hs = []
    for t in range(T):
        carry = torch.where(reset[t].bool()[:, None], torch.zeros_like(carry), carry)
        gh = carry[:, -H:] @ w_h if lay.cell_type == "lstm" else carry @ w_h
        if lay.cell_type == "gru":
            r = torch.sigmoid(gi[t, :, :H] + gh[:, :H])
            z = torch.sigmoid(gi[t, :, H:2 * H] + gh[:, H:2 * H])
            nn_ = torch.tanh(gi[t, :, 2 * H:] + r * (gh[:, 2 * H:] + b_hn))
            carry = (1 - z) * nn_ + z * carry
            hs.append(carry)
        else:
            g = gi[t] + gh
            i_, f_, g_, o_ = torch.sigmoid(g[:, :H]), torch.sigmoid(g[:, H:2 * H]), torch.tanh(g[:, 2 * H:3 * H]), torch.sigmoid(g[:, 3 * H:])
            c = f_ * carry[:, :H] + i_ * g_
            hh = o_ * torch.tanh(c)
            carry = torch.cat([c, hh], dim=1)
            hs.append(hh)
    out = _mlp(lay.spec_post, post, torch.stack(hs).reshape(T * B, H))
    if lay.dueling:
        out = lay.value_bias(flat) + (out - out.mean(dim=-1, keepdim=True))
    return out.view(T, B, -1), carry


def q_loss_grad(lay, online: np.ndarray, target: np.ndarray, seq: Dict[str, np.ndarray], burn_in: int, prob, n: int, gamma: float,
                max_abs_reward: float, eta: float, beta: float):
    """jax.grad(_q_loss_fn) of one batch (S, B) in float64: burn-in of both networks under stop_gradient, the target's and the online
    learn-window Q, the loss oracle's d Q pushed back through the online learn window by autograd.  Returns (grad, loss dict)."""
    f64 = lambda x: torch.as_tensor(np.asarray(x), dtype=torch.float64)
    on, tg = f64(online).requires_grad_(True), f64(target)
    obs, reset, carry0 = f64(seq["obs"]), torch.as_tensor(np.asarray(seq["reset"])), f64(seq["carry0"])
    with torch.no_grad():
        _, c_on = network(lay, on.detach(), obs[:burn_in], reset[:burn_in], carry0)
        _, c_tg = network(lay, tg, obs[:burn_in], reset[:burn_in], carry0)
        q_tg, _ = network(lay, tg, obs[burn_in:], reset[burn_in:], c_tg)
    q, _ = network(lay, on, obs[burn_in:], reset[burn_in:], c_on)
    out = loss(q.detach().numpy(), q_tg.numpy(), np.asarray(seq["action"])[burn_in:], np.asarray(seq["reward"])[burn_in:],
               np.asarray(seq["done"])[burn_in:], prob, n, gamma, max_abs_reward, eta, beta)
    q.backward(f64(out["d_q"]))
    return on.grad.numpy(), out


def clip_adam(params, grad, mu, nu, count: int, lr: float, max_norm: float, b1=0.9, b2=0.999, eps=1e-5):
    """optax.chain(clip_by_global_norm, adam(eps=1e-5)) step `count` (0-based) in float64."""
    g = np.asarray(grad, np.float64)
    norm = np.sqrt(np.sum(g * g))
    g = g * (max_norm / norm) if norm > max_norm else g
    mu = b1 * mu + (1 - b1) * g
    nu = b2 * nu + (1 - b2) * g * g
    k = count + 1
    upd = -lr * (mu / (1 - b1 ** k)) / (np.sqrt(nu / (1 - b2 ** k)) + eps)
    return params + upd, mu, nu
