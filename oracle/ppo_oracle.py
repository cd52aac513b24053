"""CPU oracle for the Anakin ff_ppo hot path  --  TEST INFRASTRUCTURE, NOT PRODUCT.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` /
``--impl reference`` legs may import this module.  The product (``stoix_b200``) never does: it
fails loudly when the CUDA library is missing.

It restates, in NumPy (float64 by default, float32 on request), the arithmetic of the reference
path named by BASELINE.json's north_star.  Every function cites the reference file:line it follows
(paths relative to /root/reference).

Parity status
-------------
* GAE (``gae``): PINNED against every vector of stoix/tests/multistep_test.py (see
  tests/test_oracle_golden.py, tests/golden/multistep_vectors.json).
* Everything else (MLP, Categorical, losses, optax clip+adam, LR schedule, epoch/minibatch loop):
  **parity unpinned** by the reference's own tests (it has none for these; JAX/Flax/Optax/TFP are
  not installable here and have no wheels in /opt/wheelhouse).  They are restated from the call
  sites in stoix/systems/ppo/anakin/ff_ppo.py and the published definitions of the pinned
  third-party versions (optax 0.2.7.dev0@17411bc, flax 0.10.5, tfp 0.25.0, jax 0.5.3); the manual
  backward pass below is itself cross-checked against torch.autograd in tests/test_oracle_grads.py.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

# --------------------------------------------------------------------------------------------
# A.1  GAE  -- stoix/utils/multistep.py:14-145
# --------------------------------------------------------------------------------------------


def standardize(x: np.ndarray, eps: float = 1e-5) -> np.ndarray:
    """jax.nn.standardize(x, axis=all) as called at multistep.py:138-139 (jax 0.5.3):
    mean = E[x]; var = E[x^2] - mean^2 (single-pass form); out = (x - mean) * rsqrt(var + eps)."""
    mean = x.mean()
    var = (x * x).mean() - mean * mean
    return (x - mean) / np.sqrt(var + eps)


def gae(
    r_t: np.ndarray,
    discount_t: np.ndarray,
    lambda_,
    values: Optional[np.ndarray] = None,
    v_tm1: Optional[np.ndarray] = None,
    v_t: Optional[np.ndarray] = None,
    truncation_t: Optional[np.ndarray] = None,
    time_major: bool = False,
    standardize_advantages: bool = False,
    dtype=np.float64,
) -> Tuple[np.ndarray, np.ndarray]:
    """batch_truncated_generalized_advantage_estimation, multistep.py:14-145.

    Same argument names and meaning as the reference.  The reverse recurrence is evaluated
    sequentially in ``dtype`` in exactly the written order
    ``acc = delta + discount * lambda * acc * (1 - trunc)`` (multistep.py:119-124)."""
    r_t = np.asarray(r_t, dtype)
    discount_t = np.asarray(discount_t, dtype)
    if values is not None:  # multistep.py:82-92
        values = np.asarray(values, dtype)
        assert values.ndim == 2
        if time_major:
            v_tm1, v_t = values[:-1], values[1:]
        else:
            v_tm1, v_t = values[:, :-1], values[:, 1:]
    assert v_tm1 is not None and v_t is not None
    v_tm1 = np.asarray(v_tm1, dtype)
    v_t = np.asarray(v_t, dtype)
    assert r_t.ndim == 2 and r_t.shape == v_tm1.shape == v_t.shape == discount_t.shape
    lam = np.ones_like(discount_t) * np.asarray(lambda_, dtype)  # multistep.py:97
    if truncation_t is None:  # multistep.py:100-105
        trunc = np.zeros_like(discount_t)
    else:
        trunc = np.asarray(truncation_t).astype(dtype)
        assert trunc.shape == discount_t.shape
    if not time_major:  # multistep.py:107-113
        r_t, discount_t, v_tm1, v_t, lam, trunc = (
            a.T for a in (r_t, discount_t, v_tm1, v_t, lam, trunc)
        )
    delta = r_t + discount_t * v_t - v_tm1  # multistep.py:116
    T = r_t.shape[0]
    adv = np.zeros_like(delta)
    acc = np.zeros(r_t.shape[1], dtype)  # multistep.py:127
    one = dtype(1.0)
    for t in range(T - 1, -1, -1):  # multistep.py:119-130 (reverse scan)
        acc = delta[t] + discount_t[t] * lam[t] * acc * (one - trunc[t])
        adv[t] = acc
    targets = v_tm1 + adv  # multistep.py:132 (before standardisation)
    if not time_major:  # multistep.py:134-136
        adv, targets = adv.T, targets.T
    if standardize_advantages:  # multistep.py:138-139
        adv = standardize(adv).astype(dtype)
    return np.ascontiguousarray(adv), np.ascontiguousarray(targets)


def ppo_gae_inputs(reward, done, truncated, gamma, reward_scale, dtype=np.float64):
    """ff_ppo.py:164-169: r_t = reward*reward_scale, d_t = (1-done)*gamma, trunc = truncated."""
    r_t = np.asarray(reward, dtype) * dtype(reward_scale)
    d_t = (dtype(1.0) - np.asarray(done).astype(dtype)) * dtype(gamma)
    return r_t, d_t, np.asarray(truncated).astype(dtype)


# --------------------------------------------------------------------------------------------
# A.2 / A.3  networks -- stoix/networks/{base,torso,heads}.py
# --------------------------------------------------------------------------------------------


@dataclass
class MLPParams:
    """One network: MLPTorso(activation, use_layer_norm, activate_final=True) + Dense head (torso.py:12-33, heads.py:36,134).
    W[i] has flax layout (in, out), y = x @ W + b.  LayerNorm torsos (torso.py:26-30): torso Dense layers have NO bias
    (b[i] is then the LayerNorm SCALE) and ln_bias[i] is the LayerNorm bias; the head is always W, b."""

    W: List[np.ndarray]
    b: List[np.ndarray]
    activation: str = "relu"
    ln_bias: Optional[List[Optional[np.ndarray]]] = None   # None: no LayerNorm anywhere

    def _like(self, W, b, ln):
        return MLPParams(W, b, self.activation, ln)

    def has_ln(self, i: int) -> bool:
        return self.ln_bias is not None and i < len(self.W) - 1

    def copy(self) -> "MLPParams":
        return self._like([w.copy() for w in self.W], [b.copy() for b in self.b],
                          None if self.ln_bias is None else [None if x is None else x.copy() for x in self.ln_bias])

    def astype(self, dt) -> "MLPParams":
        return self._like([w.astype(dt) for w in self.W], [b.astype(dt) for b in self.b],
                          None if self.ln_bias is None else [None if x is None else x.astype(dt) for x in self.ln_bias])

    def flat(self) -> np.ndarray:
        """Arena order used by the CUDA library: W0,b0,W1,b1,... each row-major (LayerNorm layers: W, scale, bias)."""
        parts = []
        for i, (w, b) in enumerate(zip(self.W, self.b)):
            parts += [w.ravel(), b.ravel()]
            if self.has_ln(i):
                parts.append(self.ln_bias[i].ravel())
        return np.concatenate(parts)

    @staticmethod
    def from_flat(flat: np.ndarray, sizes: Sequence[int], activation: str = "relu", use_layer_norm: bool = False) -> "MLPParams":
        W, b, ln, o = [], [], [], 0
        n_layers = len(sizes) - 1
        for i in range(n_layers):
            n = sizes[i] * sizes[i + 1]
            W.append(flat[o : o + n].reshape(sizes[i], sizes[i + 1]).copy())
            o += n
            b.append(flat[o : o + sizes[i + 1]].copy())
            o += sizes[i + 1]
            if use_layer_norm and i < n_layers - 1:
                ln.append(flat[o : o + sizes[i + 1]].copy())
                o += sizes[i + 1]
            else:
                ln.append(None)
        assert o == flat.size
        return MLPParams(W, b, activation, ln if use_layer_norm else None)


# stoix/networks/utils.py:9-24 (flax.linen functions): value and derivative w.r.t. the pre-activation
_SQ2PI = 0.7978845608028654


def _sigmoid(z):
    return 1.0 / (1.0 + np.exp(-z))


ACTIVATIONS = {
    "relu": (lambda z: np.maximum(z, 0.0), lambda z: (z > 0).astype(z.dtype)),
    "tanh": (np.tanh, lambda z: 1.0 - np.tanh(z) ** 2),
    "silu": (lambda z: z * _sigmoid(z), lambda z: _sigmoid(z) * (1.0 + z * (1.0 - _sigmoid(z)))),
    "elu": (lambda z: np.where(z > 0, z, np.expm1(z)), lambda z: np.where(z > 0, 1.0, np.exp(z))),
    # nn.gelu(approximate=True), the flax default
    "gelu": (lambda z: 0.5 * z * (1.0 + np.tanh(_SQ2PI * (z + 0.044715 * z ** 3))),
             lambda z: 0.5 * (1.0 + np.tanh(_SQ2PI * (z + 0.044715 * z ** 3)))
             + 0.5 * z * (1.0 - np.tanh(_SQ2PI * (z + 0.044715 * z ** 3)) ** 2) * _SQ2PI * (1.0 + 3 * 0.044715 * z ** 2)),
    "sigmoid": (_sigmoid, lambda z: _sigmoid(z) * (1.0 - _sigmoid(z))),
    "softplus": (lambda z: np.logaddexp(z, 0.0), _sigmoid),
    "identity": (lambda z: z, lambda z: np.ones_like(z)),
}
ACTIVATIONS["swish"] = ACTIVATIONS["silu"]
ACTIVATIONS["none"] = ACTIVATIONS["identity"]
LN_EPS = 1e-6  # flax nn.LayerNorm default epsilon


def orthogonal_init(rng: np.random.Generator, shape, scale: float) -> np.ndarray:
    """flax.linen.initializers.orthogonal(scale): scale * Q of a normal matrix (QR, sign-fixed).
    Not bit-compatible with JAX's threefry stream (SURVEY A.7) -- parity tests inject params."""
    n_in, n_out = shape
    a = rng.standard_normal((max(n_in, n_out), min(n_in, n_out)))
    q, r = np.linalg.qr(a)
    q = q * np.sign(np.diag(r))
    if n_in < n_out:
        q = q.T
    return scale * q


def init_mlp(rng, sizes: Sequence[int], head_scale: float, dtype=np.float64) -> MLPParams:
    """torso: orthogonal(sqrt 2) (torso.py:18); head: orthogonal(head_scale) (heads.py:32,130);
    zero biases (flax Dense default)."""
    W, b = [], []
    for i in range(len(sizes) - 1):
        scale = np.sqrt(2.0) if i < len(sizes) - 2 else head_scale
        W.append(orthogonal_init(rng, (sizes[i], sizes[i + 1]), scale).astype(dtype))
        b.append(np.zeros(sizes[i + 1], dtype))
    return MLPParams(W, b)


def _bf16_round(x: np.ndarray) -> np.ndarray:
    """Round-to-nearest-even to bfloat16 precision (emulates the tensor-core operand format).
    uint32 arithmetic throughout (the carry of the rounding add never leaves 32 bits for finite inputs)."""
    x32 = np.ascontiguousarray(x, dtype=np.float32)
    u = x32.view(np.uint32)
    rounded = (u + (np.uint32(0x7FFF) + ((u >> np.uint32(16)) & np.uint32(1)))) & np.uint32(0xFFFF0000)
    out = rounded.view(np.float32).reshape(x32.shape)
    return out.astype(x.dtype if x.dtype in (np.float32, np.float64) else np.float32)


def mlp_forward(p: MLPParams, x: np.ndarray, bf16_operands: bool = False):
    """MLPTorso (activate_final=True) followed by a Dense head.  Returns (out, cache); cache[i] is the INPUT of layer i
    (what the backward pass multiplies dY with); for LayerNorm / non-relu torsos the cache also carries the
    pre-activations (`cache.pre[i]`: Dense output of torso layer i, `cache.stats[i]`: its per-row (mean, rstd)).

    ``bf16_operands=True`` emulates the tensor-core path (relu, no LayerNorm only): every GEMM operand (activations
    and weights) is rounded to bf16, products/accumulation stay in the working precision."""
    rnd = _bf16_round if bf16_operands else (lambda a: a)
    f, _ = ACTIVATIONS[p.activation]
    acts = _Cache([rnd(x)])
    h = acts[0]
    n = len(p.W)
    for i in range(n):
        if i < n - 1 and p.has_ln(i):
            assert not bf16_operands, "the bf16 emulation covers the relu / no-LayerNorm networks of the bf16 tensor-core path"
            u = h @ p.W[i]                                          # Dense(use_bias=False), torso.py:26
            mean = u.mean(axis=-1, keepdims=True)
            rstd = 1.0 / np.sqrt(((u - mean) ** 2).mean(axis=-1, keepdims=True) + LN_EPS)
            z = (u - mean) * rstd * p.b[i] + p.ln_bias[i]           # nn.LayerNorm(): scale, bias
            acts.pre.append(u), acts.stats.append((mean, rstd))
        else:
            z = h @ rnd(p.W[i]) + p.b[i]
            acts.pre.append(z), acts.stats.append(None)
        if i < n - 1:
            h = rnd(f(z))
            acts.append(h)
        else:
            out = z
    return out, acts


class _Cache(list):
    """list of layer inputs (what the existing callers index) + pre-activations / LayerNorm statistics."""

    def __init__(self, items):
        super().__init__(items)
        self.pre, self.stats = [], []


def mlp_backward(p: MLPParams, acts, dout: np.ndarray, bf16_operands: bool = False) -> MLPParams:
    """Manual reverse-mode of mlp_forward: grads wrt W[i], b[i] (LayerNorm layers: scale in b[i], bias in ln_bias[i])
    given d(loss)/d(out)."""
    rnd = _bf16_round if bf16_operands else (lambda a: a)
    _, fp = ACTIVATIONS[p.activation]
    n = len(p.W)
    gW, gb = [None] * n, [None] * n
    gln = [None] * n
    d = dout   # gradient w.r.t. the Dense output of layer i
    for i in range(n - 1, -1, -1):
        dr = rnd(d)
        gW[i] = acts[i].T @ dr
        if p.has_ln(i):
            gb[i], gln[i] = d_scale, d_lnbias   # computed when stepping through layer i's LayerNorm below (from layer i+1)
        else:
            gb[i] = d.sum(axis=0)
        if i > 0:
            dh = dr @ rnd(p.W[i]).T                                  # w.r.t. h_{i-1} = f(z_{i-1})
            j = i - 1
            if p.has_ln(j):
                u, (mean, rstd) = acts.pre[j], acts.stats[j]
                uh = (u - mean) * rstd
                dz = dh * fp(uh * p.b[j] + p.ln_bias[j])
                d_scale, d_lnbias = (dz * uh).sum(axis=0), dz.sum(axis=0)
                dhat = dz * p.b[j]
                d = rstd * (dhat - dhat.mean(axis=-1, keepdims=True) - uh * (dhat * uh).mean(axis=-1, keepdims=True))
            elif p.activation == "relu":
                d = dh * (acts[i] > 0)                               # identical to f'(z) for relu; keeps the bf16 path's form
            else:
                d = dh * fp(acts.pre[j])
    return MLPParams(gW, gb, p.activation, gln if p.ln_bias is not None else None)


def log_softmax(z: np.ndarray) -> np.ndarray:
    m = z.max(axis=-1, keepdims=True)
    s = z - m
    return s - np.log(np.exp(s).sum(axis=-1, keepdims=True))


def categorical_log_prob(logits, action):
    """tfd.Categorical(logits).log_prob(a) = log_softmax(logits)[a]  (heads.py:41)."""
    lp = log_softmax(logits)
    return np.take_along_axis(lp, np.asarray(action)[..., None].astype(np.int64), axis=-1)[..., 0]


def categorical_entropy(logits):
    """tfd.Categorical(logits).entropy() = -sum softmax * log_softmax."""
    lp = log_softmax(logits)
    return -(np.exp(lp) * lp).sum(axis=-1)


# --------------------------------------------------------------------------------------------
# A.4  losses -- stoix/utils/loss.py:17-32, 68-78 ; loss fns ff_ppo.py:191-235
# --------------------------------------------------------------------------------------------


def ppo_clip_loss(pi_log_prob_t, b_pi_log_prob_t, gae_t, epsilon):
    """loss.py:17-32."""
    ratio = np.exp(pi_log_prob_t - b_pi_log_prob_t)
    l1 = ratio * gae_t
    l2 = np.clip(ratio, 1.0 - epsilon, 1.0 + epsilon) * gae_t
    return (-np.minimum(l1, l2)).mean()


def clipped_value_loss(pred_value_t, behavior_value_t, targets_t, epsilon):
    """loss.py:68-78."""
    vclip = behavior_value_t + np.clip(pred_value_t - behavior_value_t, -epsilon, epsilon)
    l1 = np.square(pred_value_t - targets_t)
    l2 = np.square(vclip - targets_t)
    return 0.5 * np.maximum(l1, l2).mean()


def actor_loss_and_dlogits(logits, action, logp_old, adv, clip_eps, ent_coef):
    """_actor_loss_fn (ff_ppo.py:191-213) plus the analytic gradient wrt logits (SURVEY 8a).

    total = ppo_clip_loss - ent_coef * mean(entropy)."""
    m = logits.shape[0]
    lp = log_softmax(logits)
    p = np.exp(lp)
    onehot = np.zeros_like(lp)
    onehot[np.arange(m), np.asarray(action, np.int64)] = 1.0
    logp = (lp * onehot).sum(-1)
    ratio = np.exp(logp - logp_old)
    l1 = ratio * adv
    l2 = np.clip(ratio, 1.0 - clip_eps, 1.0 + clip_eps) * adv
    loss_actor = (-np.minimum(l1, l2)).mean()
    ent_i = -(p * lp).sum(-1)
    entropy = ent_i.mean()
    total = loss_actor - ent_coef * entropy
    # d(-min(l1,l2))/dlogp: branch 1 active when l1 <= l2 (ties inside the clip band carry the
    # same value and the same derivative, JAX splits 1/2+1/2 -> same total).
    in_band = (ratio >= 1.0 - clip_eps) & (ratio <= 1.0 + clip_eps)
    use1 = (l1 < l2) | in_band
    dlogp = np.where(use1, -adv * ratio, 0.0) / m
    dlogits = dlogp[:, None] * (onehot - p)
    # entropy: dH_i/dz_j = -p_j (log p_j + H_i)
    dlogits += (-ent_coef / m) * (-(p * (lp + ent_i[:, None])))
    info = {"actor_loss": loss_actor, "entropy": entropy}
    return total, dlogits, info


def critic_loss_and_dvalue(value, v_old, targets, clip_eps, vf_coef):
    """_critic_loss_fn (ff_ppo.py:215-235) plus the analytic gradient wrt value."""
    m = value.shape[0]
    diff = value - v_old
    vclip = v_old + np.clip(diff, -clip_eps, clip_eps)
    l1 = np.square(value - targets)
    l2 = np.square(vclip - targets)
    value_loss = 0.5 * np.maximum(l1, l2).mean()
    total = vf_coef * value_loss
    inside = np.abs(diff) < clip_eps  # d clip / d value
    g1 = value - targets
    g2 = (vclip - targets) * inside
    dv = np.where(l1 > l2, g1, np.where(l1 < l2, g2, 0.5 * (g1 + g2)))
    dvalue = vf_coef * dv / m
    return total, dvalue, {"value_loss": value_loss}


# --------------------------------------------------------------------------------------------
# A.5  optimiser -- optax.chain(clip_by_global_norm, adam(lr, eps=1e-5))  ff_ppo.py:456-463,264-273
# --------------------------------------------------------------------------------------------


@dataclass
class AdamState:
    mu: np.ndarray
    nu: np.ndarray
    count: int = 0  # ScaleByAdamState.count
    sched_count: int = 0  # ScaleByScheduleState.count


def linear_schedule(init_lr, count, num_updates, epochs, num_minibatches, decay=True):
    """utils/training.py:24-26 (floor division), :48-53 (constant when decay is off)."""
    if not decay:
        return init_lr
    return init_lr * (1.0 - (count // (epochs * num_minibatches)) / num_updates)


def clip_adam_step(flat_p, flat_g, st: AdamState, lr, max_grad_norm, b1=0.9, b2=0.999, eps=1e-5):
    """One optax.chain(clip_by_global_norm(max), adam(lr, eps)) update + apply_updates.
    Operates on the flat vector of ONE network (actor and critic are clipped separately)."""
    dt = flat_p.dtype
    g_norm = np.sqrt((flat_g.astype(dt) ** 2).sum())
    if g_norm >= max_grad_norm:  # optax: trigger = g_norm < max; else (g / g_norm) * max
        flat_g = (flat_g / g_norm) * dt.type(max_grad_norm)
    st.mu = b1 * st.mu + (1.0 - b1) * flat_g
    st.nu = b2 * st.nu + (1.0 - b2) * flat_g * flat_g
    st.count += 1
    mu_hat = st.mu / (1.0 - b1**st.count)
    nu_hat = st.nu / (1.0 - b2**st.count)
    u = mu_hat / (np.sqrt(nu_hat) + eps)  # eps_root = 0
    st.sched_count += 1
    return (flat_p - lr * u).astype(dt), g_norm


# --------------------------------------------------------------------------------------------
# A.6  the update step -- ff_ppo.py:164-340 with actions / permutations injected
# --------------------------------------------------------------------------------------------


@dataclass
class PPOHyper:
    """configs/system/ppo/ff_ppo.yaml:6-22."""

    gamma: float = 0.99
    gae_lambda: float = 0.95
    clip_eps: float = 0.2
    ent_coef: float = 0.01
    vf_coef: float = 0.5
    max_grad_norm: float = 0.5
    actor_lr: float = 3e-4
    critic_lr: float = 3e-4
    epochs: int = 4
    num_minibatches: int = 16
    reward_scale: float = 1.0
    standardize_advantages: bool = True
    decay_learning_rates: bool = True
    num_updates: int = 1


@dataclass
class Trajectory:
    """PPOTransition (systems/ppo/ppo_types.py:9-20), time-major (T, E, ...)."""

    obs: np.ndarray
    action: np.ndarray
    reward: np.ndarray
    done: np.ndarray
    truncated: np.ndarray
    next_obs: np.ndarray  # timestep.extras["next_obs"] (ff_ppo.py:113)
    value: Optional[np.ndarray] = None
    bootstrap_value: Optional[np.ndarray] = None
    log_prob: Optional[np.ndarray] = None


def evaluate_rollout(actor: MLPParams, critic: MLPParams, traj: Trajectory, bf16=False):
    """The network part of _env_step (ff_ppo.py:98-101,113-116) on recorded obs / actions:
    value = critic(obs), log_prob = Categorical(actor(obs)).log_prob(action),
    bootstrap_value = critic(next_obs)."""
    T, E, D = traj.obs.shape
    logits, _ = mlp_forward(actor, traj.obs.reshape(T * E, D), bf16)
    traj.log_prob = categorical_log_prob(logits, traj.action.reshape(-1)).reshape(T, E)
    v, _ = mlp_forward(critic, traj.obs.reshape(T * E, D), bf16)
    traj.value = v[:, 0].reshape(T, E)
    bv, _ = mlp_forward(critic, traj.next_obs.reshape(T * E, D), bf16)
    traj.bootstrap_value = bv[:, 0].reshape(T, E)
    return traj


def ppo_update(
    actor: MLPParams,
    critic: MLPParams,
    a_state: AdamState,
    c_state: AdamState,
    traj: Trajectory,
    perms: np.ndarray,
    h: PPOHyper,
    grad_sync=None,
    bf16: bool = False,
) -> Tuple[MLPParams, MLPParams, Dict[str, np.ndarray], np.ndarray, np.ndarray]:
    """GAE + epochs x minibatches of _update_minibatch (ff_ppo.py:164-340).

    ``perms``: (epochs, T*E) int permutations of the flat index t*E+e (ff_ppo.py:298-307);
    minibatch i of an epoch is perm[i*mb:(i+1)*mb].  ``grad_sync(actor_flat_g, critic_flat_g,
    metrics)`` models the two pmeans (ff_ppo.py:253-261); identity when None."""
    dt = traj.reward.dtype
    T, E, D = traj.obs.shape
    r_t, d_t, trunc = ppo_gae_inputs(traj.reward, traj.done, traj.truncated, h.gamma, h.reward_scale, dt.type)
    adv, targets = gae(
        r_t, d_t, h.gae_lambda, v_tm1=traj.value, v_t=traj.bootstrap_value, truncation_t=trunc,
        time_major=True, standardize_advantages=h.standardize_advantages, dtype=dt.type,
    )
    B = T * E
    mb = B // h.num_minibatches
    flat = lambda x: x.reshape((B,) + x.shape[2:])  # merge_leading_dims, jax_utils.py:29-43
    obs, act, lp_old, v_old = flat(traj.obs), flat(traj.action), flat(traj.log_prob), flat(traj.value)
    adv_f, tgt_f = flat(adv), flat(targets)
    sizes_a = [actor.W[0].shape[0]] + [w.shape[1] for w in actor.W]
    sizes_c = [critic.W[0].shape[0]] + [w.shape[1] for w in critic.W]
    metrics = {k: np.zeros((h.epochs, h.num_minibatches), dt) for k in ("actor_loss", "entropy", "value_loss")}
    for ep in range(h.epochs):
        perm = perms[ep]
        for i in range(h.num_minibatches):
            idx = perm[i * mb : (i + 1) * mb]
            # actor
            logits, a_acts = mlp_forward(actor, obs[idx], bf16)
            _, dlogits, a_info = actor_loss_and_dlogits(logits, act[idx], lp_old[idx], adv_f[idx], h.clip_eps, h.ent_coef)
            a_g = mlp_backward(actor, a_acts, dlogits, bf16).flat()
            # critic (same pre-update params, ff_ppo.py:238-247)
            v, c_acts = mlp_forward(critic, obs[idx], bf16)
            _, dvalue, c_info = critic_loss_and_dvalue(v[:, 0], v_old[idx], tgt_f[idx], h.clip_eps, h.vf_coef)
            c_g = mlp_backward(critic, c_acts, dvalue[:, None], bf16).flat()
            info = {**a_info, **c_info}
            if grad_sync is not None:
                a_g, c_g, info = grad_sync(a_g, c_g, info)
            a_lr = linear_schedule(h.actor_lr, a_state.sched_count, h.num_updates, h.epochs, h.num_minibatches, h.decay_learning_rates)
            c_lr = linear_schedule(h.critic_lr, c_state.sched_count, h.num_updates, h.epochs, h.num_minibatches, h.decay_learning_rates)
            a_new, _ = clip_adam_step(actor.flat(), a_g.astype(dt), a_state, a_lr, h.max_grad_norm)
            c_new, _ = clip_adam_step(critic.flat(), c_g.astype(dt), c_state, c_lr, h.max_grad_norm)
            actor = MLPParams.from_flat(a_new, sizes_a, actor.activation, actor.ln_bias is not None)
            critic = MLPParams.from_flat(c_new, sizes_c, critic.activation, critic.ln_bias is not None)
            for k in metrics:
                metrics[k][ep, i] = info[k]
    return actor, critic, metrics, adv, targets


# --------------------------------------------------------------------------------------------
# shapes -- stoix/utils/total_timestep_checker.py:57-61, 88-96, 104-131
# --------------------------------------------------------------------------------------------


def derive_shapes(total_num_envs, num_devices, update_batch_size, total_timesteps, rollout_length, num_evaluation):
    num_envs = total_num_envs // (num_devices * update_batch_size)
    num_updates = int(total_timesteps) // rollout_length // update_batch_size // num_envs // num_devices
    return num_envs, num_updates, num_updates // num_evaluation
