"""fp64 restatement of ff_mpo and ff_mpo_continuous (stoix/systems/mpo/*.py, stoix/utils/multistep.py) for the tests.

Rules restated here, and where they come from:
  - categorical_mpo_loss (discrete_loss.py:20-147), differentiated as jax.grad does: q is a constant, the temperature reaches the
    loss through the temperature loss AND through the E-step weights of the cross-entropy (the reference stops no gradient there),
    alpha is a constant in the KL penalty and the KL a constant in the alpha loss.  The KL and the entropies of a Categorical are
    tfp's closed forms (upstream knowledge: tfp Categorical.kl_divergence / entropy / cross_entropy).
  - mpo_loss (continuous_loss.py:152-303), the decoupled tanh-Normal loss: a literal fp64 torch transcription, differentiated by
    autograd with the reference's stop-gradients (the weights, and each alpha in its KL penalty); the log-probability is that of
    events inside the clip band (distributions.py:56-80), and the Normal KL tfp's closed form (upstream knowledge).
  - one optimiser step: optax chain(clip_by_global_norm, adam(eps=1e-5)) per segment (upstream knowledge), the -18 clamp of the duals
    and optax.incremental_update of the targets.
  - batch_general_off_policy_returns_from_q_and_v and batch_retrace_continuous (multistep.py:210-311), time-major here.
  - the sequence buffer.  flashbax is not installed here; its rules as fbx.make_trajectory_buffer applies them with add_batch_size
    = E, period = 1, min_length_time_axis = sample_sequence_length = S, max_length_time_axis = L (ff_mpo.py:539-546) are upstream
    knowledge, the same rules tests/rainbow_oracle.py states for the prioritised variant:
      * time-major ring, one write index for all envs (flashbax trajectory_buffer: `current_index`);
      * a sequence (env e, start row p) is sampleable only if its S rows are written and do not straddle the write head;
      * sampling is uniform: env uniform over E, start uniform over the sampleable starts.
    This project fixes how a draw maps to a start: the k-th sampleable start counted from the oldest written row, (w - c + k) mod L.
"""
from __future__ import annotations

import numpy as np


def softplus(x):
    return np.logaddexp(0.0, x)


def sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def log_softmax(z):
    m = z.max(-1, keepdims=True)
    return z - (m + np.log(np.exp(z - m).sum(-1, keepdims=True)))


METRICS = ("temperature", "alpha", "loss_temperature", "loss_alpha", "loss_policy", "loss_kl", "kl_nonparametric", "entropy_online",
           "entropy_target", "kl_mean_rel", "kl_q_rel", "q_min", "q_max")


def categorical_loss(zo, zt, q, duals, epsilon, epsilon_policy):
    """zo / zt (M, A) online / target logits, q (A, M) target Q of every action, duals [log_temperature, log_alpha].
    Returns (d_head (M, A), dual_grad (2), metrics dict)."""
    zo, zt, q = (np.asarray(x, np.float64) for x in (zo, zt, q))
    M, A = zo.shape
    qb = q.T                                              # [B, D]
    lt, la = float(duals[0]), float(duals[1])
    eta, alpha = softplus(lt) + 1e-8, softplus(la) + 1e-8
    lpo, lpt = log_softmax(zo), log_softmax(zt)
    po, pt = np.exp(lpo), np.exp(lpt)
    u = qb / eta + lpt
    lse = np.log(np.exp(u - u.max(-1, keepdims=True)).sum(-1)) + u.max(-1)
    w = np.exp(u - lse[:, None])
    ce = -(w * lpo).sum(-1)
    kl = (pt * (lpt - lpo)).sum(-1)
    mean_kl = kl.mean()
    wq = (w * qb).sum(-1)
    d_head = ((po - w) + alpha * (po - pt)) / M
    g_eta = epsilon + lse.mean() - wq.mean() / eta + (w * (qb - wq[:, None]) * lpo).sum(-1).mean() / eta ** 2
    dual_grad = np.array([g_eta * sigmoid(lt), (epsilon_policy - mean_kl) * sigmoid(la)])
    klnp = (w * (np.log(w) - lpt)).sum(-1)
    metrics = {
        "temperature": eta, "alpha": alpha, "loss_temperature": eta * (epsilon + lse.mean()), "loss_alpha": alpha * (epsilon_policy - mean_kl),
        "loss_policy": ce.mean(), "loss_kl": alpha * mean_kl, "kl_nonparametric": klnp.mean(), "entropy_online": -(po * lpo).sum(-1).mean(),
        "entropy_target": -(pt * lpt).sum(-1).mean(), "kl_mean_rel": mean_kl / epsilon_policy, "kl_q_rel": klnp.mean() / epsilon,
        "q_min": qb.min(0).mean(), "q_max": qb.max(0).mean(),
    }
    return d_head, dual_grad, metrics


def retrace(q_t, v_t, r_t, d_t, log_rho, lam):
    """Time-major targets (K, E): g_{K-1} = r + d v, g_k = r_k + d_k (v_k - c_k q_k + c_k g_{k+1}), c = lam min(1, exp(log_rho))."""
    v_t, r_t, d_t = (np.asarray(x, np.float64) for x in (v_t, r_t, d_t))
    K = v_t.shape[0]
    c = lam * np.minimum(1.0, np.exp(np.asarray(log_rho, np.float64)))
    q_t = np.asarray(q_t, np.float64)
    g = np.zeros_like(v_t)
    g[K - 1] = r_t[K - 1] + d_t[K - 1] * v_t[K - 1]
    for k in range(K - 2, -1, -1):
        g[k] = r_t[k] + d_t[k] * (v_t[k] - c[k] * q_t[k] + c[k] * g[k + 1])
    return g


def gae_targets(r, d, lam, v):
    """batch_truncated_generalized_advantage_estimation's value targets, time-major: r, d (K, E), v (K + 1, E)."""
    K = r.shape[0]
    adv = np.zeros_like(r, dtype=np.float64)
    acc = 0.0
    for k in range(K - 1, -1, -1):
        delta = r[k] + d[k] * v[k + 1] - v[k]
        acc = delta + d[k] * lam * acc
        adv[k] = acc
    return adv + v[:K]


def n_step_targets(r, d, v, n):
    """batch_n_step_bootstrapped_returns with lambda 1, time-major (multistep.py:148-207)."""
    T = r.shape[0]
    out = np.zeros_like(r, dtype=np.float64)
    for t in range(T):
        s_end = min(t + n, T)
        g = v[min(t + n - 1, T - 1)]
        for s in range(s_end - 1, t - 1, -1):
            g = r[s] + d[s] * g
        out[t] = g
    return out


def q_grad(q, targets):
    """dq (S, B) of mean 0.5 (q[:S-1] - targets)^2 and the loss."""
    S, B = q.shape
    td = q[: S - 1].astype(np.float64) - targets
    dq = np.zeros((S, B))
    dq[: S - 1] = td / ((S - 1) * B)
    return dq, 0.5 * (td ** 2).mean()


class SequenceRing:
    """The trajectory buffer's rules (module docstring) on L time rows of E envs."""

    def __init__(self, L: int, E: int, D: int):
        self.L, self.E, self.w, self.c = L, E, 0, 0
        self.obs = np.zeros((L, E, D), np.float32)
        self.action = np.zeros((L, E), np.int32)
        self.reward = np.zeros((L, E), np.float32)
        self.done = np.zeros((L, E), np.uint8)
        self.log_prob = np.zeros((L, E), np.float32)

    def add(self, obs, action, reward, done, log_prob):
        T = reward.shape[0]
        for t in range(max(0, T - self.L), T):
            p = (self.w + t) % self.L
            self.obs[p], self.action[p], self.reward[p], self.done[p], self.log_prob[p] = obs[t], action[t], reward[t], done[t], log_prob[t]
        self.w, self.c = (self.w + T) % self.L, min(self.c + T, self.L)

    def valid_starts(self, S: int):
        """Every start row whose S rows are written and do not straddle the write head, oldest first."""
        return [(self.w - self.c + k) % self.L for k in range(self.c - S + 1)]

    def sample(self, S: int, idx):
        """idx (B, 2) = (env, k): sequence b is env idx[b, 0] from the idx[b, 1]-th valid start; time-major (S, B, ...) outputs."""
        starts = self.valid_starts(S)
        rows = [[((starts[k] + t) % self.L, e) for (e, k) in idx] for t in range(S)]
        pick = lambda a: np.stack([np.stack([a[p, e] for (p, e) in row]) for row in rows])
        return pick(self.obs), pick(self.action), pick(self.reward), pick(self.done), pick(self.log_prob), [(e, starts[k]) for (e, k) in idx]


CONTINUOUS_METRICS = ("temperature", "alpha_mean", "alpha_stddev", "loss_temperature", "loss_alpha_mean", "loss_alpha_stddev", "loss_policy_mean",
                      "loss_policy_stddev", "loss_kl_mean", "loss_kl_stddev", "kl_mean", "kl_stddev", "kl_nonparametric")


def _tanh_normal_log_prob(loc, scale, a, lo, hi):
    """log-probability of events strictly inside the clip band of AffineTanhTransformedDistribution (distributions.py:56-80): the Normal
    log-density of u = atanh((a - shift) / s) minus the log-det-Jacobian of a = shift + s tanh(u)."""
    import torch
    s, sh = (hi - lo) / 2.0, (hi + lo) / 2.0
    u = torch.atanh((a - sh) / s)
    z = (u - loc) / scale
    return -0.5 * z * z - torch.log(scale) - 0.5 * np.log(2 * np.pi) - (2.0 * (np.log(2.0) - u - torch.nn.functional.softplus(-2.0 * u))) - np.log(s)


def continuous_loss(h, ht, q, acts, duals, epsilon, epsilon_mean, epsilon_stddev, per_dim, lo, hi, min_scale=1e-3):
    """mpo_loss (continuous_loss.py:152-303) in fp64, differentiated by torch autograd with the reference's stop-gradients: h / ht (M, 2A)
    online / target loc | raw scale, q (N, M), acts (N, M, A) target draws (inside the clip band), duals [lt, la_mean (C), la_stddev (C)].
    Returns (d_head (M, 2A), dual_grad, metrics dict)."""
    import torch
    t = lambda x: torch.as_tensor(np.asarray(x), dtype=torch.float64)
    h, duals = t(h).requires_grad_(True), t(duals).requires_grad_(True)
    ht, q, acts = t(ht), t(q), t(acts)
    M, A = h.shape[0], h.shape[1] // 2
    C = A if per_dim else 1
    sp = torch.nn.functional.softplus
    temperature = sp(duals[0]) + 1e-8
    alpha_mean, alpha_stddev = sp(duals[1: 1 + C]) + 1e-8, sp(duals[1 + C: 1 + 2 * C]) + 1e-8
    loc, scale = h[:, :A], sp(h[:, A:]) + min_scale
    loc_t, scale_t = ht[:, :A], sp(ht[:, A:]) + min_scale
    tempered = q / temperature
    w = torch.softmax(tempered, 0).detach()
    lse = torch.logsumexp(tempered, 0)
    loss_temperature = temperature * (epsilon + lse.mean() - np.log(q.shape[0]))
    klnp = (w * torch.log(q.shape[0] * w + 1e-8)).sum(0)
    lp_m = _tanh_normal_log_prob(loc[None], scale_t[None], acts, lo, hi).sum(-1)          # fixed stddev
    lp_s = _tanh_normal_log_prob(loc_t[None], scale[None], acts, lo, hi).sum(-1)          # fixed mean
    loss_policy_mean = (-(lp_m * w).sum(0)).mean()
    loss_policy_stddev = (-(lp_s * w).sum(0)).mean()
    kl = lambda mb, sb, m, s_: torch.log(s_ / sb) + (sb ** 2 + (mb - m) ** 2) / (2 * s_ ** 2) - 0.5
    kl_mean, kl_stddev = kl(loc_t, scale_t, loc, scale_t), kl(loc_t, scale_t, loc_t, scale)
    if not per_dim:
        kl_mean, kl_stddev = kl_mean.sum(-1), kl_stddev.sum(-1)
    mkm, mks = kl_mean.mean(0), kl_stddev.mean(0)
    loss_kl_mean, loss_alpha_mean = (alpha_mean.detach() * mkm).sum(), (alpha_mean * (epsilon_mean - mkm.detach())).sum()
    loss_kl_stddev, loss_alpha_stddev = (alpha_stddev.detach() * mks).sum(), (alpha_stddev * (epsilon_stddev - mks.detach())).sum()
    loss = loss_policy_mean + loss_policy_stddev + loss_kl_mean + loss_kl_stddev + loss_alpha_mean + loss_alpha_stddev + loss_temperature
    loss.backward()
    f = lambda x: float(x.detach().mean())
    metrics = {"temperature": f(temperature), "alpha_mean": f(alpha_mean), "alpha_stddev": f(alpha_stddev), "loss_temperature": f(loss_temperature),
               "loss_alpha_mean": f(loss_alpha_mean), "loss_alpha_stddev": f(loss_alpha_stddev), "loss_policy_mean": f(loss_policy_mean),
               "loss_policy_stddev": f(loss_policy_stddev), "loss_kl_mean": f(loss_kl_mean), "loss_kl_stddev": f(loss_kl_stddev),
               "kl_mean": f(kl_mean), "kl_stddev": f(kl_stddev), "kl_nonparametric": f(klnp)}
    return h.grad.numpy(), duals.grad.numpy(), metrics


def adam_clamp_polyak(params, grads, mu, nu, count, segments, lrs, max_norms, tau, target, dual_slice, b1=0.9, b2=0.999, eps=1e-5):
    """One optimiser step of the learner in fp64: per segment chain(clip_by_global_norm, adam(eps=1e-5)) (optax rules, upstream
    knowledge), then the duals clamped at -18, then target = tau online + (1 - tau) target over [actor | Q]."""
    p, mu, nu = params.astype(np.float64).copy(), mu.astype(np.float64).copy(), nu.astype(np.float64).copy()
    for (off, n), lr, mx in zip(segments, lrs, max_norms):
        g = grads[off: off + n].astype(np.float64)
        norm = np.sqrt((g * g).sum())
        g = g * (mx / norm) if norm > mx else g
        mu[off: off + n] = b1 * mu[off: off + n] + (1 - b1) * g
        nu[off: off + n] = b2 * nu[off: off + n] + (1 - b2) * g * g
        mh, nh = mu[off: off + n] / (1 - b1 ** count), nu[off: off + n] / (1 - b2 ** count)
        p[off: off + n] -= lr * mh / (np.sqrt(nh) + eps)
    p[dual_slice] = np.maximum(p[dual_slice], -18.0)
    new_target = tau * p[: target.size] + (1 - tau) * target.astype(np.float64)
    return p, new_target
