// Fused PPO losses + analytic output gradients of the fp32 path (one thread per minibatch row), and their value-only faces.
//
// Reference: _actor_loss_fn / _critic_loss_fn (stoix/systems/ppo/anakin/ff_ppo.py:191-235) with ppo_clip_loss
// (stoix/utils/loss.py:17-32), ppo_penalty_loss (:35-47), dpo_loss (:50-65) and clipped_value_loss (:68-78); the tanh-Normal
// head of ff_ppo_continuous.py:191-213 (stoix/networks/distributions.py:56-88).  The reference gets gradients from jax.grad;
// here they are written in closed form (SURVEY.md 8a "Gradient formulas", DESIGN.md section 6):
//   clip         dL/dlogp_i  = -(1/m) A_i ratio_i  [unclipped branch active]
//   KL penalty   total_i = -ratio_i A_i + beta KL_i - ent_coef H_i, KL_i = KL(behaviour_i || pi_i), no ratio clipping
//   DPO          total_i = -(ratio_i A_i - drift_i) - ent_coef H_i, drift = 1[A>=0] relu(x1 - alpha tanh(x1/alpha))
//                + 1[A<0] relu(x2 - beta tanh(x2/beta)), x1 = (ratio - 1) A, x2 = log(ratio) A; d/dlogp = -ratio A
//                + 1[A>=0] 1[y1>0] tanh^2(x1/alpha) A ratio + 1[A<0] 1[y2>0] tanh^2(x2/beta) A  (relu'(0) = 0)
//   Categorical  dlogp/dz_j  = 1[j=a] - p_j ;  dH/dz_j = -p_j (log p_j + H);  dKL/dz_j = p_j - pb_j
//   tanh-Normal  log_prob of the stored action and the seeded entropy estimate (stx_tanh_normal.cuh); the KL is that of the
//                base Normals summed over the dims (the shared affine-tanh bijector cancels)
//   critic       dL/dv_i     = (vf/m) * { (v-tgt)            if (v-tgt)^2 > (vclip-tgt)^2
//                                       { (vclip-tgt)*1[|v-vold|<eps]  otherwise }
// Advantage standardisation (multistep.py:138-139) is applied on load from (mean, rstd).  The behaviour policy of the KL
// penalty is the rollout actor's head output stored per batch row; rows are read through the permutation.
//
// ppo_actor_loss_kernel<Head, Loss> is instantiated for the five (head, loss) pairs the reference has: Categorical x {clip,
// KL penalty} and tanh-Normal x {clip, KL penalty, DPO}.  A term a loss does not have is removed at compile time, so every
// instantiation evaluates exactly the float expressions of its pair.
#pragma once
#include "stx_common.cuh"
#include "stx_loss_rows.cuh"
#include "stx_tanh_normal.cuh"

namespace stx {

constexpr int kMaxActions = 32;  // Categorical logits / tanh-Normal dims per thread
constexpr int kSlotKl = 6;       // metrics slot of kl_divergence (0 actor_loss, 1 entropy, 2 value_loss, 3 advantages, 4 / 5 value, target)

struct ActorLossArgs {
  LossRows r;
  const float* head;       // (mb, A) logits or (mb, 2A) tanh-Normal head outputs
  const float* behaviour;  // KL penalty: (B, head width) behaviour head outputs, row r.src(m)
  const int32_t* action;   // Categorical: (B) stored actions
  StxTanhNormalPpo tn;     // tanh-Normal: (B, A) stored actions, entropy noise and action bounds
  const float* logp_old;
  const float* adv;
  const float* adv_stats;  // nullable
  float* dhead;            // same shape as head
  int A;
  float clip_eps, kl_coef, dpo_alpha, dpo_beta, ent_coef;
};

// ---- heads: load a row, logp(stored action), entropy and (KL) KL(behaviour || pi); then write d head --------------------

// The row's logits (and the behaviour logits) stay in registers.
template <bool KL>
struct CategoricalRow {
  float z[kMaxActions], zb[kMaxActions];
  float lse, lse_b, logp = 0.f, ent = 0.f, kl = 0.f;
  int A, a;

  __device__ __forceinline__ void load(const ActorLossArgs& g, int64_t m, int64_t src) {
    A = g.A;
    float zmax = -INFINITY, bmax = -INFINITY;
#pragma unroll
    for (int j = 0; j < kMaxActions; ++j)
      if (j < A) {
        z[j] = g.head[m * A + j];
        zmax = fmaxf(zmax, z[j]);
        if constexpr (KL) {
          zb[j] = g.behaviour[src * A + j];
          bmax = fmaxf(bmax, zb[j]);
        }
      }
    float se = 0.f, sb = 0.f;
#pragma unroll
    for (int j = 0; j < kMaxActions; ++j)
      if (j < A) {
        se += expf(z[j] - zmax);
        if constexpr (KL) sb += expf(zb[j] - bmax);
      }
    lse = zmax + logf(se);
    if constexpr (KL) lse_b = bmax + logf(sb);
    a = g.action[src];
#pragma unroll
    for (int j = 0; j < kMaxActions; ++j)
      if (j < A) {
        const float lp = z[j] - lse;
        ent -= expf(lp) * lp;
        if constexpr (KL) {
          const float lpb = zb[j] - lse_b;
          kl += expf(lpb) * (lpb - lp);
        }
        if (j == a) logp = lp;
      }
  }

  // d/dz_j [ loss - ent_coef H (+ beta KL) ] / m, given dlogp = d loss / d logp / m, ck = beta / m, ce = ent_coef / m
  __device__ __forceinline__ void backward(const ActorLossArgs& g, int64_t m, float dlogp, float ck, float ce) const {
#pragma unroll
    for (int j = 0; j < kMaxActions; ++j)
      if (j < A) {
        const float lp = z[j] - lse, p = expf(lp);
        if constexpr (KL)
          g.dhead[m * A + j] = dlogp * ((j == a ? 1.f : 0.f) - p) + ck * (p - expf(zb[j] - lse_b)) + ce * p * (lp + ent);
        else  // the fused multiply-add is spelled out: left to the compiler, this kernel's shape fuses the other product
          g.dhead[m * A + j] = __fmaf_rn(dlogp, (j == a ? 1.f : 0.f) - p, ce * p * (lp + ent));
      }
  }
};

// Two passes over the dims, four at a time: the second regenerates the entropy noise of the first (layout in include/stx.h),
// so the entropy draws of every loss on this head match.
template <bool KL>
struct TanhNormalRow {
  HeadGeom geo;
  const float *h, *hb, *act;
  uint64_t call;
  float logp = 0.f, ent = 0.f, kl = 0.f;
  int A;

  __device__ __forceinline__ void load(const ActorLossArgs& g, int64_t m, int64_t src) {
    A = g.A;
    geo = head_geom(g.tn.minimum, g.tn.maximum, kTanhNormalEpsilon);
    h = g.head + m * 2 * A;
    hb = KL ? g.behaviour + src * 2 * A : nullptr;
    act = g.tn.action + src * A;
    call = g.tn.offset + (g.tn.dev_counter ? *g.tn.dev_counter : 0ull);
    for (int j0 = 0; j0 < A; j0 += 4) {
      float e[4];
      entropy_noise(g.tn.eps_in, A, g.tn.seed, m, call, j0, e);
      for (int k = 0; k < 4 && j0 + k < A; ++k) {
        const int j = j0 + k;
        const float loc = h[j], sigma = softplusf(h[A + j]) + g.tn.min_scale;
        logp += tanh_normal_log_prob_given(loc, sigma, act[j], geo).lp;
        ent += tanh_normal_entropy_dim(loc, sigma, e[k], geo);
        if constexpr (KL) kl += normal_kl(hb[j], softplusf(hb[A + j]) + g.tn.min_scale, loc, sigma).kl;
        if (g.tn.eps_out) g.tn.eps_out[m * A + j] = e[k];
      }
    }
  }

  // d/d(loc, raw scale) of the dlogp-weighted log_prob minus ce * H (plus ck * KL); dH/dloc = -2 tanh(u'),
  // dH/dsigma = 1/sigma - 2 tanh(u') eps', dsigma/draw = sigmoid(raw)
  __device__ __forceinline__ void backward(const ActorLossArgs& g, int64_t m, float dlogp, float ck, float ce) const {
    for (int j0 = 0; j0 < A; j0 += 4) {
      float e[4];
      entropy_noise(g.tn.eps_in, A, g.tn.seed, m, call, j0, e);
      for (int k = 0; k < 4 && j0 + k < A; ++k) {
        const int j = j0 + k;
        const float loc = h[j], raw = h[A + j], sigma = softplusf(raw) + g.tn.min_scale;
        const TanhNormalDim t = tanh_normal_log_prob_given(loc, sigma, act[j], geo);
        const float th = tanhf(loc + sigma * e[k]);
        float d_loc = dlogp * t.d_loc + ce * 2.f * th;
        float d_sigma = dlogp * t.d_sigma - ce * (1.f / sigma - 2.f * th * e[k]);
        if constexpr (KL) {
          const NormalKl q = normal_kl(hb[j], softplusf(hb[A + j]) + g.tn.min_scale, loc, sigma);
          d_loc += ck * q.d_mu;
          d_sigma += ck * q.d_sigma;
        }
        g.dhead[m * 2 * A + j] = d_loc;
        g.dhead[m * 2 * A + A + j] = d_sigma * sigmoidf_(raw);
      }
    }
  }
};

// ---- losses: (ratio, log ratio, advantage) -> the row's surrogate and d(surrogate)/d logp / m ------------------------------
// kKl: the loss adds beta KL_i (the kernel adds it, the face takes mean KL).  kExtraSlot: the metrics slot of the third per-row
// metric (the advantage for clip, KL for the penalty; none for DPO).  kFaceParts: partials per block of the value face.
struct LossTerm {
  float loss, dlogp;
};

struct ClipLoss {
  static constexpr bool kKl = false;
  static constexpr int kExtraSlot = 3, kFaceParts = 1;
  float eps;
  __device__ static ClipLoss make(const ActorLossArgs& g) { return {g.clip_eps}; }
  __device__ __forceinline__ LossTerm operator()(float ratio, float /*ld*/, float adv, float inv_m) const {
    const float l1 = ratio * adv;
    const float rc = fminf(fmaxf(ratio, 1.0f - eps), 1.0f + eps);
    const float l2 = rc * adv;
    const bool in_band = (ratio >= 1.0f - eps) && (ratio <= 1.0f + eps);
    return {-fminf(l1, l2), ((l1 < l2) || in_band) ? -adv * ratio * inv_m : 0.f};
  }
};

struct KlPenaltyLoss {
  static constexpr bool kKl = true;
  static constexpr int kExtraSlot = kSlotKl, kFaceParts = 2;
  __device__ static KlPenaltyLoss make(const ActorLossArgs&) { return {}; }
  __device__ __forceinline__ LossTerm operator()(float ratio, float /*ld*/, float adv, float inv_m) const {
    return {-ratio * adv, -adv * ratio * inv_m};
  }
};

struct DpoLoss {
  static constexpr bool kKl = false;
  static constexpr int kExtraSlot = -1, kFaceParts = 2;
  float alpha, beta;
  __device__ static DpoLoss make(const ActorLossArgs& g) { return {g.dpo_alpha, g.dpo_beta}; }
  __device__ __forceinline__ LossTerm operator()(float ratio, float ld, float adv, float inv_m) const {
    const float x1 = (ratio - 1.f) * adv, x2 = ld * adv;
    const float t1 = tanhf(x1 / alpha), t2 = tanhf(x2 / beta);
    const float y1 = x1 - alpha * t1, y2 = x2 - beta * t2;
    const bool pos = adv >= 0.f;
    const float drift = pos ? fmaxf(y1, 0.f) : fmaxf(y2, 0.f);
    // -ratio A + tanh^2(x1/alpha) A ratio = -ratio A sech^2(x1/alpha): written as the product, it keeps its digits where tanh -> 1
    const float sh1 = 1.f / coshf(x1 / alpha);
    float d;
    if (pos)
      d = y1 > 0.f ? -ratio * adv * sh1 * sh1 : -ratio * adv;
    else
      d = y2 > 0.f ? (t2 * t2 - ratio) * adv : -ratio * adv;
    return {-(ratio * adv - drift), d * inv_m};
  }
};

template <template <bool> class Head, class Loss>
__global__ void __launch_bounds__(256) ppo_actor_loss_kernel(ActorLossArgs g) {
  const int64_t m = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  double s_actor = 0.0, s_ent = 0.0, s_extra = 0.0;
  const float inv_m = 1.0f / (float)g.r.mb;
  if (m < g.r.mb) {
    const int64_t src = g.r.src(m);
    Head<Loss::kKl> row;
    row.load(g, m, src);
    float adv = g.adv[src];
    if (g.adv_stats) adv = (adv - g.adv_stats[0]) * g.adv_stats[1];
    const float ld = row.logp - g.logp_old[src];
    const LossTerm t = Loss::make(g)(expf(ld), ld, adv, inv_m);
    if constexpr (Loss::kKl)
      s_actor = (double)(t.loss + g.kl_coef * row.kl);
    else
      s_actor = (double)t.loss;
    s_ent = (double)row.ent;
    s_extra = (double)(Loss::kKl ? row.kl : adv);
    row.backward(g, m, t.dlogp, g.kl_coef * inv_m, g.ent_coef * inv_m);
  }
  if constexpr (Loss::kExtraSlot >= 0)
    reduce_metrics<3>({s_actor, s_ent, s_extra}, {0, 1, Loss::kExtraSlot}, g.r);
  else
    reduce_metrics<2>({s_actor, s_ent}, {0, 1}, g.r);
}

// ---- critic ------------------------------------------------------------------------------------------------------------
struct ValueTerm {
  float loss, dv;  // dv: d loss / d v, with the tie rule below
};
__device__ __forceinline__ ValueTerm clipped_value(float v, float vo, float tg, float eps) {
  const float diff = v - vo;
  const float vclip = vo + fminf(fmaxf(diff, -eps), eps);
  const float e1 = v - tg, e2 = vclip - tg;
  const float q1 = e1 * e1, q2 = e2 * e2;
  const float g2 = (fabsf(diff) < eps) ? e2 : 0.f;
  return {0.5f * fmaxf(q1, q2), q1 > q2 ? e1 : (q1 < q2 ? g2 : 0.5f * (e1 + g2))};
}

// Metrics slots 2 (value_loss), 4 (mean value), 5 (mean target).
__global__ void __launch_bounds__(256) ppo_critic_loss_kernel(LossRows r, const float* value, const float* v_old, const float* tgt, float* dvalue,
                                                              float clip_eps, float vf_coef) {
  const int64_t m = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  double s_vloss = 0.0, s_pred = 0.0, s_tgt = 0.0;
  const float inv_m = 1.0f / (float)r.mb;
  if (m < r.mb) {
    const int64_t src = r.src(m);
    const float v = value[m], tg = tgt[src];
    const ValueTerm t = clipped_value(v, v_old[src], tg, clip_eps);
    s_vloss = (double)t.loss, s_pred = (double)v, s_tgt = (double)tg;
    dvalue[m] = vf_coef * t.dv * inv_m;
  }
  reduce_metrics<3>({s_vloss, s_pred, s_tgt}, {2, 4, 5}, r);
}

// ---- value-only faces of the loss utilities: the mean over n elements, deterministic two-level reduction -----------------
// Face::kParts partials per block; stx_loss_scratch_bytes() holds 2 * kNumSMs of them, so the grid is capped at
// 2 * kNumSMs / kParts blocks.
template <class Loss>
struct SurrogateFace {  // ppo_clip_loss, ppo_penalty_loss (out[0] the loss, out[1] mean KL), dpo_loss
  static constexpr int kParts = Loss::kFaceParts;
  const float *lp, *lp_old, *gae, *kl;
  Loss loss;
  float beta;  // the KL penalty's coefficient
  __device__ __forceinline__ void add(int64_t i, double (&acc)[kParts]) const {
    const float ld = lp[i] - lp_old[i];
    acc[0] += (double)loss(expf(ld), ld, gae[i], 1.f).loss;
    if constexpr (Loss::kKl) acc[1] += (double)kl[i];
  }
  __device__ __forceinline__ void finish(const double (&s)[kParts], int64_t n, float* out) const {
    if constexpr (Loss::kKl) {
      const double mean_kl = s[1] / (double)n;
      out[0] = (float)(s[0] / (double)n + (double)beta * mean_kl);
      out[1] = (float)mean_kl;
    } else {
      out[0] = (float)(s[0] / (double)n);
    }
  }
};

struct ValueFace {  // clipped_value_loss
  static constexpr int kParts = 1;
  const float *v, *v_old, *tgt;
  float eps;
  __device__ __forceinline__ void add(int64_t i, double (&acc)[kParts]) const { acc[0] += (double)clipped_value(v[i], v_old[i], tgt[i], eps).loss; }
  __device__ __forceinline__ void finish(const double (&s)[kParts], int64_t n, float* out) const { out[0] = (float)(s[0] / (double)n); }
};

template <class Face>
__global__ void __launch_bounds__(256) loss_face_kernel(Face f, int64_t n, double* __restrict__ partials, unsigned int* counter, float* __restrict__ out) {
  constexpr int P = Face::kParts;
  __shared__ double sm[32];
  double acc[P] = {};
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += stride) f.add(i, acc);
  double b[P];
#pragma unroll
  for (int k = 0; k < P; ++k) b[k] = block_sum<double>(acc[k], sm);
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = 0; k < P; ++k) partials[P * blockIdx.x + k] = b[k];
  }
  if (last_block_ticket(counter, gridDim.x)) {
    double s[P] = {};
    for (unsigned int i = threadIdx.x; i < gridDim.x; i += blockDim.x) {
#pragma unroll
      for (int k = 0; k < P; ++k) s[k] += partials[P * i + k];
    }
#pragma unroll
    for (int k = 0; k < P; ++k) s[k] = block_sum<double>(s[k], sm);
    if (threadIdx.x == 0) f.finish(s, n, out);
  }
}

}  // namespace stx
