// The PPO variants (fp32): KL-penalty PPO on the Categorical and tanh-Normal heads, and DPO on the tanh-Normal head.
//
// Reference: stoix/utils/loss.py:35-47 (ppo_penalty_loss), :50-65 (dpo_loss); their use in
// stoix/systems/ppo/anakin/ff_ppo_penalty.py:137,150-178, ff_ppo_penalty_continuous.py:137,150-179 and
// ff_dpo_continuous.py:148-170.  Each variant changes only the actor loss of ff_ppo's _update_minibatch, so each is one
// per-row kernel between the fp32 actor forward and backward (stx_mlp.cu), followed by the critic half the clip path runs.
// The gradients are written in closed form (DESIGN.md section 6):
//   KL penalty   total_i = -ratio_i A_i + beta KL_i - ent_coef H_i, KL_i = KL(behaviour_i || pi_i), no ratio clipping;
//                Categorical d/dz_j = -(1/m) A ratio (1[j=a] - p_j) + (beta/m)(p_j - pb_j) + (ent_coef/m) p_j (log p_j + H);
//                tanh-Normal: the KL of the base Normals summed over the dims (the shared affine-tanh bijector cancels).
//   DPO          total_i = -(ratio_i A_i - drift_i) - ent_coef H_i, drift = 1[A>=0] relu(x1 - alpha tanh(x1/alpha))
//                + 1[A<0] relu(x2 - beta tanh(x2/beta)), x1 = (ratio - 1) A, x2 = log(ratio) A; d/dlogp = -ratio A
//                + 1[A>=0] 1[y1>0] tanh^2(x1/alpha) A ratio + 1[A<0] 1[y2>0] tanh^2(x2/beta) A  (relu'(0) = 0).
// The behaviour policy is the rollout actor's head output stored per (t, e) row; rows are read through the permutation.
#include "stx_common.cuh"
#include "stx_ppo_halves.cuh"
#include "stx_tanh_normal.cuh"

namespace stx {
namespace {

constexpr int kMaxVariantActions = 32;  // Categorical logits / tanh-Normal dims per thread, as on the clip path
constexpr int kSlotKl = 6;              // metrics slot of kl_divergence (0 actor_loss, 1 entropy, 2 value_loss as on the clip path)

struct CatPenaltyArgs {
  const float* logits;     // (mb, A)
  const float* behaviour;  // (B, A) behaviour logits, row idx[m]
  const int32_t* idx;      // perm + mb_off (nullable -> row0 + m)
  int64_t row0;
  const int32_t* action;
  const float* logp_old;
  const float* adv;
  const float* adv_stats;  // nullable
  float* dlogits;          // (mb, A)
  int64_t mb;
  int A;
  float kl_coef, ent_coef;
  double* partials;        // [grid][6]
  unsigned int* counter;
  float* metrics;          // slots 0, 1, kSlotKl accumulated with weight
  float weight;
};

// Deterministic metric reduction of the clip-path loss kernels: per-block partials, then the last block sums them in block
// order.  Partial column k feeds metrics[slot[k]].
template <int N>
__device__ __forceinline__ void reduce_metrics(const double (&v)[N], const int (&slot)[N], double* partials, unsigned int* counter,
                                               float* metrics, float weight, int64_t mb) {
  __shared__ double sm[32];
#pragma unroll
  for (int k = 0; k < N; ++k) {
    const double r = block_sum<double>(v[k], sm);
    if (threadIdx.x == 0) partials[(int64_t)blockIdx.x * 6 + k] = r;
  }
  if (last_block_ticket(counter, gridDim.x)) {
#pragma unroll
    for (int k = 0; k < N; ++k) {
      double s = 0.0;
      for (unsigned int i = threadIdx.x; i < gridDim.x; i += blockDim.x) s += partials[(int64_t)i * 6 + k];
      s = block_sum<double>(s, sm);
      if (threadIdx.x == 0) metrics[slot[k]] += weight * (float)(s / (double)mb);
    }
  }
}

// One thread per minibatch row: Categorical KL-penalty PPO (ff_ppo_penalty.py:150-178).  The row's logits and its
// behaviour logits stay in registers.
__global__ void __launch_bounds__(256) ppo_penalty_categorical_kernel(CatPenaltyArgs g) {
  const int64_t m = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  double s_actor = 0.0, s_ent = 0.0, s_kl = 0.0;
  const float inv_m = 1.0f / (float)g.mb;
  if (m < g.mb) {
    const int64_t src = g.idx ? (int64_t)g.idx[m] : g.row0 + m;
    const int A = g.A;
    float z[kMaxVariantActions], zb[kMaxVariantActions];
    float zmax = -INFINITY, bmax = -INFINITY;
#pragma unroll
    for (int j = 0; j < kMaxVariantActions; ++j)
      if (j < A) {
        z[j] = g.logits[m * A + j];
        zb[j] = g.behaviour[src * A + j];
        zmax = fmaxf(zmax, z[j]);
        bmax = fmaxf(bmax, zb[j]);
      }
    float se = 0.f, sb = 0.f;
#pragma unroll
    for (int j = 0; j < kMaxVariantActions; ++j)
      if (j < A) {
        se += expf(z[j] - zmax);
        sb += expf(zb[j] - bmax);
      }
    const float lse = zmax + logf(se), lse_b = bmax + logf(sb);
    const int a = g.action[src];
    float adv = g.adv[src];
    if (g.adv_stats) adv = (adv - g.adv_stats[0]) * g.adv_stats[1];
    float ent = 0.f, kl = 0.f, logp_a = 0.f;
#pragma unroll
    for (int j = 0; j < kMaxVariantActions; ++j)
      if (j < A) {
        const float lp = z[j] - lse, lpb = zb[j] - lse_b;
        ent -= expf(lp) * lp;
        kl += expf(lpb) * (lpb - lp);
        if (j == a) logp_a = lp;
      }
    const float ratio = expf(logp_a - g.logp_old[src]);
    s_actor = (double)(-ratio * adv + g.kl_coef * kl);
    s_ent = (double)ent;
    s_kl = (double)kl;
    const float dlogp = -adv * ratio * inv_m, ck = g.kl_coef * inv_m, ce = g.ent_coef * inv_m;
#pragma unroll
    for (int j = 0; j < kMaxVariantActions; ++j)
      if (j < A) {
        const float lp = z[j] - lse, p = expf(lp), pb = expf(zb[j] - lse_b);
        g.dlogits[m * A + j] = dlogp * ((j == a ? 1.f : 0.f) - p) + ck * (p - pb) + ce * p * (lp + ent);
      }
  }
  reduce_metrics<3>({s_actor, s_ent, s_kl}, {0, 1, kSlotKl}, g.partials, g.counter, g.metrics, g.weight, g.mb);
}

struct TnVariantArgs {
  const float* head;       // (mb, 2A)
  const float* behaviour;  // (B, 2A) behaviour head outputs, row idx[m] (KL penalty only)
  const int32_t* idx;      // perm + mb_off (nullable -> row0 + m)
  int64_t row0;
  StxTanhNormalPpo hd;
  const float* logp_old;
  const float* adv;
  const float* adv_stats;  // nullable
  float* dhead;            // (mb, 2A)
  int64_t mb;
  int A;
  float kl_coef, dpo_alpha, dpo_beta, ent_coef;
  double* partials;        // [grid][6]
  unsigned int* counter;
  float* metrics;          // slots 0, 1 (and kSlotKl for the KL penalty) accumulated with weight
  float weight;
};

// KL(N(mb, sb) || N(mu, s)) of one dimension and its derivatives with respect to the second distribution's mu and s.  The value
// is tfp's arrangement, 0.5 (dm / s)^2 + 0.5 expm1(2 d) - d with d = log sb - log s: no cancellation near KL = 0, where the
// penalty starts every update, and exactly 0 for equal distributions.
struct NormalKl {
  float kl, d_mu, d_sigma;
};
__device__ __forceinline__ NormalKl normal_kl(float mu_b, float sigma_b, float mu, float sigma) {
  const float dm = mu_b - mu, q = sigma_b * sigma_b + dm * dm, inv = 1.f / sigma, dls = logf(sigma_b) - logf(sigma), z = dm * inv;
  NormalKl r;
  r.kl = 0.5f * z * z + 0.5f * expm1f(2.f * dls) - dls;
  r.d_mu = -dm * inv * inv;
  r.d_sigma = inv - q * inv * inv * inv;
  return r;
}

// One thread per minibatch row: the tanh-Normal actor loss of the variant.  Log-prob of the stored action and the entropy
// noise as in ppo_tanh_normal_loss_kernel (stx_ppo_continuous.cu), so the entropy draws match ff_ppo_continuous exactly.
template <int KIND>
__global__ void __launch_bounds__(256) ppo_variant_tanh_normal_kernel(TnVariantArgs g) {
  const int64_t m = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  double s_actor = 0.0, s_ent = 0.0, s_kl = 0.0;
  const float inv_m = 1.0f / (float)g.mb;
  if (m < g.mb) {
    const int64_t src = g.idx ? (int64_t)g.idx[m] : g.row0 + m;
    const int A = g.A;
    const HeadGeom geo = head_geom(g.hd.minimum, g.hd.maximum, kTanhNormalEpsilon);
    const float* h = g.head + m * 2 * A;
    const float* hb = KIND == STX_PPO_KL_PENALTY ? g.behaviour + src * 2 * A : nullptr;
    const float* act = g.hd.action + src * A;
    const uint64_t call = g.hd.offset + (g.hd.dev_counter ? *g.hd.dev_counter : 0ull);
    float logp = 0.f, ent = 0.f, kl = 0.f;
    for (int j0 = 0; j0 < A; j0 += 4) {
      float e[4];
      entropy_noise(g.hd.eps_in, A, g.hd.seed, m, call, j0, e);
      for (int k = 0; k < 4 && j0 + k < A; ++k) {
        const int j = j0 + k;
        const float loc = h[j], sigma = softplusf(h[A + j]) + g.hd.min_scale;
        logp += tanh_normal_log_prob_given(loc, sigma, act[j], geo).lp;
        ent += tanh_normal_entropy_dim(loc, sigma, e[k], geo);
        if (KIND == STX_PPO_KL_PENALTY) kl += normal_kl(hb[j], softplusf(hb[A + j]) + g.hd.min_scale, loc, sigma).kl;
        if (g.hd.eps_out) g.hd.eps_out[m * A + j] = e[k];
      }
    }
    float adv = g.adv[src];
    if (g.adv_stats) adv = (adv - g.adv_stats[0]) * g.adv_stats[1];
    const float ld = logp - g.logp_old[src];
    const float ratio = expf(ld);
    float dlogp;  // d(per-row actor loss)/d logp, divided by m
    if (KIND == STX_PPO_KL_PENALTY) {
      s_actor = (double)(-ratio * adv + g.kl_coef * kl);
      s_kl = (double)kl;
      dlogp = -adv * ratio * inv_m;
    } else {
      const float x1 = (ratio - 1.f) * adv, x2 = ld * adv;
      const float t1 = tanhf(x1 / g.dpo_alpha), t2 = tanhf(x2 / g.dpo_beta);
      const float y1 = x1 - g.dpo_alpha * t1, y2 = x2 - g.dpo_beta * t2;
      const bool pos = adv >= 0.f;
      const float drift = pos ? fmaxf(y1, 0.f) : fmaxf(y2, 0.f);
      s_actor = (double)(-(ratio * adv - drift));
      // -ratio A + tanh^2(x1/alpha) A ratio = -ratio A sech^2(x1/alpha): written as the product, it keeps its digits where tanh -> 1
      const float sh1 = 1.f / coshf(x1 / g.dpo_alpha);
      float d;
      if (pos)
        d = y1 > 0.f ? -ratio * adv * sh1 * sh1 : -ratio * adv;
      else
        d = y2 > 0.f ? (t2 * t2 - ratio) * adv : -ratio * adv;
      dlogp = d * inv_m;
    }
    s_ent = (double)ent;
    const float ck = g.kl_coef * inv_m, ce = g.ent_coef * inv_m;
    for (int j0 = 0; j0 < A; j0 += 4) {
      float e[4];
      entropy_noise(g.hd.eps_in, A, g.hd.seed, m, call, j0, e);
      for (int k = 0; k < 4 && j0 + k < A; ++k) {
        const int j = j0 + k;
        const float loc = h[j], raw = h[A + j], sigma = softplusf(raw) + g.hd.min_scale;
        const TanhNormalDim t = tanh_normal_log_prob_given(loc, sigma, act[j], geo);
        const float th = tanhf(loc + sigma * e[k]);
        float d_loc = dlogp * t.d_loc + ce * 2.f * th;
        float d_sigma = dlogp * t.d_sigma - ce * (1.f / sigma - 2.f * th * e[k]);
        if (KIND == STX_PPO_KL_PENALTY) {
          const NormalKl q = normal_kl(hb[j], softplusf(hb[A + j]) + g.hd.min_scale, loc, sigma);
          d_loc += ck * q.d_mu;
          d_sigma += ck * q.d_sigma;
        }
        g.dhead[m * 2 * A + j] = d_loc;
        g.dhead[m * 2 * A + A + j] = d_sigma * sigmoidf_(raw);
      }
    }
  }
  if (KIND == STX_PPO_KL_PENALTY)
    reduce_metrics<3>({s_actor, s_ent, s_kl}, {0, 1, kSlotKl}, g.partials, g.counter, g.metrics, g.weight, g.mb);
  else
    reduce_metrics<2>({s_actor, s_ent}, {0, 1}, g.partials, g.counter, g.metrics, g.weight, g.mb);
}

// Per-row KL(p || q): Categorical logit pairs (TANH = false) or tanh-Normal head pairs summed over the A dims (TANH = true).
template <bool TANH>
__global__ void row_kl_kernel(const float* __restrict__ p, const float* __restrict__ q, int64_t M, int A, float min_scale, float* __restrict__ kl) {
  const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (r >= M) return;
  float s = 0.f;
  if (TANH) {
    const float *hp = p + r * 2 * A, *hq = q + r * 2 * A;
    for (int j = 0; j < A; ++j)
      s += normal_kl(hp[j], softplusf(hp[A + j]) + min_scale, hq[j], softplusf(hq[A + j]) + min_scale).kl;
  } else {
    const float *zp = p + r * A, *zq = q + r * A;
    float pm = -INFINITY, qm = -INFINITY;
    for (int j = 0; j < A; ++j) pm = fmaxf(pm, zp[j]), qm = fmaxf(qm, zq[j]);
    float ps = 0.f, qs = 0.f;
    for (int j = 0; j < A; ++j) ps += expf(zp[j] - pm), qs += expf(zq[j] - qm);
    const float lp0 = pm + logf(ps), lq0 = qm + logf(qs);
    for (int j = 0; j < A; ++j) {
      const float lp = zp[j] - lp0;
      s += expf(lp) * (lp - (zq[j] - lq0));
    }
  }
  kl[r] = s;
}

// Value-only faces of the two losses (stx_loss_api.cu's reduction): out[0] = the actor loss, out[1] = mean KL (penalty only).
//   KIND 0 (ppo_penalty_loss): -mean(ratio A) + beta mean(kl);  KIND 1 (dpo_loss): -mean(ratio A - drift).
template <int KIND>
__global__ void __launch_bounds__(256) variant_loss_value_kernel(const float* __restrict__ lp, const float* __restrict__ lp_old,
                                                                 const float* __restrict__ gae, const float* __restrict__ kl, int64_t n,
                                                                 float c0, float c1, double* __restrict__ partials, unsigned int* counter,
                                                                 float* __restrict__ out) {
  __shared__ double sm[32];
  double acc = 0.0, acc_kl = 0.0;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += stride) {
    const float ld = lp[i] - lp_old[i], ratio = expf(ld), a = gae[i];
    if (KIND == 0) {
      acc += (double)(-ratio * a);
      acc_kl += (double)kl[i];
    } else {
      const float x1 = (ratio - 1.f) * a, x2 = ld * a;
      const float drift = a >= 0.f ? fmaxf(x1 - c0 * tanhf(x1 / c0), 0.f) : fmaxf(x2 - c1 * tanhf(x2 / c1), 0.f);
      acc += (double)(-(ratio * a - drift));
    }
  }
  const double b0 = block_sum<double>(acc, sm), b1 = block_sum<double>(acc_kl, sm);
  if (threadIdx.x == 0) partials[2 * blockIdx.x] = b0, partials[2 * blockIdx.x + 1] = b1;
  if (last_block_ticket(counter, gridDim.x)) {
    double s0 = 0.0, s1 = 0.0;
    for (unsigned int i = threadIdx.x; i < gridDim.x; i += blockDim.x) s0 += partials[2 * i], s1 += partials[2 * i + 1];
    s0 = block_sum<double>(s0, sm);
    s1 = block_sum<double>(s1, sm);
    if (threadIdx.x == 0) {
      const double mean_kl = s1 / (double)n;
      out[0] = (float)(s0 / (double)n + (KIND == 0 ? (double)c0 * mean_kl : 0.0));
      if (KIND == 0) out[1] = (float)mean_kl;
    }
  }
}

bool head_ok(const StxTanhNormalPpo* hd) { return hd && hd->action && hd->maximum > hd->minimum && hd->min_scale >= 0.f; }

int check_variant(const StxPpoVariant* v, bool categorical, const char* who) {
  STX_REQUIRE(v, STX_E_ARG, "%s: null variant", who);
  STX_REQUIRE(v->kind == STX_PPO_KL_PENALTY || (!categorical && v->kind == STX_PPO_DPO), STX_E_UNSUPPORTED,
              "%s: variant kind %d (the %s head has %s)", who, v->kind, categorical ? "Categorical" : "tanh-Normal",
              categorical ? "STX_PPO_KL_PENALTY only" : "STX_PPO_KL_PENALTY and STX_PPO_DPO");
  STX_REQUIRE(v->kind != STX_PPO_KL_PENALTY || v->behaviour, STX_E_ARG, "%s: the KL penalty needs the behaviour head outputs", who);
  STX_REQUIRE(v->kind != STX_PPO_DPO || (v->dpo_alpha > 0.f && v->dpo_beta > 0.f), STX_E_ARG, "%s: DPO needs alpha > 0 and beta > 0", who);
  return STX_OK;
}

int launch_cat(const CatPenaltyArgs& g, cudaStream_t st) {
  ppo_penalty_categorical_kernel<<<(unsigned)((g.mb + 255) / 256), 256, 0, st>>>(g);
  STX_LAUNCH_OK();
  return STX_OK;
}

int launch_tn(int kind, const TnVariantArgs& g, cudaStream_t st) {
  const unsigned grid = (unsigned)((g.mb + 255) / 256);
  if (kind == STX_PPO_KL_PENALTY)
    ppo_variant_tanh_normal_kernel<STX_PPO_KL_PENALTY><<<grid, 256, 0, st>>>(g);
  else
    ppo_variant_tanh_normal_kernel<STX_PPO_DPO><<<grid, 256, 0, st>>>(g);
  STX_LAUNCH_OK();
  return STX_OK;
}

int check_minibatch(const StxMlp* actor, const StxMlp* critic, const StxPpoBatch* b, int64_t mb_off, int64_t mb, const StxPpoHyper* h,
                    float* grad_arena, float* metrics, int precision, void* workspace, size_t workspace_bytes, const char* who) {
  STX_REQUIRE(precision == STX_PREC_F32, STX_E_UNSUPPORTED,
              "%s: precision=%d; the KL-penalty and DPO losses have only the fp32 path (STX_PREC_F32)", who, precision);
  if (int rc = simt_check_mlp(actor, who)) return rc;
  if (int rc = simt_check_mlp(critic, who)) return rc;
  STX_REQUIRE(b && h && grad_arena && metrics && workspace, STX_E_ARG, "%s: null pointer", who);
  STX_REQUIRE(b->obs && b->log_prob && b->value && b->advantages && b->targets, STX_E_ARG, "%s: null batch field", who);
  STX_REQUIRE(mb > 0 && mb_off >= 0 && mb_off + mb <= b->B, STX_E_SHAPE, "%s: minibatch [%lld,%lld) outside batch %lld", who, (long long)mb_off,
              (long long)(mb_off + mb), (long long)b->B);
  STX_REQUIRE(actor->sizes[0] == critic->sizes[0], STX_E_SHAPE, "%s: actor/critic input dims differ", who);
  STX_REQUIRE(critic->sizes[critic->n_layers] == 1, STX_E_SHAPE, "%s: critic head must be scalar", who);
  STX_REQUIRE(!h->standardize_advantages || b->adv_stats, STX_E_ARG, "%s: standardize_advantages needs adv_stats", who);
  STX_REQUIRE(workspace_bytes >= stx_ppo_workspace_bytes(actor, critic, mb, STX_PREC_F32), STX_E_WORKSPACE, "%s: workspace %zu < %zu", who,
              workspace_bytes, stx_ppo_workspace_bytes(actor, critic, mb, STX_PREC_F32));
  return STX_OK;
}

}  // namespace
}  // namespace stx

using namespace stx;

extern "C" int stx_categorical_kl(const float* logits_p, const float* logits_q, int64_t M, int A, float* kl, void* stream) {
  STX_REQUIRE(logits_p && logits_q && kl && M > 0 && A > 0, STX_E_ARG, "stx_categorical_kl: bad arguments");
  row_kl_kernel<false><<<(unsigned)((M + 127) / 128), 128, 0, (cudaStream_t)stream>>>(logits_p, logits_q, M, A, 0.f, kl);
  STX_LAUNCH_OK();
  return STX_OK;
}

extern "C" int stx_tanh_normal_kl(const float* head_p, const float* head_q, int64_t M, int A, float min_scale, float* kl, void* stream) {
  STX_REQUIRE(head_p && head_q && kl && M > 0 && A > 0 && min_scale >= 0.f, STX_E_ARG, "stx_tanh_normal_kl: bad arguments");
  row_kl_kernel<true><<<(unsigned)((M + 127) / 128), 128, 0, (cudaStream_t)stream>>>(head_p, head_q, M, A, min_scale, kl);
  STX_LAUNCH_OK();
  return STX_OK;
}

extern "C" int stx_ppo_penalty_loss(const float* pi_log_prob_t, const float* b_pi_log_prob_t, const float* gae_t, const float* kl, int64_t n,
                                    float beta, float* out, void* scratch, void* stream) {
  STX_REQUIRE(pi_log_prob_t && b_pi_log_prob_t && gae_t && kl && out && scratch && n > 0, STX_E_ARG, "stx_ppo_penalty_loss: bad arguments");
  const int64_t blocks = (n + 255) / 256 < kNumSMs ? (n + 255) / 256 : kNumSMs;  // two partials per block in stx_loss_scratch_bytes()
  variant_loss_value_kernel<0><<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(
      pi_log_prob_t, b_pi_log_prob_t, gae_t, kl, n, beta, 0.f, reinterpret_cast<double*>(reinterpret_cast<char*>(scratch) + 16),
      reinterpret_cast<unsigned int*>(scratch), out);
  STX_LAUNCH_OK();
  return STX_OK;
}

extern "C" int stx_dpo_loss(const float* pi_log_prob_t, const float* b_pi_log_prob_t, const float* gae_t, int64_t n, float alpha, float beta,
                            float* out, void* scratch, void* stream) {
  STX_REQUIRE(pi_log_prob_t && b_pi_log_prob_t && gae_t && out && scratch && n > 0 && alpha > 0.f && beta > 0.f, STX_E_ARG,
              "stx_dpo_loss: bad arguments");
  const int64_t blocks = (n + 255) / 256 < kNumSMs ? (n + 255) / 256 : kNumSMs;
  variant_loss_value_kernel<1><<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(
      pi_log_prob_t, b_pi_log_prob_t, gae_t, nullptr, n, alpha, beta, reinterpret_cast<double*>(reinterpret_cast<char*>(scratch) + 16),
      reinterpret_cast<unsigned int*>(scratch), out);
  STX_LAUNCH_OK();
  return STX_OK;
}

extern "C" int stx_ppo_penalty_head_grads(const float* logits, const int32_t* idx, int64_t row0, const StxPpoVariant* v, const int32_t* action,
                                          const float* logp_old, const float* adv, const float* adv_stats, int64_t mb, int A, float ent_coef,
                                          float* d_logits, float* metrics, float weight, void* scratch, void* stream) {
  if (int rc = check_variant(v, true, "stx_ppo_penalty_head_grads")) return rc;
  STX_REQUIRE(logits && action && logp_old && adv && d_logits && metrics && scratch && mb > 0, STX_E_ARG,
              "stx_ppo_penalty_head_grads: null pointer or empty minibatch");
  STX_REQUIRE(A > 0 && A <= kMaxVariantActions, STX_E_SHAPE, "stx_ppo_penalty_head_grads: A=%d (max %d)", A, kMaxVariantActions);
  CatPenaltyArgs g{};
  g.logits = logits, g.behaviour = v->behaviour, g.idx = idx, g.row0 = row0, g.action = action, g.logp_old = logp_old, g.adv = adv;
  g.adv_stats = adv_stats, g.dlogits = d_logits, g.mb = mb, g.A = A, g.kl_coef = v->kl_coef, g.ent_coef = ent_coef;
  g.counter = reinterpret_cast<unsigned int*>(scratch);  // the layout of stx_ppo_head_scratch_bytes
  g.partials = reinterpret_cast<double*>(reinterpret_cast<char*>(scratch) + 256);
  g.metrics = metrics, g.weight = weight;
  return launch_cat(g, (cudaStream_t)stream);
}

extern "C" int stx_ppo_variant_tanh_normal_head_grads(const float* head_out, const int32_t* idx, int64_t row0, const StxTanhNormalPpo* head,
                                                      const StxPpoVariant* v, const float* logp_old, const float* adv, const float* adv_stats,
                                                      int64_t mb, int A, float ent_coef, float* d_head_out, float* metrics, float weight,
                                                      void* scratch, void* stream) {
  if (int rc = check_variant(v, false, "stx_ppo_variant_tanh_normal_head_grads")) return rc;
  STX_REQUIRE(head_out && head_ok(head) && logp_old && adv && d_head_out && metrics && scratch && mb > 0, STX_E_ARG,
              "stx_ppo_variant_tanh_normal_head_grads: null pointer, empty minibatch or bad action bounds");
  STX_REQUIRE(A > 0 && A <= kMaxVariantActions, STX_E_SHAPE, "stx_ppo_variant_tanh_normal_head_grads: A=%d (max %d)", A, kMaxVariantActions);
  TnVariantArgs g{};
  g.head = head_out, g.behaviour = v->behaviour, g.idx = idx, g.row0 = row0, g.hd = *head, g.logp_old = logp_old, g.adv = adv;
  g.adv_stats = adv_stats, g.dhead = d_head_out, g.mb = mb, g.A = A;
  g.kl_coef = v->kl_coef, g.dpo_alpha = v->dpo_alpha, g.dpo_beta = v->dpo_beta, g.ent_coef = ent_coef;
  g.counter = reinterpret_cast<unsigned int*>(scratch);
  g.partials = reinterpret_cast<double*>(reinterpret_cast<char*>(scratch) + 256);
  g.metrics = metrics, g.weight = weight;
  return launch_tn(v->kind, g, (cudaStream_t)stream);
}

extern "C" int stx_ppo_penalty_minibatch_grads(const StxMlp* actor, const StxMlp* critic, const StxPpoBatch* b, const StxPpoVariant* v,
                                               int64_t mb_off, int64_t mb, const StxPpoHyper* h, float grad_weight, float* grad_arena,
                                               float* metrics, int precision, void* workspace, size_t workspace_bytes, void* stream) {
  const char* who = "stx_ppo_penalty_minibatch_grads";
  if (int rc = check_minibatch(actor, critic, b, mb_off, mb, h, grad_arena, metrics, precision, workspace, workspace_bytes, who)) return rc;
  if (int rc = check_variant(v, true, who)) return rc;
  STX_REQUIRE(b->action, STX_E_ARG, "%s: null batch action", who);
  const int A = actor->sizes[actor->n_layers];
  STX_REQUIRE(A <= kMaxVariantActions, STX_E_SHAPE, "%s: action_dim %d > %d", who, A, kMaxVariantActions);
  cudaStream_t st = (cudaStream_t)stream;
  int64_t aoff, coff, total;
  stx_ppo_arena_offsets(actor, critic, &aoff, &coff, &total);
  const int D = actor->sizes[0];
  const float* obs = reinterpret_cast<const float*>(b->obs);
  const int32_t* idx = b->perm ? b->perm + mb_off : nullptr;
  const float* x = idx ? obs : obs + mb_off * (int64_t)D;  // without a permutation: the contiguous row range from mb_off

  // ---- actor: forward, loss, backward (ff_ppo_penalty.py:149-178, 200-204) ----
  SimtHeadBufs hb{};
  if (int rc = simt_net_forward(actor, x, D, idx, mb, workspace, &hb, st)) return rc;
  CatPenaltyArgs g{};
  g.logits = hb.head, g.behaviour = v->behaviour, g.idx = idx, g.row0 = mb_off, g.action = b->action, g.logp_old = b->log_prob;
  g.adv = b->advantages, g.adv_stats = h->standardize_advantages ? b->adv_stats : nullptr, g.dlogits = hb.dhead, g.mb = mb, g.A = A;
  g.kl_coef = v->kl_coef, g.ent_coef = h->ent_coef, g.partials = hb.loss_partials, g.counter = hb.counter;
  g.metrics = metrics, g.weight = grad_weight;
  if (int rc = launch_cat(g, st)) return rc;
  if (int rc = simt_net_backward(actor, x, D, idx, mb, workspace, grad_weight, grad_arena + aoff, h->overwrite_grads, st)) return rc;
  // ---- critic: the clip path's own half (ff_ppo_penalty.py:180-198, 206-210) ----
  return simt_ppo_critic_grads(critic, b, mb_off, mb, h, grad_weight, grad_arena + coff, metrics, workspace, st);
}

extern "C" int stx_ppo_variant_continuous_minibatch_grads(const StxMlp* actor, const StxMlp* critic, const StxPpoBatch* b,
                                                          const StxTanhNormalPpo* head, const StxPpoVariant* v, int64_t mb_off, int64_t mb,
                                                          const StxPpoHyper* h, float grad_weight, float* grad_arena, float* metrics,
                                                          int precision, void* workspace, size_t workspace_bytes, void* stream) {
  const char* who = "stx_ppo_variant_continuous_minibatch_grads";
  if (int rc = check_minibatch(actor, critic, b, mb_off, mb, h, grad_arena, metrics, precision, workspace, workspace_bytes, who)) return rc;
  if (int rc = check_variant(v, false, who)) return rc;
  STX_REQUIRE(head_ok(head), STX_E_ARG, "%s: null head / action or bad action bounds", who);
  const int head_w = actor->sizes[actor->n_layers], A = head_w / 2;
  STX_REQUIRE(head_w % 2 == 0 && A <= kMaxVariantActions, STX_E_SHAPE, "%s: actor head width %d is not 2A with A <= %d", who, head_w,
              kMaxVariantActions);
  cudaStream_t st = (cudaStream_t)stream;
  int64_t aoff, coff, total;
  stx_ppo_arena_offsets(actor, critic, &aoff, &coff, &total);
  const int D = actor->sizes[0];
  const float* obs = reinterpret_cast<const float*>(b->obs);
  const int32_t* idx = b->perm ? b->perm + mb_off : nullptr;
  const float* x = idx ? obs : obs + mb_off * (int64_t)D;

  // ---- actor: forward, loss, backward (ff_ppo_penalty_continuous.py:149-179, ff_dpo_continuous.py:148-170) ----
  SimtHeadBufs hb{};
  if (int rc = simt_net_forward(actor, x, D, idx, mb, workspace, &hb, st)) return rc;
  TnVariantArgs g{};
  g.head = hb.head, g.behaviour = v->behaviour, g.idx = idx, g.row0 = mb_off, g.hd = *head, g.logp_old = b->log_prob, g.adv = b->advantages;
  g.adv_stats = h->standardize_advantages ? b->adv_stats : nullptr, g.dhead = hb.dhead, g.mb = mb, g.A = A;
  g.kl_coef = v->kl_coef, g.dpo_alpha = v->dpo_alpha, g.dpo_beta = v->dpo_beta, g.ent_coef = h->ent_coef;
  g.partials = hb.loss_partials, g.counter = hb.counter, g.metrics = metrics, g.weight = grad_weight;
  if (int rc = launch_tn(v->kind, g, st)) return rc;
  if (int rc = simt_net_backward(actor, x, D, idx, mb, workspace, grad_weight, grad_arena + aoff, h->overwrite_grads, st)) return rc;
  // ---- critic: the clip path's own half ----
  return simt_ppo_critic_grads(critic, b, mb_off, mb, h, grad_weight, grad_arena + coff, metrics, workspace, st);
}
