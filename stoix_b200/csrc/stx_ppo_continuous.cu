// Continuous-action PPO (fp32): the tanh-Normal head under the PPO losses.
//
// Reference: stoix/systems/ppo/anakin/ff_ppo_continuous.py:98-101 (rollout: sample, then log_prob of the sampled action),
// :191-213, 239-247 (_actor_loss_fn: log_prob of the STORED action under the new parameters, ppo_clip_loss, the seeded entropy
// estimate `entropy(seed=key)`, jax.grad), stoix/networks/distributions.py:56-88 (log_prob, entropy).  The gradients are
// written in closed form (DESIGN.md section 6); the critic half and both networks' forward / backward are the fp32 PPO path's
// own (stx_mlp.cu).  Counter layout of the entropy noise: include/stx.h.
#include "stx_common.cuh"
#include "stx_ppo_halves.cuh"
#include "stx_tanh_normal.cuh"

namespace stx {
namespace {

constexpr int kMaxTanhNormalDims = 32;

// Rollout / face: log_prob of given actions, one thread per row.
__global__ void tanh_normal_log_prob_kernel(const float* __restrict__ head, int64_t M, int A, const float* __restrict__ action, int64_t ld_action,
                                            float minimum, float maximum, float min_scale, float* __restrict__ log_prob) {
  const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (r >= M) return;
  const HeadGeom g = head_geom(minimum, maximum, kTanhNormalEpsilon);
  float lp = 0.f;
  for (int j = 0; j < A; ++j) {
    const float loc = head[r * 2 * A + j], sigma = softplusf(head[r * 2 * A + A + j]) + min_scale;
    lp += tanh_normal_log_prob_given(loc, sigma, action[r * ld_action + j], g).lp;
  }
  log_prob[r] = lp;
}

struct TnLossArgs {
  const float* head;      // (mb, 2A)
  const int32_t* idx;     // perm + mb_off (nullable -> row0 + m)
  int64_t row0;
  StxTanhNormalPpo hd;
  const float* logp_old;
  const float* adv;
  const float* adv_stats; // nullable
  float* dhead;           // (mb, 2A)
  int64_t mb;
  int A;
  float clip_eps, ent_coef;
  double* partials;       // [grid][6]
  unsigned int* counter;
  float* metrics;         // slots 0 (actor_loss), 1 (entropy), 3 (advantages) accumulated with weight
  float weight;
};

// Face of the estimate (AffineTanhNormal.entropy(seed)): one thread per row, noise keyed by the row index.
__global__ void tanh_normal_entropy_kernel(const float* __restrict__ head, int64_t M, int A, const float* __restrict__ eps_in, uint64_t seed,
                                           uint64_t offset, const uint64_t* __restrict__ dev_counter, float minimum, float maximum,
                                           float min_scale, float* __restrict__ entropy, float* __restrict__ eps_out) {
  const int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (r >= M) return;
  const HeadGeom g = head_geom(minimum, maximum, kTanhNormalEpsilon);
  const uint64_t call = offset + (dev_counter ? *dev_counter : 0ull);
  float h = 0.f;
  for (int j0 = 0; j0 < A; j0 += 4) {
    float e[4];
    entropy_noise(eps_in, A, seed, r, call, j0, e);
    for (int k = 0; k < 4 && j0 + k < A; ++k) {
      const int j = j0 + k;
      h += tanh_normal_entropy_dim(head[r * 2 * A + j], softplusf(head[r * 2 * A + A + j]) + min_scale, e[k], g);
      if (eps_out) eps_out[r * A + j] = e[k];
    }
  }
  entropy[r] = h;
}

// One thread per minibatch row: log_prob of the stored action, the clipped surrogate (the branch / tie rules of
// ppo_loss_grad_kernel), the entropy estimate, and d(total actor loss)/d(head_out) for all 2A columns.
__global__ void __launch_bounds__(256) ppo_tanh_normal_loss_kernel(TnLossArgs g) {
  const int64_t m = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  float s_actor = 0.f, s_ent = 0.f, s_adv = 0.f;
  const float inv_m = 1.0f / (float)g.mb;
  if (m < g.mb) {
    const int64_t src = g.idx ? (int64_t)g.idx[m] : g.row0 + m;
    const int A = g.A;
    const HeadGeom geo = head_geom(g.hd.minimum, g.hd.maximum, kTanhNormalEpsilon);
    const float* h = g.head + m * 2 * A;
    const float* act = g.hd.action + src * A;
    const uint64_t call = g.hd.offset + (g.hd.dev_counter ? *g.hd.dev_counter : 0ull);
    float logp = 0.f, ent = 0.f;
    for (int j0 = 0; j0 < A; j0 += 4) {
      float e[4];
      entropy_noise(g.hd.eps_in, A, g.hd.seed, m, call, j0, e);
      for (int k = 0; k < 4 && j0 + k < A; ++k) {
        const int j = j0 + k;
        const float loc = h[j], sigma = softplusf(h[A + j]) + g.hd.min_scale;
        logp += tanh_normal_log_prob_given(loc, sigma, act[j], geo).lp;
        ent += tanh_normal_entropy_dim(loc, sigma, e[k], geo);
        if (g.hd.eps_out) g.hd.eps_out[m * A + j] = e[k];
      }
    }
    float adv = g.adv[src];
    if (g.adv_stats) adv = (adv - g.adv_stats[0]) * g.adv_stats[1];
    const float ratio = expf(logp - g.logp_old[src]);
    const float l1 = ratio * adv;
    const float rc = fminf(fmaxf(ratio, 1.0f - g.clip_eps), 1.0f + g.clip_eps);
    const float l2 = rc * adv;
    s_actor = -fminf(l1, l2);
    s_ent = ent;
    s_adv = adv;
    const bool in_band = (ratio >= 1.0f - g.clip_eps) && (ratio <= 1.0f + g.clip_eps);
    const float dlogp = ((l1 < l2) || in_band) ? -adv * ratio * inv_m : 0.f;
    const float ce = g.ent_coef * inv_m;
    for (int j0 = 0; j0 < A; j0 += 4) {
      float e[4];
      entropy_noise(g.hd.eps_in, A, g.hd.seed, m, call, j0, e);
      for (int k = 0; k < 4 && j0 + k < A; ++k) {
        const int j = j0 + k;
        const float loc = h[j], raw = h[A + j], sigma = softplusf(raw) + g.hd.min_scale;
        const TanhNormalDim t = tanh_normal_log_prob_given(loc, sigma, act[j], geo);
        const float th = tanhf(loc + sigma * e[k]);
        // d/d[.] of dlogp-weighted log_prob minus ent_coef/m * H  (dH/dloc = -2 tanh(u'), dH/dsigma = 1/sigma - 2 tanh(u') eps')
        const float d_loc = dlogp * t.d_loc + ce * 2.f * th;
        const float d_sigma = dlogp * t.d_sigma - ce * (1.f / sigma - 2.f * th * e[k]);
        g.dhead[m * 2 * A + j] = d_loc;
        g.dhead[m * 2 * A + A + j] = d_sigma * sigmoidf_(raw);
      }
    }
  }
  __shared__ double sm[32];
  constexpr int kSlots[3] = {0, 1, 3};
  const double red[3] = {(double)s_actor, (double)s_ent, (double)s_adv};
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const double r = block_sum<double>(red[k], sm);
    if (threadIdx.x == 0) g.partials[(int64_t)blockIdx.x * 6 + kSlots[k]] = r;
  }
  if (last_block_ticket(g.counter, gridDim.x)) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      double s = 0.0;
      for (unsigned int i = threadIdx.x; i < gridDim.x; i += blockDim.x) s += g.partials[(int64_t)i * 6 + kSlots[k]];
      s = block_sum<double>(s, sm);
      if (threadIdx.x == 0) g.metrics[kSlots[k]] += g.weight * (float)(s / (double)g.mb);
    }
  }
}

int launch_loss(const TnLossArgs& g, cudaStream_t st) {
  ppo_tanh_normal_loss_kernel<<<(unsigned)((g.mb + 255) / 256), 256, 0, st>>>(g);
  STX_LAUNCH_OK();
  return STX_OK;
}

bool head_ok(const StxTanhNormalPpo* hd) { return hd && hd->action && hd->maximum > hd->minimum && hd->min_scale >= 0.f; }

}  // namespace
}  // namespace stx

using namespace stx;

extern "C" int stx_tanh_normal_log_prob(const float* head_out, int64_t M, int A, const float* action, int64_t ld_action, float minimum,
                                        float maximum, float min_scale, float* log_prob, void* stream) {
  STX_REQUIRE(head_out && action && log_prob && M > 0 && A > 0 && ld_action >= A && maximum > minimum, STX_E_ARG,
              "stx_tanh_normal_log_prob: bad arguments");
  tanh_normal_log_prob_kernel<<<(unsigned)((M + 127) / 128), 128, 0, (cudaStream_t)stream>>>(head_out, M, A, action, ld_action, minimum, maximum,
                                                                                            min_scale, log_prob);
  STX_LAUNCH_OK();
  return STX_OK;
}

extern "C" int stx_tanh_normal_entropy(const float* head_out, int64_t M, int A, const float* eps_in, uint64_t seed, uint64_t offset,
                                       const uint64_t* dev_counter, float minimum, float maximum, float min_scale, float* entropy, float* eps_out,
                                       void* stream) {
  STX_REQUIRE(head_out && entropy && M > 0 && A > 0 && maximum > minimum, STX_E_ARG, "stx_tanh_normal_entropy: bad arguments");
  tanh_normal_entropy_kernel<<<(unsigned)((M + 127) / 128), 128, 0, (cudaStream_t)stream>>>(head_out, M, A, eps_in, seed, offset, dev_counter, minimum,
                                                                                           maximum, min_scale, entropy, eps_out);
  STX_LAUNCH_OK();
  return STX_OK;
}

extern "C" int stx_ppo_tanh_normal_head_grads(const float* head_out, const int32_t* idx, int64_t row0, const StxTanhNormalPpo* head,
                                              const float* logp_old, const float* adv, const float* adv_stats, int64_t mb, int A, float clip_eps,
                                              float ent_coef, float* d_head_out, float* metrics, float weight, void* scratch, void* stream) {
  STX_REQUIRE(head_out && head_ok(head) && logp_old && adv && d_head_out && metrics && scratch && mb > 0, STX_E_ARG,
              "stx_ppo_tanh_normal_head_grads: null pointer, empty minibatch or bad action bounds");
  STX_REQUIRE(A > 0 && A <= kMaxTanhNormalDims, STX_E_SHAPE, "stx_ppo_tanh_normal_head_grads: A=%d (max %d)", A, kMaxTanhNormalDims);
  TnLossArgs g{};
  g.head = head_out, g.idx = idx, g.row0 = row0, g.hd = *head, g.logp_old = logp_old, g.adv = adv, g.adv_stats = adv_stats;
  g.dhead = d_head_out, g.mb = mb, g.A = A, g.clip_eps = clip_eps, g.ent_coef = ent_coef;
  g.counter = reinterpret_cast<unsigned int*>(scratch);  // the layout of stx_ppo_head_scratch_bytes
  g.partials = reinterpret_cast<double*>(reinterpret_cast<char*>(scratch) + 256);
  g.metrics = metrics, g.weight = weight;
  return launch_loss(g, (cudaStream_t)stream);
}

extern "C" int stx_ppo_continuous_minibatch_grads(const StxMlp* actor, const StxMlp* critic, const StxPpoBatch* b, const StxTanhNormalPpo* head,
                                                  int64_t mb_off, int64_t mb, const StxPpoHyper* h, float grad_weight, float* grad_arena,
                                                  float* metrics, int precision, void* workspace, size_t workspace_bytes, void* stream) {
  STX_REQUIRE(precision == STX_PREC_F32, STX_E_UNSUPPORTED,
              "stx_ppo_continuous_minibatch_grads: precision=%d; the tanh-Normal head has only the fp32 path (STX_PREC_F32)", precision);
  if (int rc = simt_check_mlp(actor, "stx_ppo_continuous_minibatch_grads(actor)")) return rc;
  if (int rc = simt_check_mlp(critic, "stx_ppo_continuous_minibatch_grads(critic)")) return rc;
  STX_REQUIRE(b && h && grad_arena && metrics && workspace, STX_E_ARG, "stx_ppo_continuous_minibatch_grads: null pointer");
  STX_REQUIRE(head_ok(head), STX_E_ARG, "stx_ppo_continuous_minibatch_grads: null head / action or bad action bounds");
  STX_REQUIRE(b->obs && b->log_prob && b->value && b->advantages && b->targets, STX_E_ARG, "stx_ppo_continuous_minibatch_grads: null batch field");
  STX_REQUIRE(mb > 0 && mb_off >= 0 && mb_off + mb <= b->B, STX_E_SHAPE, "stx_ppo_continuous_minibatch_grads: minibatch [%lld,%lld) outside batch %lld",
              (long long)mb_off, (long long)(mb_off + mb), (long long)b->B);
  STX_REQUIRE(actor->sizes[0] == critic->sizes[0], STX_E_SHAPE, "actor/critic input dims differ");
  STX_REQUIRE(critic->sizes[critic->n_layers] == 1, STX_E_SHAPE, "critic head must be scalar");
  const int head_w = actor->sizes[actor->n_layers], A = head_w / 2;
  STX_REQUIRE(head_w % 2 == 0 && A <= kMaxTanhNormalDims, STX_E_SHAPE,
              "stx_ppo_continuous_minibatch_grads: actor head width %d is not 2A with A <= %d", head_w, kMaxTanhNormalDims);
  STX_REQUIRE(!h->standardize_advantages || b->adv_stats, STX_E_ARG, "standardize_advantages needs adv_stats");
  STX_REQUIRE(workspace_bytes >= stx_ppo_workspace_bytes(actor, critic, mb, STX_PREC_F32), STX_E_WORKSPACE,
              "stx_ppo_continuous_minibatch_grads: workspace %zu < %zu", workspace_bytes, stx_ppo_workspace_bytes(actor, critic, mb, STX_PREC_F32));
  cudaStream_t st = (cudaStream_t)stream;
  int64_t aoff, coff, total;
  stx_ppo_arena_offsets(actor, critic, &aoff, &coff, &total);
  const int D = actor->sizes[0];
  const float* obs = reinterpret_cast<const float*>(b->obs);
  const int32_t* idx = b->perm ? b->perm + mb_off : nullptr;
  const float* x = idx ? obs : obs + mb_off * (int64_t)D;  // without a permutation: the contiguous row range from mb_off

  // ---- actor: forward, loss, backward (ff_ppo_continuous.py:191-213, 239-242) ----
  SimtHeadBufs hb{};
  if (int rc = simt_net_forward(actor, x, D, idx, mb, workspace, &hb, st)) return rc;
  TnLossArgs g{};
  g.head = hb.head, g.idx = idx, g.row0 = mb_off, g.hd = *head, g.logp_old = b->log_prob, g.adv = b->advantages;
  g.adv_stats = h->standardize_advantages ? b->adv_stats : nullptr, g.dhead = hb.dhead, g.mb = mb, g.A = A;
  g.clip_eps = h->clip_eps, g.ent_coef = h->ent_coef, g.partials = hb.loss_partials, g.counter = hb.counter;
  g.metrics = metrics, g.weight = grad_weight;
  if (int rc = launch_loss(g, st)) return rc;
  if (int rc = simt_net_backward(actor, x, D, idx, mb, workspace, grad_weight, grad_arena + aoff, h->overwrite_grads, st)) return rc;
  // ---- critic: the discrete fp32 path's own half (ff_ppo_continuous.py:215-235, 244-247) ----
  return simt_ppo_critic_grads(critic, b, mb_off, mb, h, grad_weight, grad_arena + coff, metrics, workspace, st);
}
