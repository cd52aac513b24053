// The PPO losses of the fp32 path: the minibatch entries (actor forward, actor loss, actor backward, then the critic half),
// the loss heads on precomputed network outputs, the value-only and KL faces, and the tanh-Normal rollout faces.  The bf16
// minibatch (stx_tc_ppo.cu) shares only the validation here.  Kernels: stx_ppo_loss.cuh; networks: stx_mlp.cu.  PQN's Q loss
// (stx_q_loss_grads) and the DQN family's one-step Q losses (stx_q_td_loss_grads) live here too: they reuse the rows and the metric
// reduction of these losses.
//
// Reference: the _update_minibatch of stoix/systems/ppo/anakin/ff_ppo.py:184-247, ff_ppo_continuous.py:184-247,
// ff_ppo_penalty.py:149-210, ff_ppo_penalty_continuous.py:149-210 and ff_dpo_continuous.py:148-170: each changes only the
// actor loss, so each is one per-row kernel between the fp32 actor forward and backward, followed by the same critic half.
#include "stx_common.cuh"
#include "stx_ppo_halves.cuh"
#include "stx_ppo_loss.cuh"
#include "stx_tanh_normal.cuh"

namespace stx {

// implemented in stx_tc_mlp.cu
int tc_ppo_minibatch_grads(const StxMlp* actor, const StxMlp* critic, const StxPpoBatch* batch, int64_t mb_off, int64_t mb,
                           const StxPpoHyper* hyper, float grad_weight, float* grad_arena, float* metrics, void* ws, size_t ws_bytes,
                           cudaStream_t st);

namespace {

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
  } else {  // no register arrays: A is not bounded here
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

template <class Face>
int launch_face(const Face& f, int64_t n, float* out, void* scratch, void* stream) {
  const int64_t cap = 2 / Face::kParts * kNumSMs, need = (n + 255) / 256;  // the partials of stx_loss_scratch_bytes()
  loss_face_kernel<Face><<<(unsigned)(need < cap ? need : cap), 256, 0, (cudaStream_t)stream>>>(
      f, n, reinterpret_cast<double*>(reinterpret_cast<char*>(scratch) + 16), reinterpret_cast<unsigned int*>(scratch), out);
  STX_LAUNCH_OK();
  return STX_OK;
}

using ActorLossLaunch = int (*)(const ActorLossArgs&, cudaStream_t);

template <template <bool> class Head, class Loss>
int launch_actor_loss(const ActorLossArgs& g, cudaStream_t st) {
  ppo_actor_loss_kernel<Head, Loss><<<(unsigned)((g.r.mb + 255) / 256), 256, 0, st>>>(g);
  STX_LAUNCH_OK();
  return STX_OK;
}

ActorLossLaunch tanh_normal_variant(int kind) {
  return kind == STX_PPO_KL_PENALTY ? launch_actor_loss<TanhNormalRow, KlPenaltyLoss> : launch_actor_loss<TanhNormalRow, DpoLoss>;
}

int launch_critic_loss(const LossRows& r, const float* value, const float* v_old, const float* tgt, float* dvalue, float clip_eps,
                       float vf_coef, cudaStream_t st) {
  ppo_critic_loss_kernel<<<(unsigned)((r.mb + 255) / 256), 256, 0, st>>>(r, value, v_old, tgt, dvalue, clip_eps, vf_coef);
  STX_LAUNCH_OK();
  return STX_OK;
}

// The rows of a head-grad entry: `scratch` has the layout of stx_ppo_head_scratch_bytes (counter, partials from byte 256).
LossRows scratch_rows(const int32_t* idx, int64_t row0, int64_t mb, float* metrics, float weight, void* scratch) {
  return {idx, row0, mb, reinterpret_cast<double*>(reinterpret_cast<char*>(scratch) + 256), reinterpret_cast<unsigned int*>(scratch), metrics,
          weight};
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

// The checks every PPO minibatch entry shares; `precision` sizes the workspace.  fp32_only (nullable) names what refuses any
// other precision.
int check_minibatch(const StxMlp* actor, const StxMlp* critic, const StxPpoBatch* b, int64_t mb_off, int64_t mb, const StxPpoHyper* h,
                    const float* grad_arena, const float* metrics, int precision, const char* fp32_only, const void* workspace,
                    size_t workspace_bytes, const char* who) {
  STX_REQUIRE(!fp32_only || precision == STX_PREC_F32, STX_E_UNSUPPORTED, "%s: precision=%d; %s only the fp32 path (STX_PREC_F32)", who,
              precision, fp32_only);
  char net[96];
  snprintf(net, sizeof net, "%s(actor)", who);
  if (int rc = simt_check_mlp(actor, net)) return rc;
  snprintf(net, sizeof net, "%s(critic)", who);
  if (int rc = simt_check_mlp(critic, net)) return rc;
  STX_REQUIRE(b && h && grad_arena && metrics && workspace, STX_E_ARG, "%s: null pointer", who);
  STX_REQUIRE(b->obs && b->log_prob && b->value && b->advantages && b->targets, STX_E_ARG, "%s: null batch field", who);
  STX_REQUIRE(mb > 0 && mb_off >= 0 && mb_off + mb <= b->B, STX_E_SHAPE, "%s: minibatch [%lld,%lld) outside batch %lld", who, (long long)mb_off,
              (long long)(mb_off + mb), (long long)b->B);
  STX_REQUIRE(actor->sizes[0] == critic->sizes[0], STX_E_SHAPE, "%s: actor/critic input dims differ", who);
  STX_REQUIRE(critic->sizes[critic->n_layers] == 1, STX_E_SHAPE, "%s: critic head must be scalar", who);
  STX_REQUIRE(!h->standardize_advantages || b->adv_stats, STX_E_ARG, "%s: standardize_advantages needs adv_stats", who);
  const size_t need = stx_ppo_workspace_bytes(actor, critic, mb, precision);
  STX_REQUIRE(workspace_bytes >= need, STX_E_WORKSPACE, "%s: workspace %zu < %zu", who, workspace_bytes, need);
  return STX_OK;
}

// A of the actor head, which has per_action outputs per action dim (Categorical 1, tanh-Normal 2); A <= kMaxActions.
int head_dims(const StxMlp* actor, int per_action, int* A, const char* who) {
  const int w = actor->sizes[actor->n_layers];
  *A = w / per_action;
  STX_REQUIRE(w % per_action == 0 && *A <= kMaxActions, STX_E_SHAPE, "%s: actor head width %d is not %d x A with A <= %d", who, w, per_action,
              kMaxActions);
  return STX_OK;
}

// The fp32 minibatch (checked by check_minibatch): actor forward, the actor loss `launch` on g (whose head-specific fields the
// caller has set), actor backward into grad_arena + aoff; then the critic's forward, clipped value loss and backward into
// grad_arena + coff.  Both networks carve `workspace` as stx_ppo_workspace_bytes() sizes it.
int fp32_minibatch(const StxMlp* actor, const StxMlp* critic, const StxPpoBatch* b, int64_t mb_off, int64_t mb, const StxPpoHyper* h,
                   float grad_weight, float* grad_arena, float* metrics, void* workspace, ActorLossArgs g, ActorLossLaunch launch,
                   cudaStream_t st) {
  int64_t aoff, coff;
  stx_ppo_arena_offsets(actor, critic, &aoff, &coff, nullptr);
  const int D = actor->sizes[0];
  const float* obs = reinterpret_cast<const float*>(b->obs);
  const int32_t* idx = b->perm ? b->perm + mb_off : nullptr;
  const float* x = idx ? obs : obs + mb_off * (int64_t)D;  // without a permutation: the contiguous row range from mb_off

  SimtHeadBufs hb{};
  if (int rc = simt_net_forward(actor, x, D, idx, mb, workspace, &hb, st)) return rc;
  g.r = {idx, mb_off, mb, hb.loss_partials, hb.counter, metrics, grad_weight};
  g.head = hb.head, g.dhead = hb.dhead, g.logp_old = b->log_prob, g.adv = b->advantages;
  g.adv_stats = h->standardize_advantages ? b->adv_stats : nullptr, g.clip_eps = h->clip_eps, g.ent_coef = h->ent_coef;
  if (int rc = launch(g, st)) return rc;
  if (int rc = simt_net_backward(actor, x, D, idx, mb, workspace, grad_weight, grad_arena + aoff, h->overwrite_grads, st)) return rc;

  if (int rc = simt_net_forward(critic, x, D, idx, mb, workspace, &hb, st)) return rc;
  const LossRows r{idx, mb_off, mb, hb.loss_partials, hb.counter, metrics, grad_weight};
  if (int rc = launch_critic_loss(r, hb.head, b->value, b->targets, hb.dhead, h->clip_eps, h->vf_coef, st)) return rc;
  return simt_net_backward(critic, x, D, idx, mb, workspace, grad_weight, grad_arena + coff, h->overwrite_grads, st);
}

// ---- PQN Q loss + its gradient with respect to the Q rows (one thread per minibatch row).
//
// Reference: _q_loss_fn of stoix/systems/q_learning/ff_pqn.py:139-162 under jax.grad: td = target - q[a], td_loss above,
// averaged over the minibatch (d q = -g / mb in column a; every other column 0).  Rows are read through the permutation and
// the metric is reduced with the PPO losses' LossRows / reduce_metrics (stx_ppo_loss.cuh).
__global__ void __launch_bounds__(256) q_loss_kernel(LossRows r, const float* __restrict__ q, const int32_t* __restrict__ action,
                                                     const float* __restrict__ targets, int A, float delta, float* __restrict__ dq) {
  const int64_t m = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  double s_loss = 0.0;
  const float inv_m = 1.0f / (float)r.mb;
  if (m < r.mb) {
    const int64_t src = r.src(m);
    const int a = action[src];
    const float td = targets[src] - q[m * A + a];
    float loss, g;
    td_loss(td, delta, loss, g);
    s_loss = (double)loss;
    for (int j = 0; j < A; ++j) dq[m * A + j] = j == a ? -g * inv_m : 0.f;
  }
  reduce_metrics<1>({s_loss}, {0}, r);
}

// ---- one-step Q-learning losses of the DQN family (one thread per sampled row); see stx_q_td_loss_grads in stx.h.
// The bootstrap value of the row's successor, one struct per rule.  q_t / q_aux point at the row.
struct MaxTarget {  // q_learning: max_a q_t
  __device__ __forceinline__ static float next_value(const float* q_t, const float*, int A, const StxQTdHyper&) {
    float v = q_t[0];
    for (int j = 1; j < A; ++j) v = fmaxf(v, q_t[j]);
    return v;
  }
  __device__ __forceinline__ static float bonus(const float*, int, int, const StxQTdHyper&) { return 0.f; }
};
struct DoubleTarget {  // double_q_learning: q_t_value[argmax q_t_selector], the first maximal index (jnp.argmax)
  __device__ __forceinline__ static float next_value(const float* q_t, const float* sel, int A, const StxQTdHyper&) {
    int best = 0;
    float bv = sel[0];
    for (int j = 1; j < A; ++j)
      if (sel[j] > bv) bv = sel[j], best = j;
    return q_t[best];
  }
  __device__ __forceinline__ static float bonus(const float*, int, int, const StxQTdHyper&) { return 0.f; }
};
struct MunchausenTarget {  // munchausen_q_learning: soft-Bellman value tau logsumexp(q_t / tau) and the clipped log-policy bonus
  // tau logsumexp(q / tau) = max q + tau log sum exp((q - max q) / tau): with tau = 0.03 the exponents of the plain form run to
  // the hundreds, here they are <= 0.
  __device__ __forceinline__ static float max_and_log_sum(const float* q, int A, float tau, float& mx) {
    mx = q[0];
    for (int j = 1; j < A; ++j) mx = fmaxf(mx, q[j]);
    float s = 0.f;
    for (int j = 0; j < A; ++j) s += expf((q[j] - mx) / tau);
    return logf(s);
  }
  __device__ __forceinline__ static float next_value(const float* q_t, const float*, int A, const StxQTdHyper& h) {
    float mx;
    const float ls = max_and_log_sum(q_t, A, h.entropy_temperature, mx);
    return mx + h.entropy_temperature * ls;
  }
  // alpha clip(tau log_softmax(q_tm1_target / tau)[a], clip_value_min, 0), tau log_softmax(q / tau)[a] = (q[a] - max q) - tau log s
  __device__ __forceinline__ static float bonus(const float* q_tgt, int a, int A, const StxQTdHyper& h) {
    float mx;
    const float ls = max_and_log_sum(q_tgt, A, h.entropy_temperature, mx);
    const float m = (q_tgt[a] - mx) - h.entropy_temperature * ls;
    return h.munchausen_coefficient * fminf(fmaxf(m, h.clip_value_min), 0.f);
  }
};

template <class Rule, bool REG>
__global__ void __launch_bounds__(256) q_td_loss_kernel(LossRows r, const float* __restrict__ q_tm1, const float* __restrict__ q_t,
                                                        const float* __restrict__ q_aux, const int32_t* __restrict__ action,
                                                        const float* __restrict__ reward, const uint8_t* __restrict__ done,
                                                        const float* __restrict__ discount, int A, StxQTdHyper h, float* __restrict__ dq) {
  const int64_t m = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  double s_loss = 0.0;
  const float inv_m = 1.0f / (float)r.mb;
  if (m < r.mb) {
    const int a = action[m];
    const float rt = fminf(fmaxf(reward[m], -h.max_abs_reward), h.max_abs_reward);          // jnp.clip(reward, -max, max)
    const float dt = discount ? discount[m] : (1.f - (float)done[m]) * h.gamma;               // (1 - done) gamma
    const float* aux = q_aux ? q_aux + m * A : nullptr;
    const float target = (rt + Rule::bonus(aux, a, A, h)) + dt * Rule::next_value(q_t + m * A, aux, A, h);
    const float qa = q_tm1[m * A + a];
    float loss, g;
    td_loss(target - qa, h.huber_delta, loss, g);
    float da = -g * inv_m;
    if (REG) {  // + regularizer_coeff mean(q_tm1[a]) (ff_dqn_reg.py:174-176)
      loss += h.regularizer_coeff * qa;
      da += h.regularizer_coeff * inv_m;
    }
    s_loss = (double)loss;
    for (int j = 0; j < A; ++j) dq[m * A + j] = j == a ? da : 0.f;
  }
  reduce_metrics<1>({s_loss}, {0}, r);
}

}  // namespace
}  // namespace stx

using namespace stx;

// ---- value-only faces of the loss utilities (the training path fuses the same arithmetic with its gradient) --------------
extern "C" size_t stx_loss_scratch_bytes(void) { return 16 + sizeof(double) * 2 * stx::kNumSMs; }

extern "C" int stx_ppo_clip_loss(const float* pi_log_prob_t, const float* b_pi_log_prob_t, const float* gae_t, int64_t n, float epsilon, float* out,
                                 void* scratch, void* stream) {
  STX_REQUIRE(pi_log_prob_t && b_pi_log_prob_t && gae_t && out && scratch && n > 0, STX_E_ARG, "stx_ppo_clip_loss: bad arguments");
  return launch_face(SurrogateFace<ClipLoss>{pi_log_prob_t, b_pi_log_prob_t, gae_t, nullptr, {epsilon}, 0.f}, n, out, scratch, stream);
}

extern "C" int stx_clipped_value_loss(const float* pred_value_t, const float* behavior_value_t, const float* targets_t, int64_t n, float epsilon,
                                      float* out, void* scratch, void* stream) {
  STX_REQUIRE(pred_value_t && behavior_value_t && targets_t && out && scratch && n > 0, STX_E_ARG, "stx_clipped_value_loss: bad arguments");
  return launch_face(ValueFace{pred_value_t, behavior_value_t, targets_t, epsilon}, n, out, scratch, stream);
}

extern "C" int stx_ppo_penalty_loss(const float* pi_log_prob_t, const float* b_pi_log_prob_t, const float* gae_t, const float* kl, int64_t n,
                                    float beta, float* out, void* scratch, void* stream) {
  STX_REQUIRE(pi_log_prob_t && b_pi_log_prob_t && gae_t && kl && out && scratch && n > 0, STX_E_ARG, "stx_ppo_penalty_loss: bad arguments");
  return launch_face(SurrogateFace<KlPenaltyLoss>{pi_log_prob_t, b_pi_log_prob_t, gae_t, kl, {}, beta}, n, out, scratch, stream);
}

extern "C" int stx_dpo_loss(const float* pi_log_prob_t, const float* b_pi_log_prob_t, const float* gae_t, int64_t n, float alpha, float beta,
                            float* out, void* scratch, void* stream) {
  STX_REQUIRE(pi_log_prob_t && b_pi_log_prob_t && gae_t && out && scratch && n > 0 && alpha > 0.f && beta > 0.f, STX_E_ARG,
              "stx_dpo_loss: bad arguments");
  return launch_face(SurrogateFace<DpoLoss>{pi_log_prob_t, b_pi_log_prob_t, gae_t, nullptr, {alpha, beta}, 0.f}, n, out, scratch, stream);
}

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

// ---- PPO loss heads on precomputed network outputs (the recurrent system runs its networks outside the fused PPO kernels) ----
extern "C" size_t stx_ppo_head_scratch_bytes(int64_t mb) { return 256 + (size_t)((mb + 255) / 256) * 6 * sizeof(double); }

extern "C" int stx_ppo_head_grads(const float* logits, const float* value, const int32_t* idx, int64_t row0, const int32_t* action,
                                  const float* logp_old, const float* v_old, const float* adv, const float* targets, const float* adv_stats,
                                  int64_t mb, int A, float clip_eps, float ent_coef, float vf_coef, float* d_logits, float* d_value, float* metrics,
                                  float weight, void* scratch, void* stream) {
  STX_REQUIRE((logits || value) && action && logp_old && v_old && adv && targets && metrics && scratch && mb > 0, STX_E_ARG,
              "stx_ppo_head_grads: null pointer or mb=%lld", (long long)mb);
  STX_REQUIRE(!logits || (d_logits && A > 0 && A <= kMaxActions), STX_E_SHAPE, "stx_ppo_head_grads: A=%d (max %d) / null d_logits", A, kMaxActions);
  STX_REQUIRE(!value || d_value, STX_E_ARG, "stx_ppo_head_grads: null d_value");
  cudaStream_t st = (cudaStream_t)stream;
  const LossRows r = scratch_rows(idx, row0, mb, metrics, weight, scratch);
  if (logits) {  // actor then critic: each is one launch of the kernel the fused fp32 path uses
    ActorLossArgs g{};
    g.r = r, g.head = logits, g.action = action, g.logp_old = logp_old, g.adv = adv, g.adv_stats = adv_stats, g.dhead = d_logits, g.A = A;
    g.clip_eps = clip_eps, g.ent_coef = ent_coef;
    if (int rc = launch_actor_loss<CategoricalRow, ClipLoss>(g, st)) return rc;
  }
  return value ? launch_critic_loss(r, value, v_old, targets, d_value, clip_eps, vf_coef, st) : STX_OK;
}

extern "C" int stx_ppo_tanh_normal_head_grads(const float* head_out, const int32_t* idx, int64_t row0, const StxTanhNormalPpo* head,
                                              const float* logp_old, const float* adv, const float* adv_stats, int64_t mb, int A, float clip_eps,
                                              float ent_coef, float* d_head_out, float* metrics, float weight, void* scratch, void* stream) {
  STX_REQUIRE(head_out && head_ok(head) && logp_old && adv && d_head_out && metrics && scratch && mb > 0, STX_E_ARG,
              "stx_ppo_tanh_normal_head_grads: null pointer, empty minibatch or bad action bounds");
  STX_REQUIRE(A > 0 && A <= kMaxActions, STX_E_SHAPE, "stx_ppo_tanh_normal_head_grads: A=%d (max %d)", A, kMaxActions);
  ActorLossArgs g{};
  g.r = scratch_rows(idx, row0, mb, metrics, weight, scratch);
  g.head = head_out, g.tn = *head, g.logp_old = logp_old, g.adv = adv, g.adv_stats = adv_stats, g.dhead = d_head_out, g.A = A;
  g.clip_eps = clip_eps, g.ent_coef = ent_coef;
  return launch_actor_loss<TanhNormalRow, ClipLoss>(g, (cudaStream_t)stream);
}

extern "C" int stx_ppo_penalty_head_grads(const float* logits, const int32_t* idx, int64_t row0, const StxPpoVariant* v, const int32_t* action,
                                          const float* logp_old, const float* adv, const float* adv_stats, int64_t mb, int A, float ent_coef,
                                          float* d_logits, float* metrics, float weight, void* scratch, void* stream) {
  if (int rc = check_variant(v, true, "stx_ppo_penalty_head_grads")) return rc;
  STX_REQUIRE(logits && action && logp_old && adv && d_logits && metrics && scratch && mb > 0, STX_E_ARG,
              "stx_ppo_penalty_head_grads: null pointer or empty minibatch");
  STX_REQUIRE(A > 0 && A <= kMaxActions, STX_E_SHAPE, "stx_ppo_penalty_head_grads: A=%d (max %d)", A, kMaxActions);
  ActorLossArgs g{};
  g.r = scratch_rows(idx, row0, mb, metrics, weight, scratch);
  g.head = logits, g.behaviour = v->behaviour, g.action = action, g.logp_old = logp_old, g.adv = adv, g.adv_stats = adv_stats;
  g.dhead = d_logits, g.A = A, g.kl_coef = v->kl_coef, g.ent_coef = ent_coef;
  return launch_actor_loss<CategoricalRow, KlPenaltyLoss>(g, (cudaStream_t)stream);
}

extern "C" int stx_ppo_variant_tanh_normal_head_grads(const float* head_out, const int32_t* idx, int64_t row0, const StxTanhNormalPpo* head,
                                                      const StxPpoVariant* v, const float* logp_old, const float* adv, const float* adv_stats,
                                                      int64_t mb, int A, float ent_coef, float* d_head_out, float* metrics, float weight,
                                                      void* scratch, void* stream) {
  if (int rc = check_variant(v, false, "stx_ppo_variant_tanh_normal_head_grads")) return rc;
  STX_REQUIRE(head_out && head_ok(head) && logp_old && adv && d_head_out && metrics && scratch && mb > 0, STX_E_ARG,
              "stx_ppo_variant_tanh_normal_head_grads: null pointer, empty minibatch or bad action bounds");
  STX_REQUIRE(A > 0 && A <= kMaxActions, STX_E_SHAPE, "stx_ppo_variant_tanh_normal_head_grads: A=%d (max %d)", A, kMaxActions);
  ActorLossArgs g{};
  g.r = scratch_rows(idx, row0, mb, metrics, weight, scratch);
  g.head = head_out, g.behaviour = v->behaviour, g.tn = *head, g.logp_old = logp_old, g.adv = adv, g.adv_stats = adv_stats;
  g.dhead = d_head_out, g.A = A, g.kl_coef = v->kl_coef, g.dpo_alpha = v->dpo_alpha, g.dpo_beta = v->dpo_beta, g.ent_coef = ent_coef;
  return tanh_normal_variant(v->kind)(g, (cudaStream_t)stream);
}

// ---- whole minibatches: both networks' forward, loss and backward --------------------------------------------------------
extern "C" int stx_ppo_minibatch_grads(const StxMlp* actor, const StxMlp* critic, const StxPpoBatch* b, int64_t mb_off, int64_t mb,
                                       const StxPpoHyper* h, float grad_weight, float* grad_arena, float* metrics, int precision, void* workspace,
                                       size_t workspace_bytes, void* stream) {
  const char* who = "stx_ppo_minibatch_grads";
  if (int rc = check_minibatch(actor, critic, b, mb_off, mb, h, grad_arena, metrics, precision, nullptr, workspace, workspace_bytes, who))
    return rc;
  STX_REQUIRE(b->action, STX_E_ARG, "%s: null batch action", who);
  ActorLossArgs g{};
  if (int rc = head_dims(actor, 1, &g.A, who)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (precision == STX_PREC_BF16)
    return tc_ppo_minibatch_grads(actor, critic, b, mb_off, mb, h, grad_weight, grad_arena, metrics, workspace, workspace_bytes, st);
  STX_REQUIRE(precision == STX_PREC_F32, STX_E_UNSUPPORTED, "%s: precision=%d", who, precision);
  g.action = b->action;
  return fp32_minibatch(actor, critic, b, mb_off, mb, h, grad_weight, grad_arena, metrics, workspace, g, launch_actor_loss<CategoricalRow, ClipLoss>,
                        st);
}

extern "C" int stx_ppo_continuous_minibatch_grads(const StxMlp* actor, const StxMlp* critic, const StxPpoBatch* b, const StxTanhNormalPpo* head,
                                                  int64_t mb_off, int64_t mb, const StxPpoHyper* h, float grad_weight, float* grad_arena,
                                                  float* metrics, int precision, void* workspace, size_t workspace_bytes, void* stream) {
  const char* who = "stx_ppo_continuous_minibatch_grads";
  if (int rc = check_minibatch(actor, critic, b, mb_off, mb, h, grad_arena, metrics, precision, "the tanh-Normal head has", workspace,
                               workspace_bytes, who))
    return rc;
  STX_REQUIRE(head_ok(head), STX_E_ARG, "%s: null head / action or bad action bounds", who);
  ActorLossArgs g{};
  if (int rc = head_dims(actor, 2, &g.A, who)) return rc;
  g.tn = *head;
  return fp32_minibatch(actor, critic, b, mb_off, mb, h, grad_weight, grad_arena, metrics, workspace, g, launch_actor_loss<TanhNormalRow, ClipLoss>,
                        (cudaStream_t)stream);
}

extern "C" int stx_ppo_penalty_minibatch_grads(const StxMlp* actor, const StxMlp* critic, const StxPpoBatch* b, const StxPpoVariant* v,
                                               int64_t mb_off, int64_t mb, const StxPpoHyper* h, float grad_weight, float* grad_arena,
                                               float* metrics, int precision, void* workspace, size_t workspace_bytes, void* stream) {
  const char* who = "stx_ppo_penalty_minibatch_grads";
  if (int rc = check_minibatch(actor, critic, b, mb_off, mb, h, grad_arena, metrics, precision, "the KL-penalty loss has", workspace,
                               workspace_bytes, who))
    return rc;
  if (int rc = check_variant(v, true, who)) return rc;
  STX_REQUIRE(b->action, STX_E_ARG, "%s: null batch action", who);
  ActorLossArgs g{};
  if (int rc = head_dims(actor, 1, &g.A, who)) return rc;
  g.behaviour = v->behaviour, g.action = b->action, g.kl_coef = v->kl_coef;
  return fp32_minibatch(actor, critic, b, mb_off, mb, h, grad_weight, grad_arena, metrics, workspace, g,
                        launch_actor_loss<CategoricalRow, KlPenaltyLoss>, (cudaStream_t)stream);
}

extern "C" int stx_ppo_variant_continuous_minibatch_grads(const StxMlp* actor, const StxMlp* critic, const StxPpoBatch* b,
                                                          const StxTanhNormalPpo* head, const StxPpoVariant* v, int64_t mb_off, int64_t mb,
                                                          const StxPpoHyper* h, float grad_weight, float* grad_arena, float* metrics,
                                                          int precision, void* workspace, size_t workspace_bytes, void* stream) {
  const char* who = "stx_ppo_variant_continuous_minibatch_grads";
  if (int rc = check_minibatch(actor, critic, b, mb_off, mb, h, grad_arena, metrics, precision, "the KL-penalty and DPO losses have", workspace,
                               workspace_bytes, who))
    return rc;
  if (int rc = check_variant(v, false, who)) return rc;
  STX_REQUIRE(head_ok(head), STX_E_ARG, "%s: null head / action or bad action bounds", who);
  ActorLossArgs g{};
  if (int rc = head_dims(actor, 2, &g.A, who)) return rc;
  g.behaviour = v->behaviour, g.tn = *head, g.kl_coef = v->kl_coef, g.dpo_alpha = v->dpo_alpha, g.dpo_beta = v->dpo_beta;
  return fp32_minibatch(actor, critic, b, mb_off, mb, h, grad_weight, grad_arena, metrics, workspace, g, tanh_normal_variant(v->kind),
                        (cudaStream_t)stream);
}

extern "C" int stx_q_loss_grads(const float* q, const int32_t* idx, int64_t row0, const int32_t* action, const float* targets, int64_t mb, int A,
                                float huber_delta, float* d_q, float* metrics, float weight, void* scratch, void* stream) {
  STX_REQUIRE(q && action && targets && d_q && metrics && scratch, STX_E_ARG, "stx_q_loss_grads: null pointer");
  STX_REQUIRE(mb > 0 && A > 0 && row0 >= 0, STX_E_SHAPE, "stx_q_loss_grads: mb=%lld A=%d row0=%lld", (long long)mb, A, (long long)row0);
  const LossRows r = scratch_rows(idx, row0, mb, metrics, weight, scratch);
  q_loss_kernel<<<(unsigned)((mb + 255) / 256), 256, 0, (cudaStream_t)stream>>>(r, q, action, targets, A, huber_delta, d_q);
  STX_LAUNCH_OK();
  return STX_OK;
}

extern "C" int stx_q_td_loss_grads(int rule, const float* q_tm1, const float* q_t, const float* q_aux, const int32_t* action, const float* reward,
                                   const uint8_t* done, const float* discount, int64_t M, int A, const StxQTdHyper* hyper, float* d_q, float* metrics,
                                   float weight, void* scratch, void* stream) {
  const char* who = "stx_q_td_loss_grads";
  STX_REQUIRE(q_tm1 && q_t && action && reward && (done || discount) && hyper && d_q && metrics && scratch, STX_E_ARG, "%s: null pointer", who);
  STX_REQUIRE(M > 0 && A > 0, STX_E_SHAPE, "%s: M=%lld A=%d", who, (long long)M, A);
  STX_REQUIRE(rule >= STX_Q_DQN && rule <= STX_Q_DQN_REG, STX_E_UNSUPPORTED, "%s: rule %d", who, rule);
  STX_REQUIRE((rule != STX_Q_DOUBLE && rule != STX_Q_MUNCHAUSEN) || q_aux, STX_E_ARG, "%s: rule %d needs q_aux (%s)", who, rule,
              rule == STX_Q_DOUBLE ? "q_t_selector" : "q_tm1_target");
  STX_REQUIRE(rule != STX_Q_MUNCHAUSEN || hyper->entropy_temperature > 0.f, STX_E_ARG, "%s: entropy_temperature must be > 0", who);
  const LossRows r = scratch_rows(nullptr, 0, M, metrics, weight, scratch);
  const unsigned grid = (unsigned)((M + 255) / 256);
  cudaStream_t st = (cudaStream_t)stream;
  const StxQTdHyper h = *hyper;
  switch (rule) {
    case STX_Q_DQN: q_td_loss_kernel<MaxTarget, false><<<grid, 256, 0, st>>>(r, q_tm1, q_t, nullptr, action, reward, done, discount, A, h, d_q); break;
    case STX_Q_DOUBLE: q_td_loss_kernel<DoubleTarget, false><<<grid, 256, 0, st>>>(r, q_tm1, q_t, q_aux, action, reward, done, discount, A, h, d_q); break;
    case STX_Q_MUNCHAUSEN:
      q_td_loss_kernel<MunchausenTarget, false><<<grid, 256, 0, st>>>(r, q_tm1, q_t, q_aux, action, reward, done, discount, A, h, d_q);
      break;
    default: q_td_loss_kernel<MaxTarget, true><<<grid, 256, 0, st>>>(r, q_tm1, q_t, nullptr, action, reward, done, discount, A, h, d_q); break;
  }
  STX_LAUNCH_OK();
  return STX_OK;
}
