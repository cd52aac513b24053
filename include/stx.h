/*
 * stx.h -- C ABI of libstoixb200.so: the H100-native (sm_90a) kernels behind Stoix's Anakin ff_ppo hot path.
 *
 * The reference (EdanToledo/Stoix) has no FFI/plugin registry: its boundary is Python-level
 * (SURVEY.md section 8b).  This header is the C boundary a maintainer binds (ctypes stub in
 * INTEGRATION.md) to replace the JAX/XLA implementation of each reference function cited below.
 * All paths are relative to the reference checkout.
 *
 * Conventions (every entry point):
 *   - every pointer is a DEVICE pointer owned by the caller unless marked "host";
 *   - no allocation, no synchronisation, no host<->device copy inside; work is enqueued on the
 *     `stream` argument (a cudaStream_t passed as void*), so every call is CUDA-graph capturable;
 *   - return 0 on success, <0 for an invalid argument (STX_E_*), >0 for a cudaError_t;
 *     stx_last_error_string() describes the last failure on the calling thread;
 *   - re-entrant per stream; scratch/workspace buffers must not be shared by concurrent streams.
 *   - tensors are row-major and time-major: a (T, E) trajectory field has flat index t*E + e,
 *     matching merge_leading_dims (stoix/utils/jax_utils.py:29-43).
 */
#ifndef STX_H_
#define STX_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define STX_VERSION 100 /* major*100 + minor */

#define STX_OK 0
#define STX_E_ARG (-1)      /* null pointer / negative size */
#define STX_E_SHAPE (-2)    /* unsupported shape for this kernel */
#define STX_E_ALIGN (-3)    /* pointer or leading dimension not aligned as required */
#define STX_E_UNSUPPORTED (-4)
#define STX_E_WORKSPACE (-5) /* workspace too small */

#define STX_MAX_LAYERS 7 /* Dense layers per network (hidden layers + head) */

/* Compute precision of the MLP GEMMs. */
#define STX_PREC_F32 0  /* fp32 CUDA-core GEMMs: the parity path (reference is fp32 everywhere) */
#define STX_PREC_BF16 1 /* bf16 operands on wgmma tensor cores, fp32 accumulate, fp32 master weights */

/* Torso activation (stoix/networks/utils.py:9-24; flax.linen functions).  STX_PREC_BF16 kernels implement RELU only. */
#define STX_ACT_RELU 0
#define STX_ACT_TANH 1
#define STX_ACT_SILU 2     /* = swish */
#define STX_ACT_ELU 3
#define STX_ACT_GELU 4     /* nn.gelu default (tanh approximation) */
#define STX_ACT_SIGMOID 5
#define STX_ACT_SOFTPLUS 6
#define STX_ACT_IDENTITY 7 /* "identity" / "none" */

/*
 * One feed-forward network = MLPTorso(activation, use_layer_norm, activate_final=True) + Dense head
 * (stoix/networks/torso.py:12-33, heads.py:30-41 CategoricalHead, heads.py:129-134 ScalarCriticHead;
 * composed by FeedForwardActor / FeedForwardCritic, stoix/networks/base.py:18-59).
 * `params` is a flat fp32 arena, layer after layer.  Torso layer i without LayerNorm: W_i (sizes[i] x sizes[i+1],
 * row-major, the flax (in, out) kernel layout, y = x @ W + b) followed by b_i (sizes[i+1]).  With use_layer_norm
 * (torso.py:26-30: Dense(use_bias=False) -> nn.LayerNorm() -> activation): W_i, LayerNorm scale_i, LayerNorm bias_i
 * (sizes[i+1] each).  The head (last layer) is always W, b.
 */
typedef struct StxMlp {
  int32_t n_layers;                   /* Dense layers including the head, 1..STX_MAX_LAYERS */
  int32_t sizes[STX_MAX_LAYERS + 1];  /* sizes[0] = input dim, sizes[n_layers] = head width */
  const float* params;                /* fp32 arena, stx_mlp_param_count() floats */
  const void* params_bf16;            /* bf16 shadow arena (same layout), STX_PREC_BF16 only; may be NULL for F32 */
  int32_t activation;                 /* STX_ACT_* of the torso layers (0 = relu) */
  int32_t use_layer_norm;             /* 1: torso layers are Dense(no bias) + LayerNorm(eps 1e-6) */
} StxMlp;

/* Hyper-parameters of _actor_loss_fn / _critic_loss_fn
 * (stoix/systems/ppo/anakin/ff_ppo.py:191-235; configs/system/ppo/ff_ppo.yaml:6-22). */
typedef struct StxPpoHyper {
  float clip_eps;
  float ent_coef;
  float vf_coef;
  int32_t standardize_advantages; /* 1: use (adv - stats[0]) * stats[1] on load (multistep.py:138-139) */
  int32_t overwrite_grads;        /* 1: grad_arena = weight * g (no prior zero fill needed); 0: grad_arena += weight * g */
  int32_t reserved;
  void* adam_scratch;             /* nullable; bf16 path with overwrite_grads: also leave sum(g^2) partials of both
                                     optimiser segments in this stx_clip_adam_step scratch (then call it with prenorm = 1) */
} StxPpoHyper;

/* One optimiser = optax.chain(clip_by_global_norm(max_grad_norm), adam(lr, eps=1e-5))
 * (ff_ppo.py:449-463) over one contiguous segment of the flat arenas. */
typedef struct StxAdamSeg {
  int64_t offset;      /* first float of the segment in the arenas (multiple of 4; stx_ppo_arena_offsets gives 8) */
  int64_t count;       /* floats in the segment (padding excluded or zero-filled) */
  float init_lr;       /* system.actor_lr / critic_lr */
  float max_grad_norm; /* system.max_grad_norm */
} StxAdamSeg;

typedef struct StxAdamHyper {
  float b1, b2, eps;         /* optax.adam defaults 0.9 / 0.999, eps=1e-5 at ff_ppo.py:458,462 */
  float grad_scale;          /* grads are multiplied by this before clipping (1/world for a summed all-reduce) */
  int32_t decay;             /* system.decay_learning_rates: lr(k) = init_lr*(1-(k // steps_per_update)/num_updates), utils/training.py:24-26 */
  int32_t steps_per_update;  /* epochs * num_minibatches */
  int32_t num_updates;       /* arch.num_updates */
  int32_t prenorm;           /* 1: the scratch already holds the sum-of-squares partials of the (unscaled) gradients,
                                written by stx_ppo_minibatch_grads(adam_scratch): skip the norm pass and the grid barrier */
} StxAdamHyper;

/* ---------------------------------------------------------------------------------------------- */
int stx_version(void);
const char* stx_last_error_string(void);
/* Kernel launches enqueued by this library in this process so far (host-side count; launches replayed
 * from a captured CUDA graph are counted once, at capture). */
unsigned long long stx_launch_count(void);
/* "" or where a tensor-core kernel's bounded mbarrier wait timed out before it trapped (a synchronisation protocol bug):
 * block, thread, wait tag and phase parity of the first thread to time out in this process.  Host memory: readable after
 * the trap has made the CUDA context unusable. */
const char* stx_tc_trap_message(void);
/* Test hook: out[0] += the number of fp32 bit patterns in [lo, hi] where the call-free device reciprocal (fn 0) or square
 * root (fn 1) differs in any bit from 1.0f / x or sqrtf(x) on the device; out[1] = min(out[1], the first such pattern). */
int stx_debug_callfree_math(int fn, uint32_t lo, uint32_t hi, unsigned long long* out, void* stream);
/* Floats in one network arena (no padding). */
int64_t stx_mlp_param_count(const StxMlp* mlp);

/* ------------------------------------------------------------------ K2: GAE -------------------
 * Replaces batch_truncated_generalized_advantage_estimation, stoix/utils/multistep.py:14-145, in the
 * time-major form ff_ppo calls (ff_ppo.py:164-179).
 *
 * stx_gae_ppo_f32: inputs exactly as ff_ppo feeds them -- reward (T,E) f32, value = v_tm1 (T,E),
 * bootstrap_value = v_t (T,E), done / truncated (T,E) uint8 (0/1).  Computes
 *   r = reward*reward_scale; disc = (1-done)*gamma; delta = r + disc*v_t - v_tm1
 *   acc_t = delta_t + disc_t*lambda*acc_{t+1}*(1-trunc_t)  (reverse in t, acc_T = 0)
 *   adv = acc; targets = v_tm1 + adv.
 * standardize: 0 = none; 1 = also write stats[0]=mean(adv), stats[1]=rsqrt(E[adv^2]-mean^2+1e-5)
 *   (jax.nn.standardize over the whole (T,E) shard) leaving adv raw -- the PPO kernels apply it on
 *   load; 2 = as 1 and adv is standardised in place (materialised, +8 B/element).
 * scratch: >= stx_gae_scratch_bytes(T,E) bytes, zero-initialised once by the caller, reusable.
 */
size_t stx_gae_scratch_bytes(int T, int E);
int stx_gae_ppo_f32(const float* reward, const float* v_tm1, const float* v_t, const uint8_t* done,
                    const uint8_t* truncated, int T, int E, float gamma, float lambda_,
                    float reward_scale, int standardize, float* adv, float* targets, float* stats,
                    void* scratch, void* stream);
/* Tuning hook for experiments: force the env-quads per block (2, 4 or 8); 0 restores the heuristic. */
void stx_gae_set_tuning(int quads);
/* Generic face of the same function: float discount_t (T,E), optional per-element lambda (NULL ->
 * scalar lambda_), optional float truncation_t (NULL -> zeros).  Same outputs. */
int stx_gae_generic_f32(const float* r_t, const float* discount_t, const float* lambda_t,
                        float lambda_, const float* v_tm1, const float* v_t,
                        const float* truncation_t, int T, int E, int standardize, float* adv,
                        float* targets, float* stats, void* scratch, void* stream);

/* ------------------------------------------------------------------ K1: MLP forward -----------
 * Replaces FeedForwardActor/FeedForwardCritic.apply (stoix/networks/base.py:18-59) for MLP torsos.
 * x: (M, sizes[0]) f32 (STX_PREC_F32) or bf16 (STX_PREC_BF16), row stride ldx elements; row_idx
 * (nullable) gathers rows: row m reads x[row_idx[m]].  out: (M, sizes[n_layers]) f32.
 * workspace >= stx_mlp_forward_workspace_bytes(...).
 */
size_t stx_mlp_forward_workspace_bytes(const StxMlp* mlp, int64_t M, int precision);
int stx_mlp_forward(const StxMlp* mlp, const void* x, int64_t ldx, const int32_t* row_idx,
                    int64_t M, float* out, int precision, void* workspace, size_t workspace_bytes,
                    void* stream);

/* Bring-up / test hook of the bf16 tensor-core forward: as stx_mlp_forward(STX_PREC_BF16) and also
 * writes the bf16-rounded hidden activations h1, h2 ((M, 256) f32 each, nullable). */
int stx_tc_debug_forward(const StxMlp* mlp, const void* x, int64_t ldx, int64_t M, float* out, float* h1,
                         float* h2, void* stream);

/* Grid cap (CTAs) of the persistent bf16 forward kernel for the stx_mlp_forward launches that follow; 0 = one CTA per SM.
 * Lets a forward pass run beside another persistent kernel (the learner evaluates the critic on the SMs the rollout
 * kernel leaves idle) instead of queueing CTAs behind it.  Host-side state, read at launch time. */
void stx_tc_set_forward_ctas(int n);

/* Profiling hook kept for ABI compatibility: the K3a kernel of this build records no clock64() stamps, so the
 * buffer is left untouched.  Synchronous (not for capture). */
int stx_tc_debug_set_clock_buffer(long long* buf);
/* Profiling hook of the K3 launches: device buffer of [gridDim][8] int64 filled per CTA of K3a / K3b with
 * {role, total cycles, -, tiles (K3a) / -, -, chunks (K3b)} (see stx_tc_ppo.cu g_prof_buf); NULL disables. */
int stx_tc_debug_set_prof_buffer(long long* buf);

/* Categorical head ops on logits (E, A) -- tfd.Categorical (stoix/networks/heads.py:41) as used at
 * ff_ppo.py:100-101.  If sample != 0: action = argmax_j(logits_j + Gumbel_j) with Philox4x32-10
 * keyed by seed with counter (row, call = offset + *dev_counter); else `action` is an input.
 * dev_counter (nullable device uint64) lets a captured CUDA graph draw fresh numbers on every
 * replay: the caller bumps it with stx_counter_add at the end of the graph.  Always writes
 * log_prob = log_softmax(logits)[action]; entropy (nullable) = -sum p log p. */
int stx_categorical(const float* logits, int64_t E, int A, int sample, uint64_t seed,
                    uint64_t offset, const uint64_t* dev_counter, int32_t* action, float* log_prob,
                    float* entropy, void* stream);

/* ------------------------------------------------------------------ K3: PPO minibatch grads ---
 * Replaces the body of _update_minibatch up to (not including) the pmean: ff_ppo.py:184-247 with
 * ppo_clip_loss / clipped_value_loss (stoix/utils/loss.py:17-32, 68-78).  For minibatch rows
 * idx = perm[mb_off : mb_off+mb] of the flat (T*E) batch it re-runs both networks on obs[idx],
 * evaluates the two losses and ACCUMULATES d(total_loss)/d(params) into grad_arena (caller zeroes
 * it; layout = [actor arena | pad to 8 | critic arena | pad to 8], see stx_ppo_arena_offsets).
 * metrics[6] += {actor_loss, entropy, value_loss, mean(adv used), mean(pred value), mean(target)}.
 * obs: (B, D) f32 or bf16 per `precision`; perm NULL -> identity.
 */
typedef struct StxPpoBatch {
  const void* obs;          /* (B, D) */
  const int32_t* action;    /* (B) */
  const float* log_prob;    /* (B) behaviour log-prob, traj_batch.log_prob */
  const float* value;       /* (B) behaviour value, traj_batch.value */
  const float* advantages;  /* (B) raw (standardised on load if hyper says so) */
  const float* targets;     /* (B) */
  const float* adv_stats;   /* [mean, rstd] from stx_gae_*; NULL if not standardising */
  const int32_t* perm;      /* (B) permutation of the flat index, or NULL */
  int64_t B;
} StxPpoBatch;

/* workspace: >= stx_ppo_workspace_bytes(); its first 256 bytes must be zero on first use (the
 * kernels restore them), e.g. allocate it zero-filled once. */
void stx_ppo_arena_offsets(const StxMlp* actor, const StxMlp* critic, int64_t* actor_off,
                           int64_t* critic_off, int64_t* total);
size_t stx_ppo_workspace_bytes(const StxMlp* actor, const StxMlp* critic, int64_t mb, int precision);
int stx_ppo_minibatch_grads(const StxMlp* actor, const StxMlp* critic, const StxPpoBatch* batch,
                            int64_t mb_off, int64_t mb, const StxPpoHyper* hyper, float grad_weight,
                            float* grad_arena, float* metrics, int precision, void* workspace,
                            size_t workspace_bytes, void* stream);

/* One whole optimiser step on a minibatch = stx_ppo_minibatch_grads + stx_clip_adam_step (the body of
 * _update_minibatch, ff_ppo.py:184-284) with the gradient reduction and the optimiser fused into one launch:
 * the thread that reduces a gradient entry keeps it in a register, the blocks meet once at a grid barrier
 * for the two global norms, and the same thread applies clip + Adam to that entry.  STX_PREC_BF16 only,
 * single shard / single device (the gradients are overwritten, hyper->overwrite_grads is ignored);
 * opt->nseg must be 2 with segment 0 = actor arena and segment 1 = critic arena.  Same results as the
 * two separate calls (same reduction orders). */
typedef struct StxFusedAdam {
  float* param_arena;
  float* mu;
  float* nu;
  int32_t* counts;          /* int32[2*nseg] device */
  const StxAdamSeg* segs;   /* DEVICE pointer */
  int32_t nseg;
  int32_t reserved;
  StxAdamHyper hyper;       /* prenorm is ignored */
  void* params_bf16;        /* nullable */
  float* gnorm_out;         /* nullable, float[nseg] */
  void* scratch;            /* >= stx_adam_scratch_bytes(), zeroed once */
} StxFusedAdam;
int stx_ppo_minibatch_update(const StxMlp* actor, const StxMlp* critic, const StxPpoBatch* batch,
                             int64_t mb_off, int64_t mb, const StxPpoHyper* hyper, float grad_weight,
                             float* grad_arena, float* metrics, void* workspace, size_t workspace_bytes,
                             const StxFusedAdam* opt, void* stream);

/* Forward values of the two reference loss utilities (stoix/utils/loss.py:17-32 ppo_clip_loss,
 * :68-78 clipped_value_loss) over n elements; out[0] = mean.  scratch >= stx_loss_scratch_bytes(),
 * zeroed once.  (The training path uses the fused stx_ppo_minibatch_grads instead.) */
size_t stx_loss_scratch_bytes(void);
int stx_ppo_clip_loss(const float* pi_log_prob_t, const float* b_pi_log_prob_t, const float* gae_t,
                      int64_t n, float epsilon, float* out, void* scratch, void* stream);
int stx_clipped_value_loss(const float* pred_value_t, const float* behavior_value_t,
                           const float* targets_t, int64_t n, float epsilon, float* out, void* scratch,
                           void* stream);

/* ------------------------------------------------------------------ K4: clip + Adam -----------
 * Replaces optax.chain(clip_by_global_norm, adam) .update + optax.apply_updates for all segments in
 * one launch (ff_ppo.py:264-273).  counts: int32[2*nseg] = {adam count, schedule count} per segment,
 * kept on the device so the step is graph-replayable.  params_bf16 (nullable): bf16 shadow arena
 * refreshed in the same pass.  segs: DEVICE pointer to nseg StxAdamSeg.  gnorm_out (nullable):
 * float[nseg] pre-clip global norms.  scratch: >= stx_adam_scratch_bytes(nseg), zeroed once.
 */
size_t stx_adam_scratch_bytes(int nseg);
int stx_clip_adam_step(float* param_arena, const float* grad_arena, float* mu, float* nu,
                       int32_t* counts, const StxAdamSeg* segs, int nseg, const StxAdamHyper* hyper,
                       void* params_bf16, float* gnorm_out, void* scratch, void* stream);

/* C1 fused into K4 -- replaces jax.lax.pmean(axis "device") + both optimiser updates (ff_ppo.py:258-273) in
 * ONE launch per rank: a one-shot all-reduce by direct loads from every rank's gradient arena over NVLink peer
 * memory (summed in rank order => identical on all ranks), then global-norm clip + Adam as
 * stx_clip_adam_step (hyper->grad_scale = 1/world gives the mean).
 *   peer_grads[r]       HOST array of `world` DEVICE pointers: this call's gradient arena on rank r, peer-mapped
 *                       into this process (e.g. torch symmetric memory buffer_ptrs).
 *   peer_signal_pads[r] likewise: a zero-initialised uint32 area per rank; slots [pad_slot_offset .. +world)
 *                       are used (slot s of rank r's pad is written by rank s with release.sys stores).
 *   gsum                local fp32 arena receiving the summed gradient.
 * The caller must alternate between two gradient arenas from one call to the next (ping-pong): together with
 * the in-kernel handshake this guarantees no arena is rewritten while a peer may still read it.  Every rank
 * must issue the same sequence of calls.  CUDA-graph capturable (all state is in device memory). */
int stx_allreduce_clip_adam_step(float* param_arena, const float* const* peer_grads, void* const* peer_signal_pads,
                                 int world, int rank, int pad_slot_offset, float* gsum, float* mu, float* nu,
                                 int32_t* counts, const StxAdamSeg* segs, int nseg, const StxAdamHyper* hyper,
                                 void* params_bf16, float* gnorm_out, void* scratch, void* stream);
/* Two-shot form (the default of the learner): rank r sums slice r of the W gradient arenas (peer LOADS, rank order) and stores
 * the result into every rank's reduced-gradient buffer (peer STORES), so (W-1)/W of the arena crosses NVLink in each direction
 * instead of W-1 arenas inbound; the per-rank sum-of-squares partials of the clipping norm travel with the slices and the second
 * hand-shake replaces the grid barrier of the norm.  Every element is reduced once, by one rank => identical on all ranks.
 *   peer_gsum[r]   HOST array of `world` DEVICE pointers: rank r's reduced-gradient buffer, peer-mapped, arena_len + 128 floats
 *                  (tail: double[world][8] norm partials).  arena_len % 4 == 0; the padding between segments must hold zeros.
 *   signal pads    slots [pad_slot_offset, +8) "gradients ready", [pad_slot_offset + 8, +16) "slice stored".
 *   grid           0 = one block per SM; tests that run several virtual ranks on one device pass a small co-resident grid. */
int stx_allreduce2_clip_adam_step(float* param_arena, const float* const* peer_grads, float* const* peer_gsum, int64_t arena_len,
                                  void* const* peer_signal_pads, int world, int rank, int pad_slot_offset, float* mu, float* nu,
                                  int32_t* counts, const StxAdamSeg* segs, int nseg, const StxAdamHyper* hyper, void* params_bf16,
                                  float* gnorm_out, void* scratch, int grid, void* stream);

/* ------------------------------------------------------------------ shuffle -------------------
 * perm[i] = keyed bijection of [0, n) (cycle-walking Feistel over Philox rounds) replacing
 * jax.random.permutation + jnp.take (ff_ppo.py:294-303): the minibatch kernels gather through perm,
 * no shuffled copy of the batch is ever materialised. */
int stx_make_permutation(int32_t* perm, int64_t n, uint64_t seed, uint64_t stream_id,
                         const uint64_t* dev_counter, void* stream);
/* *counter += inc on the stream (device-resident RNG stream positions for graph replay). */
int stx_counter_add(uint64_t* counter, uint64_t inc, void* stream);

/* ------------------------------------------------------------------ synthetic Box env ---------
 * The named benchmark environment (BASELINE.json configs[1], SURVEY.md 8d): obs ~ N(0,1)^D,
 * reward ~ N(0,1), terminated ~ Bernoulli(p_term), truncated = !terminated & Bernoulli(p_trunc),
 * with stoa's AutoResetWrapper(next_obs_in_extras) + RecordEpisodeMetrics semantics
 * (stoix/utils/make_env.py:29-61, stoix/wrappers/envpool.py:94-133):
 *   next_obs  = true successor observation (extras["next_obs"]),
 *   obs_out   = reset observation where the episode ended, else next_obs,
 *   ep_return/ep_length running totals, published with is_terminal on the last step.
 * obs buffers are f32 or bf16 per obs_bf16.  Philox counter = (env, step + *dev_counter).
 */
int stx_synth_env_step(int64_t E, int D, uint64_t seed, uint64_t step, const uint64_t* dev_counter,
                       float p_term, float p_trunc, const int32_t* action, void* obs_out, void* next_obs, int obs_bf16,
                       float* reward, uint8_t* done, uint8_t* truncated, float* run_return,
                       int32_t* run_length, float* ep_return, int32_t* ep_length,
                       uint8_t* is_terminal, void* stream);

/* Fused persistent rollout of the synthetic env on the bf16 tensor-core path: the T-step scan of _env_step
 * (ff_ppo.py:81-140) for the actor side in ONE launch (grid = E/128 CTAs, each owning 128 envs for all T
 * steps): logits -> Gumbel-max action + log_prob (same Philox counters as stx_categorical with seed
 * cat_seed, call = cat_offset + t + *cat_counter) and the env step of stx_synth_env_step (step = env_step + t +
 * *env_counter), trajectory written time-major: obs (T+1,E,D) bf16 [row 0 is the input], next_obs (T,E,D)
 * bf16, the rest (T,E).  Bit-identical to the per-step path.  E % 128 == 0; actor as for STX_PREC_BF16. */
int stx_tc_rollout_synth(const StxMlp* actor, void* obs, void* next_obs, int32_t* action, float* log_prob,
                         float* reward, uint8_t* done, uint8_t* truncated, float* ep_return, int32_t* ep_length,
                         uint8_t* is_terminal, float* run_return, int32_t* run_length, int T, int64_t E,
                         uint64_t env_seed, uint64_t env_step, const uint64_t* env_counter, float p_term,
                         float p_trunc, uint64_t cat_seed, uint64_t cat_offset, const uint64_t* cat_counter,
                         void* stream);

/* ---- Observation normalisation (stoix/utils/running_statistics.py) -------------------------------------------
 * Replaces update_statistics (running_statistics.py:204-345: batched Welford, psum over the mapped axes) and normalize
 * (:348-363) on the ff_ppo call sites stoix/systems/ppo/anakin/ff_ppo.py:90-94, 113-115, 145-162.
 *   accumulate: one pass over the raw fp32 batch x[rows][D] (optional per-row weights): sums[0..D) = sum w (x - mean),
 *               sums[D..2D) = sum w (x - mean)^2, sums[2D] = sum w, in double (deterministic two-level reduction).
 *               With N ranks the caller all-reduces (SUM) the 2D+1 doubles -- the reference's two psums in one exchange.
 *   finalize:   count += W; delta = S1 / count; mean += delta; summed_variance += S2 - delta * S1;
 *               std = clip(sqrt(clip(max(sv, 0) / count, min^2, max^2)), min, max)          -- in place on the state.
 *   normalize:  out = (x - mean) / std, optional clip to [-max_abs_value, max_abs_value] (<= 0: none); out fp32 or bf16.
 * D <= 256.  scratch: stx_running_stats_scratch_bytes(D) bytes, zero-initialised once by the caller. */
size_t stx_running_stats_scratch_bytes(int D);
int stx_running_stats_accumulate(const float* x, const float* weights, int64_t rows, int D, const float* mean, double* sums,
                                 void* scratch, void* stream);
int stx_running_stats_finalize(const double* sums, int D, int64_t* count, float* mean, float* summed_variance, float* std,
                               float std_min_value, float std_max_value, void* stream);
int stx_obs_normalize(const float* x, int64_t rows, int D, const float* mean, const float* std, float max_abs_value, void* out,
                      int out_bf16, void* stream);

/* ---- Generic train-mode MLP (fp32 path): the autodiff of one network as two calls --------------------------------
 * Replaces flax `apply` + `jax.grad` for networks outside the fused PPO kernels (ff_sac's actor and twin-Q networks,
 * stoix/systems/sac/ff_sac.py:177-226): forward_train keeps the pre-activations (and LayerNorm statistics) of the torso
 * in `workspace`; backward consumes d(loss)/d(output) and produces parameter gradients into `net_grad` (nullable; layout
 * of StxMlp.params; grad = weight * g, added unless overwrite) and / or d(loss)/d(input) into `d_input` (nullable, dense
 * M x sizes[0]) -- the latter is how the actor loss reaches the policy through Q(obs, action).  One workspace per
 * forward whose backward is still pending. */
size_t stx_mlp_train_workspace_bytes(const StxMlp* mlp, int64_t M);
int stx_mlp_forward_train(const StxMlp* mlp, const float* x, int64_t ldx, const int32_t* row_idx, int64_t M, float* out, void* workspace,
                          size_t workspace_bytes, void* stream);
int stx_mlp_backward(const StxMlp* mlp, const float* x, int64_t ldx, const int32_t* row_idx, int64_t M, const float* d_out, void* workspace,
                     size_t workspace_bytes, float grad_weight, float* net_grad, int overwrite, float* d_input, void* stream);

/* ---- ff_sac building blocks (stoix/systems/sac/ff_sac.py:149-321) -------------------------------------------------
 * tanh_normal_sample: NormalAffineTanhDistributionHead (stoix/networks/heads.py:44-65) on head_out[M][2A] = (loc | scale
 *   pre-activation): action = shift + s tanh(loc + (softplus(raw) + min_scale) eps) written with leading dim ld_action
 *   (e.g. straight into the action columns of the Q networks' concat(obs, action) input), log_prob of
 *   AffineTanhTransformedDistribution (stoix/networks/distributions.py:19-79, clipped tails, epsilon 1e-3).  eps_in NULL:
 *   eps ~ N(0,1) from Philox (seed, row, offset + *dev_counter); eps_out (nullable) keeps the noise for the backward.
 * tanh_normal_backward: d(loss)/d(head_out) of loss = g_logp_scale * exp(*log_alpha) * sum_rows log_prob + sum g_action.action
 *   under the reparameterisation (eps fixed): what jax.grad sees through `.sample(seed)` + `.log_prob` in _actor_loss_fn.
 * sac_actor_seed: actor loss mean(alpha log_prob - min(q1, q2)) (:207-226): dq_k = -1/M on the arg-min network.
 * sac_q_loss:     Q loss 0.5 mean((q_k - target)^2), target = r + (1-done) gamma (min next_q - alpha next_log_prob) (:177-205).
 * sac_alpha_grad: alpha loss mean(alpha * (-log_prob - target_entropy)) and its gradient w.r.t. log_alpha (:157-175).
 *   metrics[8] (accumulated with `weight`): actor_loss, entropy, q_loss, q_error, q1_pred, q2_pred, alpha_loss, alpha.
 * polyak_update: optax.incremental_update: target = tau * online + (1 - tau) * target (:296-299).
 * uniform_indices / gather_rows_f32 / gather_u8: the sampling half of the flashbax item buffer (uniform with replacement over
 *   [0, *range)), rows gathered with a destination leading dimension. */
int stx_tanh_normal_sample(const float* head_out, int64_t M, int A, const float* eps_in, uint64_t seed, uint64_t offset,
                           const uint64_t* dev_counter, float minimum, float maximum, float min_scale, float* action, int64_t ld_action,
                           float* log_prob, float* eps_out, void* stream);
int stx_tanh_normal_backward(const float* head_out, const float* eps, int64_t M, int A, float minimum, float maximum, float min_scale,
                             const float* log_alpha, float g_logp_scale, const float* g_action, int64_t ld_g_action, float* d_head_out,
                             void* stream);
int stx_sac_actor_seed(const float* q1, const float* q2, const float* log_prob, const float* log_alpha, int64_t M, float* dq1, float* dq2,
                       float* metrics, float weight, void* stream);
int stx_sac_q_loss(const float* q1, const float* q2, const float* next_q1, const float* next_q2, const float* next_log_prob,
                   const float* reward, const uint8_t* done, const float* log_alpha, float gamma, int64_t M, float* dq1, float* dq2,
                   float* metrics, float weight, void* stream);
int stx_sac_alpha_grad(const float* log_prob, const float* log_alpha, float target_entropy, int64_t M, int autotune, float* grad,
                       float grad_weight, int overwrite, float* metrics, float weight, void* stream);
int stx_polyak_update(float* target, const float* online, int64_t n, float tau, void* stream);
int stx_uniform_indices(int32_t* idx, int64_t M, uint64_t seed, uint64_t offset, const uint64_t* dev_counter, const int64_t* range,
                        void* stream);
int stx_gather_rows_f32(const float* src, const int32_t* idx, int64_t M, int C, float* dst, int64_t ld_dst, void* stream);
int stx_gather_u8(const uint8_t* src, const int32_t* idx, int64_t M, uint8_t* dst, void* stream);

/* Transition ring buffer -- the add / sample pair of flashbax's item buffer as ff_sac uses it (stoix/systems/sac/ff_sac.py:449-456:
 * make_item_buffer(max_length, min_length, sample_batch_size, add_batches, add_sequences); add at :149-150, sample at :226-227).
 * state: DEVICE int64[2] = {write position, number of valid items}: both calls are stream-ordered and CUDA-graph replayable.
 *   add:    appends n rows (row-major, time-major order of the (T, E) batch), overwriting the oldest when full.
 *   sample: M items uniform with replacement over the valid part (Philox (seed, row/4, offset + *dev_counter), the indices of
 *           stx_uniform_indices; idx_in non-NULL overrides them) written as the network inputs of one SAC epoch with leading
 *           dimension ld >= obs_dim + act_dim: xq_old = (obs | action), xq_new[:, :obs_dim] = obs, xq_next[:, :obs_dim] = next_obs
 *           (the latter two nullable), plus reward[M], done[M], idx_out[M] (nullable). */
typedef struct StxReplay {
  float* obs;        /* [capacity][obs_dim] */
  float* action;     /* [capacity][act_dim] */
  float* reward;     /* [capacity] */
  uint8_t* done;     /* [capacity] */
  float* next_obs;   /* [capacity][obs_dim] */
  int64_t* state;    /* device int64[2] */
  int64_t capacity;
  int32_t obs_dim;
  int32_t act_dim;
} StxReplay;
int stx_replay_add(const StxReplay* rb, const float* obs, const float* action, const float* reward, const uint8_t* done,
                   const float* next_obs, int64_t n, void* stream);
int stx_replay_sample(const StxReplay* rb, int64_t M, uint64_t seed, uint64_t offset, const uint64_t* dev_counter, const int32_t* idx_in,
                      float* xq_old, float* xq_new, float* xq_next, int64_t ld, float* reward, uint8_t* done, int32_t* idx_out,
                      void* stream);

/* Discrete transition ring buffer -- the item buffer of the DQN family (stoix/systems/q_learning/ff_dqn.py:339-347), whose
 * Transition holds one integer action per row (ff_dqn.py:317-324).  Same semantics as StxReplay (same add order and overwrite,
 * device write position / fill count, the Philox indices of stx_uniform_indices, idx_in overriding them); the two rings share
 * their kernels as one template over the action type.
 *   sample: writes obs (M, obs_dim), next_obs (M, obs_dim), action (M), reward (M), done (M) and idx_out (M, nullable).  obs and
 *           next_obs may be the two halves of one (2M, obs_dim) block, so that one forward covers both (ff_mdqn's target net). */
typedef struct StxReplayDiscrete {
  float* obs;        /* [capacity][obs_dim] */
  int32_t* action;   /* [capacity] */
  float* reward;     /* [capacity] */
  uint8_t* done;     /* [capacity]: timestep.last() (ff_dqn.py:121) */
  float* next_obs;   /* [capacity][obs_dim] */
  int64_t* state;    /* device int64[2] = {write position, number of valid items} */
  int64_t capacity;
  int32_t obs_dim;
  int32_t reserved;
} StxReplayDiscrete;
int stx_replay_add_discrete(const StxReplayDiscrete* rb, const float* obs, const int32_t* action, const float* reward, const uint8_t* done,
                            const float* next_obs, int64_t n, void* stream);
int stx_replay_sample_discrete(const StxReplayDiscrete* rb, int64_t M, uint64_t seed, uint64_t offset, const uint64_t* dev_counter,
                               const int32_t* idx_in, float* obs, float* next_obs, int32_t* action, float* reward, uint8_t* done,
                               int32_t* idx_out, void* stream);

/* ------------------------------------------------------------------ recurrent PPO building blocks (fp32) ------
 * stx_gru_sequence_forward / _backward: ScannedRNN(cell_type="gru") (stoix/networks/base.py:124-159; flax.linen.GRUCell) over a
 *   (T, E) sequence with episode resets, as RecurrentActor / RecurrentCritic run it (base.py:162-222) one step at a time in the
 *   rollout (rec_ppo.py:90-101, T = 1) and over a whole chunk inside the losses (rec_ppo.py:216-247, under jax.grad).
 *     gi     [T][E][3H]  input projections W_i x + b_i of all steps (columns r | z | n): the head of the pre-torso MLP
 *     reset  [T][E]      the carry entering step t is replaced by zeros where set (done | truncated of the PREVIOUS transition)
 *     h0     [E][H], w_h [H][3H] (columns r | z | n), b_hn [H];  h_seq [T][E][H] = the cell outputs (= new carries)
 *   backward: d_h_seq = d(loss)/d(h_t) from the layers above; writes d_gi [T][E][3H]; d_w_h / d_b_hn (nullable pair) receive
 *   grad_weight * gradient (added unless overwrite); d_h0 nullable.  `workspace` (stx_gru_workspace_bytes) carries the saved gates
 *   from forward to backward.
 * stx_ppo_head_grads: _actor_loss_fn / _critic_loss_fn (rec_ppo.py:207-257, same losses as ff_ppo.py:191-235) on network outputs
 *   already computed: d(loss)/d(logits) and / or d(loss)/d(value) + the loss metrics (actor_loss, entropy, value_loss, mean
 *   advantage, mean value, mean target; accumulated with `weight`).  Row m of logits / value pairs with row idx[m] (or row0 + m) of the
 *   batch arrays.  scratch: stx_ppo_head_scratch_bytes(mb), zeroed once. */
size_t stx_gru_workspace_bytes(int T, int64_t E, int H);
int stx_gru_sequence_forward(const float* gi, const uint8_t* reset, const float* h0, const float* w_h, const float* b_hn, int T, int64_t E, int H,
                             float* h_seq, void* workspace, size_t workspace_bytes, void* stream);
int stx_gru_sequence_backward(const float* d_h_seq, const uint8_t* reset, const float* w_h, int T, int64_t E, int H, void* workspace,
                              size_t workspace_bytes, float* d_gi, float* d_w_h, float* d_b_hn, float grad_weight, int overwrite, float* d_h0,
                              void* stream);
/* LSTM form of the above: ScannedRNN(cell_type="lstm") (flax.linen.LSTMCell: i, f, g, o gates; c' = f c + i g, h' = o tanh(c')).
 *   gi [T][E][4H] (columns i | f | g | o; the four hidden biases ride on the input projection), carry [E][2H] = (c | h), both halves
 *   zeroed at a reset, w_h [H][4H]; carry_last (nullable) = the carry after step T-1.  Per-step launches (W_h does not fit one SM). */
size_t stx_lstm_workspace_bytes(int T, int64_t E, int H);
int stx_lstm_sequence_forward(const float* gi, const uint8_t* reset, const float* carry0, const float* w_h, int T, int64_t E, int H, float* h_seq,
                              float* carry_last, void* workspace, size_t workspace_bytes, void* stream);
int stx_lstm_sequence_backward(const float* d_h_seq, const uint8_t* reset, const float* w_h, int T, int64_t E, int H, void* workspace,
                               size_t workspace_bytes, float* d_gi, float* d_w_h, float grad_weight, int overwrite, float* d_carry0, void* stream);
size_t stx_ppo_head_scratch_bytes(int64_t mb);
int stx_ppo_head_grads(const float* logits, const float* value, const int32_t* idx, int64_t row0, const int32_t* action, const float* logp_old,
                       const float* v_old, const float* adv, const float* targets, const float* adv_stats, int64_t mb, int A, float clip_eps,
                       float ent_coef, float vf_coef, float* d_logits, float* d_value, float* metrics, float weight, void* scratch, void* stream);

/* ------------------------------------------------------------------ continuous-action PPO (fp32) ---------------
 * The tanh-Normal head (NormalAffineTanhDistributionHead, heads.py:44-65; head_out[M][2A] = loc | scale pre-activation,
 * sigma = softplus(raw) + min_scale) under the PPO losses of stoix/systems/ppo/anakin/ff_ppo_continuous.py.
 * stx_tanh_normal_log_prob: log_prob of GIVEN actions (row stride ld_action) by the inverse path of
 *   AffineTanhTransformedDistribution.log_prob (distributions.py:56-80): the event is clipped to [min + 1e-3, max - 1e-3],
 *   the tails score log Phi((u_lo - loc)/sigma) - log 1e-3 and log Phi(-(u_hi - loc)/sigma) - log 1e-3, the band the Normal
 *   density of atanh((a - shift)/s) plus the inverse log-det of tanh and the scale; summed over the A dims.  The gradient
 *   entries below score the stored actions with the same device function.
 * Entropy: the reference's one-sample estimate entropy(seed) (distributions.py:85-88) per row,
 *   H = sum_j [1/2 + log sqrt(2 pi) + log sigma_j + log s + fldj(loc_j + sigma_j eps'_j)], fldj(x) = 2 (log 2 - x - softplus(-2x)),
 *   with eps' held fixed under the gradient.  eps' of minibatch row m, dims 4g..4g+3: Philox4x32-10 with
 *     key     = (seed & 0xffffffff, seed >> 32)
 *     counter = (m & 0xffffffff, call & 0xffffffff, (call >> 32) ^ (g << 20) ^ ((m >> 32) << 8), 0x50504f45)
 *   call = offset + *dev_counter (dev_counter nullable); words (x, y) -> dims 4g, 4g+1 and (z, w) -> 4g+2, 4g+3 through
 *   Box-Muller (r = sqrt(-2 log u01(x)), (r cos 2 pi u01(y), r sin 2 pi u01(y))), u01 as for the other Philox draws.
 *   eps_in (nullable, (mb, A)) replaces the draw; eps_out (nullable, (mb, A)) records the noise used.
 * stx_ppo_tanh_normal_head_grads: the actor half of _update_minibatch (ff_ppo_continuous.py:191-213) on head outputs already
 *   computed: row m of head_out pairs with batch row idx[m] (or row0 + m) of action / logp_old / adv (standardised on load when
 *   adv_stats is given).  Writes d(ppo_clip_loss - ent_coef * mean H)/d(head_out) and accumulates metrics[0] actor_loss,
 *   metrics[1] entropy, metrics[3] mean advantage (with `weight`).  scratch: stx_ppo_head_scratch_bytes(mb), zeroed once.
 * stx_ppo_continuous_minibatch_grads: stx_ppo_minibatch_grads for the tanh-Normal actor: actor forward, the kernel above and
 *   the actor backward, then the critic half the discrete fp32 path runs.  STX_PREC_F32 only; A <= 32; scalar critic; the
 *   batch's int32 `action` is unused (the head's float actions replace it).  Workspace: stx_ppo_workspace_bytes(F32). */
typedef struct StxTanhNormalPpo {
  const float* action;          /* (B, A) stored actions, traj_batch.action */
  const float* eps_in;          /* (mb, A) injected entropy noise, or NULL: Philox */
  float* eps_out;               /* (mb, A) noise used, or NULL */
  const uint64_t* dev_counter;  /* device RNG stream position added to `offset`, or NULL */
  uint64_t seed;
  uint64_t offset;
  float minimum, maximum;       /* action bounds of the head */
  float min_scale;
  int32_t reserved;
} StxTanhNormalPpo;
int stx_tanh_normal_log_prob(const float* head_out, int64_t M, int A, const float* action, int64_t ld_action, float minimum, float maximum,
                             float min_scale, float* log_prob, void* stream);
/* stx_tanh_normal_entropy: the per-row estimate H above for head_out rows 0..M-1 (row r draws as minibatch row r). */
int stx_tanh_normal_entropy(const float* head_out, int64_t M, int A, const float* eps_in, uint64_t seed, uint64_t offset,
                            const uint64_t* dev_counter, float minimum, float maximum, float min_scale, float* entropy, float* eps_out,
                            void* stream);
int stx_ppo_tanh_normal_head_grads(const float* head_out, const int32_t* idx, int64_t row0, const StxTanhNormalPpo* head, const float* logp_old,
                                   const float* adv, const float* adv_stats, int64_t mb, int A, float clip_eps, float ent_coef, float* d_head_out,
                                   float* metrics, float weight, void* scratch, void* stream);
int stx_ppo_continuous_minibatch_grads(const StxMlp* actor, const StxMlp* critic, const StxPpoBatch* batch, const StxTanhNormalPpo* head,
                                       int64_t mb_off, int64_t mb, const StxPpoHyper* hyper, float grad_weight, float* grad_arena, float* metrics,
                                       int precision, void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------ PPO variants: KL penalty and DPO (fp32) --------
 * Each variant replaces only the actor loss of _update_minibatch; the critic half, the networks' forward / backward, the
 * workspace (stx_ppo_workspace_bytes(F32)) and the metric reduction are the clip path's.  No ratio clipping in either.
 * KL penalty (ppo_penalty_loss, stoix/utils/loss.py:35-47; ff_ppo_penalty.py:150-178, ff_ppo_penalty_continuous.py:150-179):
 *   actor_loss = -mean(ratio A) + kl_coef * mean(KL_i), KL_i = KL(behaviour_i || pi_i), no gradient into the behaviour policy.
 *   The behaviour policy is the actor at the start of the update (:137); its head outputs are supplied per batch row in
 *   `behaviour` ((B, A) logits or (B, 2A) loc | scale pre-activation), read as behaviour[idx[m]] like the other batch fields.
 *   Categorical KL = sum_j pb_j (log pb_j - log p_j); tanh-Normal KL = the KL of the base Normals summed over the dims,
 *   sum_j [log(s_j / sb_j) + (sb_j^2 + (mb_j - m_j)^2) / (2 s_j^2) - 1/2] (the shared affine-tanh bijector cancels).
 * DPO (dpo_loss, loss.py:50-65; ff_dpo_continuous.py:160-170), tanh-Normal only:
 *   ld = logp - logp_old, x1 = (e^ld - 1) A, x2 = ld A, drift = 1[A>=0] relu(x1 - alpha tanh(x1/alpha)) + 1[A<0] relu(x2 - beta tanh(x2/beta)),
 *   actor_loss = -mean(e^ld A - drift).
 * Entropy: exact for the Categorical, the seeded estimate of the continuous section (same noise layout) for the tanh-Normal;
 *   total = actor_loss - ent_coef * mean H.
 * Metrics accumulated with `weight`: [0] actor_loss, [1] entropy, [6] kl_divergence (KL penalty only); the minibatch entries
 *   add [2] value_loss, [4] pred_value, [5] target_value from the critic half.  metrics must hold 7 floats.
 * STX_PREC_BF16 returns STX_E_UNSUPPORTED: the bf16 tensor-core kernels implement the clipped Categorical loss only. */
#define STX_PPO_KL_PENALTY 1
#define STX_PPO_DPO 2
typedef struct StxPpoVariant {
  const float* behaviour;  /* (B, head width) behaviour head outputs, STX_PPO_KL_PENALTY; NULL for STX_PPO_DPO */
  int32_t kind;            /* STX_PPO_KL_PENALTY or STX_PPO_DPO */
  float kl_coef;           /* beta of ppo_penalty_loss (system.kl_penalty_coef) */
  float dpo_alpha;         /* alpha of dpo_loss (system.alpha) */
  float dpo_beta;          /* beta of dpo_loss (system.beta) */
} StxPpoVariant;
/* Per-row KL(p || q): tfd.Categorical.kl_divergence (logits (M, A)) and the tanh-Normal head's (head outputs (M, 2A)). */
int stx_categorical_kl(const float* logits_p, const float* logits_q, int64_t M, int A, float* kl, void* stream);
int stx_tanh_normal_kl(const float* head_p, const float* head_q, int64_t M, int A, float min_scale, float* kl, void* stream);
/* Value faces (loss.py:35-47, 50-65) with stx_loss_scratch_bytes() scratch: stx_ppo_penalty_loss writes out[0] = the actor loss
 * and out[1] = mean(kl) from per-row kl; stx_dpo_loss writes out[0]. */
int stx_ppo_penalty_loss(const float* pi_log_prob_t, const float* b_pi_log_prob_t, const float* gae_t, const float* kl, int64_t n, float beta,
                         float* out, void* scratch, void* stream);
int stx_dpo_loss(const float* pi_log_prob_t, const float* b_pi_log_prob_t, const float* gae_t, int64_t n, float alpha, float beta, float* out,
                 void* scratch, void* stream);
/* Actor halves on head outputs computed elsewhere: row m pairs with batch row idx[m] (or row0 + m); A <= 32; scratch:
 * stx_ppo_head_scratch_bytes(mb), zeroed once.  stx_ppo_penalty_head_grads is the Categorical KL penalty (v->kind must be
 * STX_PPO_KL_PENALTY); stx_ppo_variant_tanh_normal_head_grads serves both kinds. */
int stx_ppo_penalty_head_grads(const float* logits, const int32_t* idx, int64_t row0, const StxPpoVariant* v, const int32_t* action,
                               const float* logp_old, const float* adv, const float* adv_stats, int64_t mb, int A, float ent_coef, float* d_logits,
                               float* metrics, float weight, void* scratch, void* stream);
int stx_ppo_variant_tanh_normal_head_grads(const float* head_out, const int32_t* idx, int64_t row0, const StxTanhNormalPpo* head,
                                           const StxPpoVariant* v, const float* logp_old, const float* adv, const float* adv_stats, int64_t mb,
                                           int A, float ent_coef, float* d_head_out, float* metrics, float weight, void* scratch, void* stream);
/* Minibatch entries (like stx_ppo_minibatch_grads / stx_ppo_continuous_minibatch_grads): actor forward, the variant's loss
 * kernel, actor backward, critic half.  hyper->clip_eps clips only the value loss. */
int stx_ppo_penalty_minibatch_grads(const StxMlp* actor, const StxMlp* critic, const StxPpoBatch* batch, const StxPpoVariant* v, int64_t mb_off,
                                    int64_t mb, const StxPpoHyper* hyper, float grad_weight, float* grad_arena, float* metrics, int precision,
                                    void* workspace, size_t workspace_bytes, void* stream);
int stx_ppo_variant_continuous_minibatch_grads(const StxMlp* actor, const StxMlp* critic, const StxPpoBatch* batch, const StxTanhNormalPpo* head,
                                               const StxPpoVariant* v, int64_t mb_off, int64_t mb, const StxPpoHyper* hyper, float grad_weight,
                                               float* grad_arena, float* metrics, int precision, void* workspace, size_t workspace_bytes,
                                               void* stream);

/* ------------------------------------------------------------------ PQN: parallel Q-networks (fp32) ------------
 * The Q-learning system of stoix/systems/q_learning/ff_pqn.py: epsilon-greedy rollout, Q(lambda) targets, the l2 / Huber Q loss
 * and optax.chain(clip_by_global_norm, radam).
 *
 * stx_epsilon_greedy: distrax.EpsilonGreedy(preferences=q, epsilon).sample / .mode (stoix/networks/heads.py:202-217, ff_pqn.py:54-95)
 *   on q (E, A) rows.  epsilon is evaluated on the device from the optimiser count word `count` (nullable: count 0):
 *     update_no = *count / sched->steps_per_update                                          (ff_pqn.py:72)
 *     decay:    optax.linear_schedule(init_value, end_value, transition_steps) at update_no, in fp32:
 *               c = min(max(update_no, 0), transition_steps); eps = (init - end) * (1 - c / transition_steps) + end
 *               (transition_steps <= 0: eps = init_value)                                   (ff_pqn.py:286-297)
 *     constant: eps = end_value
 *   so a captured CUDA graph follows the schedule as the optimiser count advances.  Draw: two words (w0, w1) of Philox4x32-10
 *   keyed by seed with counter (row, call = offset + *dev_counter, as stx_categorical): explore if (w0 >> 8) * 2^-24 < eps
 *   (exact in fp32; always true at eps = 1), the action then being (w1 * A) >> 32 in 64-bit integers; otherwise the
 *   ((w1 * n_ties) >> 32)-th of the n_ties maximal indices.  mode != 0: the first maximal index (distrax mode()), no draw.
 *   epsilon_out / update_no_out (nullable, (E)) record the values for the episode metrics (ff_pqn.py:85-86).
 * stx_q_lambda_f32: batch_q_lambda (stoix/utils/multistep.py:533-569) over batch_lambda_returns (:314-408), time-major, on the
 *   rollout's stored flags: q_t (T, E, A) = Q of the successor rows, v_t = max_a q_t, d_t = gamma (1 - (done | truncated)),
 *   G_t = r_t + d_t [(1 - lambda) v_t + lambda G_{t+1}], the scan starting from v_t[T-1].  Evaluated as K2's chunked affine
 *   scan G_t = a_t + c_t G_{t+1} with a_t = r_t + d_t (1 - lambda) v_t, c_t = d_t lambda (last step: a = r + d v, c = 0).
 *   Writes targets (T, E) only.
 * stx_lambda_returns_f32: the generic face: float discount_t (T, E), v_t (T, E, A) reduced by max over A (A = 1:
 *   batch_lambda_returns itself), optional per-element lambda_t (NULL -> scalar lambda_).
 * stx_q_loss_grads: _q_loss_fn (ff_pqn.py:139-162) on Q rows computed elsewhere: row m of q (mb, A) pairs with batch row idx[m]
 *   (or row0 + m) of action / targets; td = targets - q[m, a]; loss = rlax.l2_loss(td) = td^2 / 2, or rlax.huber_loss(td, delta)
 *   when delta > 0; writes d q = d mean(loss) / d q: -clip(td, -delta, delta) / mb (l2: -td / mb) in column a, 0 elsewhere;
 *   metrics[0] += weight * mean(loss) (q_loss).  scratch: stx_ppo_head_scratch_bytes(mb), zeroed once.
 * stx_clip_radam_step: stx_clip_adam_step with optax.scale_by_radam (b1, b2, eps, eps_root, threshold; no nesterov) in place of
 *   scale_by_adam (ff_pqn.py:263-267): rho_inf = 2 / (1 - b2) - 1, rho_t = rho_inf - 2 t b2^t / (1 - b2^t) with t = count + 1;
 *   update = r_t mhat / (sqrt(vhat + eps_root) + eps), r_t = sqrt((rho_t - 4)(rho_t - 2) rho_inf / ((rho_inf - 4)(rho_inf - 2) rho_t))
 *   if rho_t >= threshold, else mhat.  rho_t and r_t are evaluated in double precision (in fp32 rho_t cancels catastrophically);
 *   everything else as stx_clip_adam_step.  hyper->adam.prenorm must be 0. */
typedef struct StxEpsilonSchedule {
  float init_value;          /* 1.0 in ff_pqn */
  float end_value;           /* system.training_epsilon (the constant schedule's value) */
  float transition_steps;    /* arch.num_updates * system.exploration_fraction */
  int32_t steps_per_update;  /* epochs * num_minibatches: optimiser steps per update */
  int32_t decay;             /* system.decay_epsilon */
  int32_t reserved;
} StxEpsilonSchedule;
typedef struct StxRadamHyper {
  StxAdamHyper adam;  /* b1, b2, eps, grad_scale and the learning-rate schedule, as for stx_clip_adam_step */
  float eps_root;     /* optax.radam default 0 */
  float threshold;    /* optax.radam default 5 */
} StxRadamHyper;
int stx_epsilon_greedy(const float* q, int64_t E, int A, int mode, uint64_t seed, uint64_t offset, const uint64_t* dev_counter,
                       const int32_t* count, const StxEpsilonSchedule* sched, int32_t* action, float* epsilon_out, int32_t* update_no_out,
                       void* stream);
int stx_q_lambda_f32(const float* q_t, int A, const float* r_t, const uint8_t* done, const uint8_t* truncated, int T, int E, float gamma,
                     float lambda_, float* targets, void* stream);
int stx_lambda_returns_f32(const float* r_t, const float* discount_t, const float* v_t, int A, const float* lambda_t, float lambda_, int T,
                           int E, float* targets, void* stream);
int stx_q_loss_grads(const float* q, const int32_t* idx, int64_t row0, const int32_t* action, const float* targets, int64_t mb, int A,
                     float huber_delta, float* d_q, float* metrics, float weight, void* scratch, void* stream);
int stx_clip_radam_step(float* param_arena, const float* grad_arena, float* mu, float* nu, int32_t* counts, const StxAdamSeg* segs, int nseg,
                        const StxRadamHyper* hyper, void* params_bf16, float* gnorm_out, void* scratch, void* stream);

/* ------------------------------------------------------------------ DQN family: one-step Q-learning losses (fp32) ----
 * stx_q_td_loss_grads: the _q_loss_fn of ff_dqn.py:147-178 / ff_ddqn.py / ff_mdqn.py / ff_dqn_reg.py:147-182 under jax.grad, on
 * Q rows computed elsewhere; one thread per row m of the sampled batch (rows contiguous, (M, A) each):
 *   r = clip(reward, -max_abs_reward, max_abs_reward);  d = (1 - done) gamma, done = timestep.last() (truncation cuts too)
 *   STX_Q_DQN, STX_Q_DQN_REG: target = r + d max_a q_t                           (utils/loss.py:106-124 q_learning)
 *   STX_Q_DOUBLE:             target = r + d q_t[argmax q_aux], q_aux = q_t_selector, first maximal index as jnp.argmax
 *                                                                                  (utils/loss.py:127-146 double_q_learning)
 *   STX_Q_MUNCHAUSEN:         target = r + alpha clip(tau log_softmax(q_aux / tau)[a], clip_value_min, 0) + d tau logsumexp(q_t / tau),
 *                             q_aux = q_tm1_target (the target net on obs), both in max-subtracted form (utils/loss.py:190-223)
 *   td = target - q_tm1[a];  loss = rlax.l2_loss(td), or rlax.huber_loss(td, huber_delta) when huber_delta > 0 (the element of
 *   stx_q_loss_grads); d_q = d mean(loss) / d q_tm1 in column a, 0 elsewhere.  STX_Q_DQN_REG adds regularizer_coeff mean(q_tm1[a])
 *   (ff_dqn_reg.py:174-176) to the loss: + regularizer_coeff / M in column a, and the q_loss metric includes the term.
 *   discount (nullable): per-row d given directly (the value faces of utils/loss.py take d_t); then done and gamma are unused.
 *   metrics[0] += weight * mean(loss) (q_loss).  scratch: stx_ppo_head_scratch_bytes(M), zeroed once. */
enum { STX_Q_DQN = 0, STX_Q_DOUBLE = 1, STX_Q_MUNCHAUSEN = 2, STX_Q_DQN_REG = 3 };
typedef struct StxQTdHyper {
  float gamma;
  float max_abs_reward;
  float huber_delta;
  float entropy_temperature;     /* Munchausen tau */
  float munchausen_coefficient;  /* Munchausen alpha */
  float clip_value_min;
  float regularizer_coeff;       /* DQN-Reg */
  int32_t reserved;
} StxQTdHyper;
int stx_q_td_loss_grads(int rule, const float* q_tm1, const float* q_t, const float* q_aux, const int32_t* action, const float* reward,
                        const uint8_t* done, const float* discount, int64_t M, int A, const StxQTdHyper* hyper, float* d_q, float* metrics,
                        float weight, void* scratch, void* stream);

/* Utility casts used by the bf16 path (obs / weight shadows). */
int stx_cast_f32_to_bf16(const float* src, void* dst, int64_t n, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* STX_H_ */
