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
  int32_t use_layer_norm;             /* bit STX_LN_TORSO: torso layers are Dense(no bias) + LayerNorm(eps 1e-6);
                                         bit STX_LN_FINAL: the last layer too, without activation (fp32 only) */
} StxMlp;
/* use_layer_norm bits.  STX_LN_FINAL is MLPTorso(use_layer_norm=True, activate_final=False) as DuelingQNetwork's branches use it
 * (stoix/networks/torso.py, dueling.py): the last Dense has no bias and is followed by a LayerNorm (scale, bias) and no activation;
 * its arena block is W, LayerNorm scale, LayerNorm bias like a torso layer's. */
#define STX_LN_TORSO 1
#define STX_LN_FINAL 2

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
/* Tuning hook for experiments, process-wide, for stx_gae_ppo_f32, stx_gae_generic_f32, stx_q_lambda_f32 and
 * stx_lambda_returns_f32.  code: 0 = the default selection; 2, 4, 8 = the scan kernel with that many env-quads
 * (4 envs each) per block; 416 = the scan kernel with 16 quads per block and two resident blocks per SM;
 * 500 / 501 = the TMA-pipelined kernel with 32 x 128 / 64 x 64 (envs x steps) tiles, PPO form only: where it
 * declines (E % 16, alignment) and for the other forms, the default selection runs.  Any non-zero code but
 * 500 / 501 keeps the TMA kernel off.  Returns STX_E_ARG for any other code, leaving the selection unchanged. */
int stx_gae_set_tuning(int code);
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

/* Profiling hook of the K3b launches: device buffer of [gridDim][8] int64 filled per CTA of K3b with
 * {2 + job, total cycles, cycles before the end of griddepcontrol.wait, globaltimer (ns) after it, globaltimer at exit,
 * chunks, -, -} (see stx_tc_ppo.cu g_prof_buf, scripts/k3b_jobs.py); NULL disables.  Synchronous (not for capture). */
int stx_tc_debug_set_prof_buffer(long long* buf);

/* Categorical head ops on logits (E, A) -- tfd.Categorical (stoix/networks/heads.py:41) as used at
 * ff_ppo.py:100-101.  If sample != 0: action = argmax_j(logits_j + Gumbel_j) (the first index on exact
 * ties), Gumbel_j = -log(-log u01(w)) of word j & 3 of Philox4x32-10 keyed by (seed lo, seed hi) with
 * counter (row lo, call lo, (call >> 32) ^ ((row >> 32) << 16) ^ (g << 24), "CATG" = 0x43415447),
 * call = offset + *dev_counter and group g = j / 4; else `action` is an input.  The group field has
 * 8 bits, so A <= 1024 (STX_E_SHAPE otherwise): beyond it the noise of group 256 would be group 0's.
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

/* Steps [0, T) of the synthetic env for all E envs in one launch over the whole GPU (its dynamics ignore the action):
 * exactly T calls of stx_synth_env_step with step = step + t + *dev_counter, written time-major: obs (T+1,E,D) bf16
 * [row 0 is the input, rows 1..T are written], next_obs (T,E,D) bf16, the rest (T,E); run_return / run_length carried.
 * D % 4 == 0, D <= 128. */
int stx_synth_env_trajectory(int64_t E, int D, int T, uint64_t seed, uint64_t step, const uint64_t* dev_counter, float p_term,
                             float p_trunc, void* obs, void* next_obs, float* reward, uint8_t* done, uint8_t* truncated,
                             float* ep_return, int32_t* ep_length, uint8_t* is_terminal, float* run_return, int32_t* run_length,
                             void* stream);

/* The actor side of the T-step scan of _env_step (ff_ppo.py:81-140) over observations that already exist (obs (T,E,D)
 * bf16, time-major, e.g. from stx_synth_env_trajectory; valid when the dynamics ignore the action, so no step waits for
 * the one before) in ONE persistent launch of min(T E / 64, max_ctas or one per SM) CTAs walking the 64-row tiles:
 * logits -> Gumbel-max action + log_prob (same Philox counters as stx_categorical with seed cat_seed, call = cat_offset +
 * t + *cat_counter), written (T,E).  E % 64 == 0; actor MLP [D <= 64 (multiple of 8), 256, 256, A <= 16], relu, no
 * LayerNorm, as for STX_PREC_BF16. */
int stx_tc_rollout_policy(const StxMlp* actor, const void* obs, int32_t* action, float* log_prob, int T, int64_t E,
                          uint64_t cat_seed, uint64_t cat_offset, const uint64_t* cat_counter, int max_ctas, void* stream);

/* The rollout's critic values on the bf16 tensor-core path: value[t] = critic(obs[t]), bootstrap_value[t] =
 * critic(next_obs[t]) for (T,E) rows, from one forward over obs[0..T] (next_obs[t] == obs[t+1] unless is_terminal[t])
 * and one over the next_obs rows where an episode ended.  Bit-identical to two full forward passes.  Obeys
 * stx_tc_set_forward_ctas.  ws: stx_tc_rollout_values_workspace_bytes(T, E, D) bytes. */
size_t stx_tc_rollout_values_workspace_bytes(int T, int64_t E, int D);
int stx_tc_rollout_values(const StxMlp* critic, const void* obs, const void* next_obs, const uint8_t* is_terminal, int T, int64_t E,
                          float* value, float* bootstrap_value, void* ws, size_t ws_bytes, void* stream);

/* Fused rollout of the synthetic env on the bf16 tensor-core path: stx_synth_env_trajectory followed by
 * stx_tc_rollout_policy on the same stream (env step = env_step + t + *env_counter).  Bit-identical to the per-step
 * path.  E % 64 == 0; actor as for stx_tc_rollout_policy. */
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

/* ------------------------------------------------------------------ distributional Q-learning: C51 and QR-DQN (fp32) ----
 * Head rows (M, A N) in the reference's layout: column a N + i is action a, atom / quantile i (reshape(-1, A, N), heads.py:251,288).
 * stx_dist_q_values: the expected Q of each action, q (M, A), that EpsilonGreedy acts on; one thread per (row, action), i in order:
 *   STX_DIST_CATEGORICAL: sum_i softmax(logits[a, :])_i atoms_i, the softmax in max-subtracted form (heads.py:252-253); atoms (N)
 *   STX_DIST_QUANTILE:    (sum_i q[a, i]) / N, jnp.mean (heads.py:289); atoms unused
 * stx_categorical_q_loss_grads: categorical_double_q_learning (utils/loss.py:81-103) under jax.grad, as ff_c51.py:159-188 calls it:
 *   r = clip(reward, +-max_abs_reward), d = (1 - done) gamma (or discount[m]), a* = first argmax of q_sel (M, A);
 *   p = softmax(logits_t[a*]); target_z = r + d atoms_t; t = rlax.categorical_l2_project(target_z, p, atoms_tm1);
 *   loss = -sum_j t_j log_softmax(logits_tm1[a])_j; d_logits = (softmax(logits_tm1[a]) sum_j t_j - t) / M in action a's N columns,
 *   0 in the others.  The projection is a gather: target atom i sums over the source atoms j = 0..N-1 in order (no atomics).
 * stx_quantile_q_loss_grads: quantile_q_learning + quantile_regression_loss (utils/loss.py:226-314), as ff_qr_dqn.py:159-202 calls
 *   it: a* = first argmax_a of (sum_i q_sel[a, i]) / N (q_sel nullable -> q_t, the reference's selector); target_j = r + d q_t[a*, j];
 *   delta_ij = target_j - q_tm1[a, i]; w_ij = |tau_i - 1[delta_ij < 0]| (delta = 0 weighs tau_i); loss = sum_i mean_j w_ij rho(delta_ij)
 *   with rho = rlax.huber_loss(., huber_delta) when huber_delta > 0, else |.|; d q_tm1[a, i] = -(sum_j w_ij rho'(delta_ij)) / (N M),
 *   rho' = clip(delta, -huber_delta, huber_delta), or for |.| JAX's select(delta >= 0, 1, -1) (slope +1 at 0); 0 in other columns.
 *   The row is spread over TPR threads (32 / 64 / 128 / 256 for N <= 32 / 64 / 128 / larger, 256 / TPR rows per CTA); thread i
 *   accumulates over j in order and the row's loss is a fixed-order tree, so two launches give the same bits.
 * Both losses: atoms_* / tau are read at row m as ptr + m ld_* (ld 0: one shared row); discount (nullable, per row) replaces
 *   (1 - done) gamma; loss_rows (nullable, (M)) receives each row's loss; metrics[0] += weight mean(loss).
 *   N <= STX_DIST_MAX_N (shared-memory bound), else STX_E_SHAPE.  scratch: stx_dist_q_scratch_bytes(M), zeroed once. */
enum { STX_DIST_CATEGORICAL = 0, STX_DIST_QUANTILE = 1 };
#define STX_DIST_MAX_N 2048
typedef struct StxDistQHyper {
  float gamma;
  float max_abs_reward;
  float huber_delta;  /* QR-DQN kappa; unused by C51 */
  int32_t reserved;
} StxDistQHyper;
size_t stx_dist_q_scratch_bytes(int64_t M);
int stx_dist_q_values(int kind, const float* head, int64_t M, int A, int N, const float* atoms, float* q, void* stream);
int stx_categorical_q_loss_grads(const float* logits_tm1, const float* logits_t, const float* q_sel, const float* atoms_tm1, int64_t ld_atoms_tm1,
                                 const float* atoms_t, int64_t ld_atoms_t, const int32_t* action, const float* reward, const uint8_t* done,
                                 const float* discount, int64_t M, int A, int N, const StxDistQHyper* hyper, float* d_logits, float* loss_rows,
                                 float* metrics, float weight, void* scratch, void* stream);
int stx_quantile_q_loss_grads(const float* q_tm1, const float* q_t, const float* q_sel, const float* tau, int64_t ld_tau, const int32_t* action,
                              const float* reward, const uint8_t* done, const float* discount, int64_t M, int A, int N, const StxDistQHyper* hyper,
                              float* d_q, float* loss_rows, float* metrics, float weight, void* scratch, void* stream);

/* stx_categorical_q_loss_grads with a per-row importance weight w (M) (ff_rainbow.py:196-204): d_logits of row m is scaled by w[m]
 * and metrics[0] += weight mean(w loss); loss_rows stays the unweighted loss (the new priorities).  w NULL is the unweighted
 * kernel itself, the same bits as stx_categorical_q_loss_grads. */
int stx_categorical_q_loss_grads_weighted(const float* logits_tm1, const float* logits_t, const float* q_sel, const float* atoms_tm1,
                                          int64_t ld_atoms_tm1, const float* atoms_t, int64_t ld_atoms_t, const int32_t* action, const float* reward,
                                          const uint8_t* done, const float* discount, const float* w, int64_t M, int A, int N,
                                          const StxDistQHyper* hyper, float* d_logits, float* loss_rows, float* metrics, float weight, void* scratch,
                                          void* stream);

/* ------------------------------------------------------------------ Rainbow: noisy layers, dueling head, prioritised ring (fp32) ----
 * Noisy layers (NoisyLinear, stoix/networks/layers.py:71-169): y = x (mu_w + sigma_w o eps_w) + mu_b + sigma_b o eps_b with factorised
 * noise eps_w = f(eps_in) f(eps_out)^T, eps_b = f(eps_out), f(z) = sign(z) sqrt|z| of standard normals, one draw per layer per call.
 *   The parameter arena holds every layer as kernel mu_w (in x out), bias mu_b (out), sigma_w (in x out), sigma_b (out), at
 *   StxNoisyLayer.param.  stx_noisy_weights writes the effective weights mu + sigma o eps of every layer into a dense StxMlp arena
 *   `eff` (at eff_w with row stride ld, the bias at eff_b), so stx_mlp_forward(_train) / stx_mlp_backward run unchanged on it; entries
 *   of `eff` no layer covers (the zero blocks of a block-diagonal layer) are never written.  Products in order, each rounded:
 *   eff_w = mu_w + sigma_w (f_in f_out), eff_b = mu_b + sigma_b f_out.
 *   noise: the f values, layer after layer f_in (in) then f_out (out) at StxNoisyLayer.noise.  draw != 0: noise element j is
 *   f(z), z = the first normal of normal2 over words (x, y) of Philox4x32-10 keyed by seed with counter (j, call, call >> 32,
 *   0x4E4F4953), call = offset + *dev_counter (nullable), and `noise` receives them; draw = 0: `noise` is an input.
 * stx_noisy_fold: the gradient of the parameters from the gradient of the effective arena under the same noise:
 *   d mu_w = g_w, d sigma_w = g_w (f_in f_out), d mu_b = g_b, d sigma_b = g_b f_out, written (overwrite) or added into `grad`
 *   (parameter layout).
 * stx_dueling_combine: head rows (M, N + A N) = (v | adv), column N + a N + i = adv[a, i]  ->  q_logits (M, A N),
 *   q[a, i] = (v[i] + adv[a, i]) - (sum_a adv[a, i]) / A, a in order (dueling.py:117).
 * stx_dueling_backward: d_head (M, N + A N) from d q_logits: dv[i] = sum_a dq[a, i], dadv[a, i] = dq[a, i] - (sum_a dq[a, i]) / A. */
#define STX_NOISY_MAX_LAYERS 8
typedef struct StxNoisyLayer {
  int64_t param;  /* first float of the layer (mu_w) in the parameter arena */
  int64_t eff_w;  /* first weight of the layer's block in the effective arena */
  int64_t eff_b;  /* first bias of the layer's block in the effective arena */
  int64_t noise;  /* first f_in of the layer in the noise buffer */
  int32_t in, out;
  int32_t ld;     /* row stride of the effective weight block (the width of its StxMlp layer) */
  int32_t reserved;
} StxNoisyLayer;
typedef struct StxNoisyNet {
  StxNoisyLayer layers[STX_NOISY_MAX_LAYERS];
  int32_t n_layers;
  int32_t reserved;
} StxNoisyNet;
int stx_noisy_weights(const StxNoisyNet* net, const float* params, float* eff, float* noise, int draw, uint64_t seed, uint64_t offset,
                      const uint64_t* dev_counter, void* stream);
int stx_noisy_fold(const StxNoisyNet* net, const float* eff_grad, const float* noise, float* grad, int overwrite, void* stream);
int stx_dueling_combine(const float* head, int64_t M, int A, int N, float* q_logits, void* stream);
int stx_dueling_backward(const float* d_q_logits, int64_t M, int A, int N, float* d_head, void* stream);

/* Prioritised trajectory ring -- fbx.make_prioritised_trajectory_buffer as ff_rainbow.py:433-442 builds it (add_batch_size = E,
 * sample_sequence_length = min_length_time_axis = n_step, period = 1, max_length_time_axis = L), with the n-step target of
 * ff_rainbow.py:222-246 computed while sampling.
 *   Storage is time-major: row (t, e) at t E + e, one write index for all envs.  Item i = e L + p is the sequence of env e
 *   starting at ring row p.  With write index w and c = min(rows written, L), the age of row p is (w - 1 - p) mod L and item
 *   (e, p) is valid iff n - 1 <= age(p) < c: its n rows are written and do not straddle the write head.  Invalid items have
 *   priority 0.  Priorities live in a sum tree of fan-out STX_PRIO_FANOUT over the E L leaves (leaf i = item i; level after
 *   level, stx_prio_tree_floats floats); a parent is the sum of its children in index order, rebuilt from them after every
 *   change (no atomics: two launches on the same state give the same bits).
 *   add:    T time rows of (T, E) batches at rows w .. w + T - 1 (mod L; only the last L if T > L), then the items starting
 *           at rows w - n + 1 .. w + T - 1 (at most L per env) are re-evaluated: valid ones get *max_priority, the others 0.
 *   sample: stratified: sample r takes v = ((r + u_r) total) / M (u_r = u_in[r], or u01 of word r & 3 of Philox (seed; r / 4,
 *           call, call >> 32, 0x5052494F), call = offset + *dev_counter) and descends from the root: at each node the children
 *           in order, entering the first with v < s (s its sum), else v -= s; if none (fp32 rounding left v at or past the node's
 *           sum), the last child with s > 0, and the last positive child at every level below, so the draw ends on the last
 *           positive item of that subtree.  The item is then within 64 h 2^-24 total of the fp64 inverse CDF (h the tree's
 *           levels; tests/prio_reference.py derives the bound).  With no valid item (total 0) every draw is item 0 with
 *           prob_out 0 and weight_out 1.  It writes
 *           the item's step-0 obs and action, step n-1 next_obs, the n-step reward G_0 (G = r_{n-1}; G_k = r_k + d_k G_{k+1},
 *           d_k = (1 - done_k) gamma, batch_discounted_returns with v = 0), done = any(done_0 .. done_{n-1}), idx_out (the item),
 *           prob_out = leaf / total and weight_out w = (1/p)^beta / max_batch (1/p)^beta, beta = linear schedule from beta0 to 1
 *           over beta_steps at *count (optax.linear_schedule: c = clip(count, 0, steps), beta = (beta0 - 1)(1 - c / steps) + 1;
 *           beta0 when steps <= 0; count nullable = 0).  obs / next_obs may be the two halves of one (2M, obs_dim) block.
 *   set_priorities: leaf idx[m] = priorities[m]^priority_exponent; for an index given twice the last occurrence in batch order
 *           wins (resolved in O(M) through `owner`); *max_priority = max(*max_priority, max_m priorities[m]^priority_exponent).
 *           Precondition, not checked on the device: every idx[m] is in [0, E L), as the sampler's idx_out is.
 *   scratch: stx_prio_scratch_bytes(), zeroed once. */
#define STX_PRIO_FANOUT 32
typedef struct StxReplayPrioritised {
  float* obs;            /* [L][E][obs_dim] */
  int32_t* action;       /* [L][E] */
  float* reward;         /* [L][E] */
  uint8_t* done;         /* [L][E]: timestep.last() */
  float* next_obs;       /* [L][E][obs_dim] */
  float* tree;           /* stx_prio_tree_floats(E L) floats, zero-initialised */
  int64_t* state;        /* device int64[2] = {write index, min(rows written, L)}, zero-initialised */
  float* max_priority;   /* device float[1]: max_recorded_priority, 1.0 initially */
  int64_t length;        /* L = max_length_time_axis */
  int32_t envs;          /* E = add_batch_size */
  int32_t obs_dim;
  int32_t n_step;        /* sample_sequence_length */
  float priority_exponent;
  int32_t* owner;        /* [E L] int32, -1 between calls: set_priorities' claim of each leaf */
} StxReplayPrioritised;
int64_t stx_prio_tree_floats(int64_t items);
size_t stx_prio_scratch_bytes(void);
int stx_replay_add_prioritised(const StxReplayPrioritised* rb, const float* obs, const int32_t* action, const float* reward, const uint8_t* done,
                               const float* next_obs, int T, void* stream);
int stx_replay_sample_prioritised(const StxReplayPrioritised* rb, int64_t M, uint64_t seed, uint64_t offset, const uint64_t* dev_counter,
                                  const float* u_in, const int32_t* count, float beta0, float beta_steps, float gamma, float* obs, float* next_obs,
                                  int32_t* action, float* reward, uint8_t* done, int32_t* idx_out, float* prob_out, float* weight_out, void* scratch,
                                  void* stream);
int stx_replay_set_priorities(const StxReplayPrioritised* rb, const int32_t* idx, const float* priorities, int64_t M, void* stream);

/* ------------------------------------------------------------------ V-MPO (fp32): stoix/systems/mpo/ff_vmpo.py, ff_vmpo_continuous.py ----
 * rlax.vmpo_loss (called at ff_vmpo.py:145-151, ff_vmpo_continuous.py:202-207) over the N = E (T-1) rows of one (device, update-batch)
 * shard, restated from rlax's published mpo_ops.py (tests/vmpo_oracle.py):
 * stx_vmpo_topk: tau = the k-th largest of adv[0..N) (k = int(0.5 N), rlax's top_k_fraction), by three radix passes over
 *   order-preserving uint32 keys (integer histograms: exact and deterministic).  With `mask` (nullable) a fourth launch writes
 *   mask[i] = (adv[i] >= tau) compared as floats (ties at tau are all selected, -0 == +0) and *count = K = |mask|.  N < 2 is
 *   refused with STX_E_SHAPE.  scratch: stx_vmpo_topk_scratch_bytes(), zeroed once.
 * stx_vmpo_loss_grads: two launches.  eta = softplus(duals[0]) + 1e-8, alpha_c = softplus(duals[1 + c]) + 1e-8; on the selected rows
 *   m = max A_i / eta, Z = sum exp(A_i / eta - m), w_i = exp(A_i / eta - m) / Z (0 elsewhere; stop-gradient), K = *count.
 *     L_pi = -sum_i w_i log pi(a_i | s_i)                                  (a sum, no 1/N)
 *     L_eta = eta (epsilon + log Z + m - log K)
 *     per KL column c: mean_kl_c = (1/N) sum_i kl_ic; L_kl = sum_c sg(alpha_c) mean_kl_c; L_alpha = sum_c alpha_c (eps_c - sg(mean_kl_c))
 *   KL columns: STX_VMPO_CATEGORICAL: one, KL(target || online) of the logits (eps_c = epsilon_alpha).  STX_VMPO_TANH_NORMAL on the
 *   pre-tanh Normals (loc | softplus(raw) + min_scale): kl_mean = KL(target || N(mu_online, sigma_target)) (eps_c = epsilon_alpha)
 *   and kl_stddev = KL(target || N(mu_target, sigma_online)) (eps_c = epsilon_stddev); per_dim: A columns of each (mean columns
 *   0..A-1, stddev columns A..2A-1), else one of each, summed over the dims.  The dual segment is [log_temperature, log_alpha_c
 *   for each column c].  Writes d_head = d (L_pi + L_kl) / d head (the tanh-Normal scale chained through sigmoid(raw)); d_value
 *   (value_rows rows, nullable when 0) = -(targets - value) / N on rows < N and 0 beyond (rlax.l2_loss(targets - v).mean());
 *   dual_grad[d] = weight g_d (overwrite) or += weight g_d with g_0 = (epsilon + log Z + m - log K - sum_i w_i A_i / eta)
 *   sigmoid(duals[0]), g_{1+c} = (eps_c - mean_kl_c) sigmoid(duals[1+c]); metrics[0..STX_VMPO_METRICS) += weight (L_pi, L_kl,
 *   L_alpha, L_eta, eta, mean alpha of the mean (or Categorical) columns, mean alpha of the stddev columns (0 for Categorical),
 *   mean advantage, value loss).  The whole-shard sums are fp64 in a fixed order.  scratch: stx_vmpo_loss_scratch_bytes(), zeroed once.
 * stx_vmpo_after_step: after the optimiser step: duals[0..n_dual) = max(-18, duals) (clip_categorical_mpo_params, discrete_loss.py:
 *   150-154; clip_dual_params, continuous_loss.py:142-147), and target[0..P) = online[0..P) when *count % period == 0
 *   (optax.periodic_update, ff_vmpo.py:266-274; *count = the actor segment's Adam count = learner_step_count).
 * stx_n_step_returns_f32: batch_n_step_bootstrapped_returns (stoix/utils/multistep.py:148-210) time-major, scalar lambda: targets
 *   start from v_t shifted by n and padded with v_t[T-1], then for i = n-1 .. 0: G_t = r + d ((1 - l) v + l G_t) at step t + i,
 *   with r = 0, d = 1, l = 1, v = v_t[T-1] past the end.  adv (nullable) = targets - v_tm1. */
#define STX_VMPO_CATEGORICAL 0
#define STX_VMPO_TANH_NORMAL 1
#define STX_VMPO_MAX_A 32
#define STX_VMPO_METRICS 9
typedef struct StxVmpoLoss {
  int32_t kind;               /* STX_VMPO_* */
  int32_t A;                  /* actions (Categorical) or action dims (tanh-Normal), 1..STX_VMPO_MAX_A */
  int32_t per_dim;            /* tanh-Normal: per_dim_constraining */
  int32_t overwrite;          /* 1: dual_grad = weight g; 0: += */
  int64_t N;                  /* rows of the shard, >= 2 */
  int64_t value_rows;         /* rows of d_value (the critic's T E rows) */
  const float* head;          /* (N, A) logits or (N, 2A) loc | raw scale of the online actor */
  const float* head_target;   /* same, target actor */
  const int32_t* action;      /* Categorical (N) */
  const float* action_cont;   /* tanh-Normal (N, A) */
  const float* adv;           /* (N) */
  const uint8_t* mask;        /* (N) selection of stx_vmpo_topk */
  const int32_t* count;       /* K */
  const float* value;         /* (N) v_tm1 of the current critic */
  const float* targets;       /* (N) value targets */
  const float* duals;         /* dual segment of the parameter arena */
  float* d_head;
  float* d_value;
  float* dual_grad;           /* dual segment of the gradient arena */
  float* metrics;
  float epsilon;              /* temperature constraint */
  float epsilon_alpha;        /* epsilon_policy (Categorical) / epsilon_mean */
  float epsilon_stddev;
  float weight;
  float minimum, maximum, min_scale;
  int32_t reserved;
} StxVmpoLoss;
size_t stx_vmpo_topk_scratch_bytes(void);
int stx_vmpo_topk(const float* adv, int64_t N, int64_t k, float* tau, uint8_t* mask, int32_t* count, void* scratch, void* stream);
size_t stx_vmpo_loss_scratch_bytes(void);
int stx_vmpo_loss_grads(const StxVmpoLoss* loss, void* scratch, void* stream);
int stx_vmpo_after_step(float* duals, int n_dual, const float* online, float* target, int64_t P, const int32_t* count, int period, void* stream);
int stx_n_step_returns_f32(const float* r_t, const float* discount_t, const float* v_t, const float* v_tm1, int T, int E, int n, float lambda_,
                           float* targets, float* adv, void* stream);

/* ------------------------------------------------------------------ MPO (fp32): stoix/systems/mpo/ff_mpo.py, ff_mpo_continuous.py ----
 * stx_replay_add_sequence / stx_replay_sample_sequence: fbx.make_trajectory_buffer as ff_mpo.py:539-546 builds it, with
 *   add_batch_size = E, max_length_time_axis = L, period = 1 (tests/mpo_oracle.py restates the rules).  Time-major ring of L x E
 *   rows, one write index for all envs: add writes batch row t to ring row (w + t) mod L (only the newest L rows of a longer batch),
 *   then w = (w + T) mod L and c = min(c + T, L) (state[0], state[1]; two launches).  sample draws, per sequence b, an env e uniform
 *   in [0, E) and k uniform in [0, c - S + 1): the S rows from start = (w - c + k) mod L, which never straddle the write head.  The
 *   draws are Philox(seed) at call offset + *dev_counter (nullable), or idx_in (B, 2) = (e, k) when given; idx_out (B, 2) = (e, start).
 *   Outputs are time-major (S, B): obs (S, B, D), action (S, B, act_words), reward, done, log_prob.  period != 1 -> STX_E_UNSUPPORTED.
 * stx_mpo_sample_actions: the target-Q input rows of M states in one launch, xq ((A + N + 1) M, D + A): block j < A holds
 *   [obs_i | one_hot(j)] (the actor loss evaluates every action, ff_mpo.py:189-197), block A + n holds [obs_i | one_hot(a_ni)] with a_ni
 *   drawn by inverse CDF from Categorical(logits_b[i]) (the bootstrap policy; its mode, the first maximum, when stochastic = 0, with
 *   N = 1), or act_in (N, M) when given, written to act_out (N, M, nullable); block A + N holds [obs_i | one_hot(action_i)].  The draw
 *   is the first j with u < the fp32 running sum of softmax_j, u = u01(word 0 of Philox(seed lo, seed hi; n M + i lo, n M + i hi,
 *   call lo, "MPOA" = 0x4D504F41 ^ call hi)), call = offset + *dev_counter; a u at or above the whole sum (fp32 rounding) takes the
 *   last action with positive fp32 probability.  Per state it also writes
 *   log_rho = log_softmax(logits_t)[action] - log_prob, r = clip(reward, +-max_abs_reward) and d = (1 - done) gamma.
 * stx_mpo_loss_grads: categorical_mpo_loss (discrete_loss.py:20-147) over M states, q (A, M): eta = softplus(duals[0]) + 1e-8,
 *   alpha = softplus(duals[1]) + 1e-8, u = q / eta + log_softmax(target), w = softmax(u), loss = mean CE(w, online) + alpha mean KL(target
 *   || online) + alpha (eps_policy - mean KL) + eta (eps + mean logsumexp u), with alpha held constant in the KL penalty and the KL held
 *   constant in the alpha loss.  d_head (M, A) = [(p_o - w) + alpha (p_o - p_t)] / M; dual_grad = weight * (dL/deta sigmoid(duals[0]),
 *   (eps_policy - mean KL) sigmoid(duals[1])), where dL/deta = eps + mean lse - mean(sum w q) / eta + mean(sum w (q - sum w q) log p_o) /
 *   eta^2 (the E-step weights carry eta's gradient into the cross-entropy, as jax.grad of the reference does).  metrics[0..13) += weight
 *   * (temperature, alpha, loss_temperature, loss_alpha, loss_policy, loss_kl, kl_nonparametric, entropy_online, entropy_target,
 *   kl_mean_rel, kl_q_rel, q_min, q_max); q_min / q_max are the reference's mean over actions of the min / max over states.  With
 *   q_boot (N, M): v = sum_n q_boot / N.  One launch; the whole-batch sums are fp64 in block order.
 * STX_MPO_TANH_NORMAL (ff_mpo_continuous.py, continuous_loss.py:26-303): the rows are NL draws a = shift + s tanh(loc + sigma eps) of
 *   the target policy ([obs | clip(a, minimum, maximum)], a itself kept in act_cont_out), N draws of the bootstrap policy (its mode
 *   shift + s tanh(loc) when stochastic = 0) and the clipped stored action; eps is Philox(seed, row, dim) at call *dev_counter, or
 *   eps_in.  log_rho sums tanh_normal_log_prob_given over the dims.  The loss: w = softmax_n(q / eta) held constant, loss_temperature
 *   = eta (eps + mean lse - log NL), the decoupled cross-entropies of N(loc_o, sigma_t) (gradient to loc) and N(loc_t, sigma_o)
 *   (gradient to the raw scale), and KL(target || fixed-stddev) / KL(target || fixed-mean) per dimension (C = A columns) or summed
 *   (C = 1), each with its alpha = softplus + 1e-8 held constant in the penalty.  dual_grad = weight * ((eps + mean lse - log NL -
 *   mean sum w q / eta) sigmoid(lt), (eps_c - mean KL_c) sigmoid(la_c)...); metrics[0..13) += weight * (temperature, alpha_mean,
 *   alpha_stddev, loss_temperature, loss_alpha_mean, loss_alpha_stddev, loss_policy_mean, loss_policy_stddev, loss_kl_mean,
 *   loss_kl_stddev, kl_mean, kl_stddev, kl_nonparametric) with the alphas and KLs averaged over their columns.
 * stx_retrace_f32: batch_general_off_policy_returns_from_q_and_v (multistep.py:210-311), time-major: q_t (K-1, E), v_t, r_t,
 *   discount_t, targets (K, E); the weights are c = lambda min(1, exp(log_rho)) (Retrace, log_rho (K-1, E)), or c_t (K-1, E) itself
 *   when c_t is given (log_rho and lambda are then not read).
 * stx_mpo_q_grad: dq (S, B) = (q - target) / (B (S-1)) on rows < S-1 and 0 on row S-1 (d of mean l2_loss); *metric += weight * that loss. */
#define STX_MPO_CATEGORICAL 0
#define STX_MPO_TANH_NORMAL 1
#define STX_MPO_MAX_A 32
#define STX_MPO_METRICS 14
typedef struct StxSeqRing {
  float* obs;                 /* (L, E, D) */
  void* action;               /* (L, E, act_words) 32-bit words: one int32 (Categorical) or A float32 (tanh-Normal) */
  float* reward;
  uint8_t* done;
  uint8_t* truncated;         /* stored, not read by the MPO targets */
  float* log_prob;            /* behaviour log-probability */
  int64_t* state;             /* [write row w, rows written c] */
  int64_t length;             /* L */
  int32_t envs, obs_dim, act_words, reserved;
} StxSeqRing;
typedef struct StxMpoRows {
  int32_t kind, A, N, D;      /* STX_MPO_*; actions (Categorical) or action dims (tanh-Normal); bootstrap rows per state; obs width */
  int64_t M;                  /* states */
  int32_t NL;                 /* actor-loss rows per state: A (Categorical) or num_samples (tanh-Normal) */
  int32_t stochastic;         /* 0: the mode of the bootstrap policy, N = 1 */
  uint64_t seed;
  const float* obs;           /* (M, D) */
  const float* logits_t;      /* (M, A) logits or (M, 2A) loc | raw scale of the target actor */
  const float* logits_b;      /* same, of the policy the bootstrap evaluates */
  const void* action;         /* (M) int32 or (M, A) float32 stored actions */
  const float* log_prob;      /* (M) behaviour log-probabilities */
  const float* reward;        /* (M) */
  const uint8_t* done;        /* (M) */
  const int32_t* act_in;      /* Categorical: (N, M) injected bootstrap actions, nullable */
  int32_t* act_out;           /* Categorical: (N, M), nullable */
  const float* eps_in;        /* tanh-Normal: (NL + N, M, A) injected standard normals, nullable */
  float* act_cont_out;        /* tanh-Normal: (NL, M, A) the unclipped actor-loss draws */
  float* xq;                  /* ((NL + N + 1) M, D + A) */
  float* log_rho;             /* (M) */
  float* r;                   /* (M) */
  float* d;                   /* (M) */
  float gamma, max_abs_reward;
  float minimum, maximum, min_scale;
  int32_t reserved;
} StxMpoRows;
typedef struct StxMpoLoss {
  int32_t kind, A, N, overwrite;
  int64_t M;
  int32_t NL, per_dim;        /* actor-loss rows per state (A for Categorical); tanh-Normal: per_dim_constraining */
  const float* head;          /* (M, A) online logits or (M, 2A) loc | raw scale */
  const float* head_target;   /* same, target actor */
  const float* q;             /* (NL, M) target Q of the actor-loss rows */
  const float* actions;       /* tanh-Normal: (NL, M, A) unclipped draws of the target policy */
  const float* q_boot;        /* (N, M) bootstrap target Q, nullable */
  const float* duals;         /* [log_temperature, log_alpha] or [log_temperature, log_alpha_mean (C), log_alpha_stddev (C)] */
  float* v;                   /* (M) mean of q_boot */
  float* d_head;
  float* dual_grad;
  float* metrics;
  float epsilon, epsilon_policy, epsilon_stddev, weight;   /* epsilon_policy is epsilon_mean for the tanh-Normal kind */
  float minimum, maximum, min_scale;
  int32_t reserved;
} StxMpoLoss;
int stx_replay_add_sequence(const StxSeqRing* rb, const float* obs, const void* action, const float* reward, const uint8_t* done,
                            const uint8_t* truncated, const float* log_prob, int T, void* stream);
int stx_replay_sample_sequence(const StxSeqRing* rb, int B, int S, int period, uint64_t seed, uint64_t offset, const uint64_t* dev_counter,
                               const int32_t* idx_in, int32_t* idx_out, float* obs, void* action, float* reward, uint8_t* done, float* log_prob,
                               void* stream);
int stx_mpo_sample_actions(const StxMpoRows* rows, uint64_t offset, const uint64_t* dev_counter, void* stream);
size_t stx_mpo_loss_scratch_bytes(void);
int stx_mpo_loss_grads(const StxMpoLoss* loss, void* scratch, void* stream);
int stx_retrace_f32(const float* q_t, const float* v_t, const float* r_t, const float* discount_t, const float* log_rho, const float* c_t, float lambda_,
                    int K, int E, float* targets, void* stream);
int stx_mpo_q_grad(const float* q, const float* targets, int S, int B, float* dq, float* metric, float weight, void* stream);

/* ------------------------------------------------------------------ R2D2 (fp32): stoix/systems/q_learning/rec_r2d2.py ----
 * Prioritised sequence ring with a period: fbx.make_prioritised_trajectory_buffer(max_size, min_length_time_axis = sample_sequence_length
 *   = S, add_batch_size = E, period = p, priority_exponent) as rec_r2d2.py:644-653 builds it (tests/r2d2_oracle.py restates the rule).
 *   Time-major storage, row (t, e) at t E + e, L = max_size // E time rows, one write index w for all envs, c = min(rows written, L).
 *   Item i = e K + k (K = L // p, k < K) is the sequence of env e starting at ring row k p; rows past K p start no item.  With
 *   age(row) = (w - 1 - row) mod L, the item is valid iff S - 1 <= age(k p) < c: its S rows are written and do not straddle the write
 *   head (Rainbow's rule with n replaced by S).  Rows hold obs, action (int32), reward, done, truncated and reset_hidden_state; the
 *   carry entering the step (RNNTransition.hstate; 2H for LSTM) is stored only at item-start rows, slot k E + e, since the loss reads
 *   only hstate[0] of a sequence.  Priorities live in the sum tree of Rainbow's ring (fan-out STX_PRIO_FANOUT over the E K leaves).
 *   add:    T rows at w .. w + T - 1 (mod L; only the newest L if T > L); then every item whose start row lies in w - S + 1 .. w + T - 1
 *           (mod L, at most L rows) is re-evaluated: valid ones get *max_priority, the others 0; every parent is rebuilt.
 *   sample: stratified as Rainbow's sampler, B strata: sequence b draws v = ((b + u_b) total) / B (u_b = u_in[b], or u01 of word b & 3
 *           of Philox(seed; b / 4, call, call >> 32, 0x5052494F), call = offset + *dev_counter) and descends the tree by Rainbow's
 *           rule (a level where no child takes v takes its last positive child, and so does every level below).  Outputs are
 *           time-major (S, B): obs (S, B, obs_dim), action, reward, done, reset; carry0 (B, carry_dim) = the stored carry of the item,
 *           idx_out (B) the item, prob_out (B) = leaf / total.  With no valid item (total 0: at the reference default, L = 97, S = 80,
 *           p = 40, the head often sits where no start row has S rows behind it) every draw is item 0 with prob 0; the loss's
 *           1e-6 keeps its importance weights finite, and set_priorities then gives that item a priority.  That flashbax does the
 *           same from an all-zero tree is inferred from its published rule, not checked against it.
 *   set_priorities: Rainbow's: leaf idx[m] = priorities[m]^priority_exponent, the last of duplicate indices wins, ancestors rebuilt,
 *           *max_priority raised.  Precondition, not checked on the device: every idx[m] is in [0, E K).
 * stx_r2d2_loss_grads: rlax.transformed_n_step_q_learning with SIGNED_HYPERBOLIC_PAIR (rec_r2d2.py:331-384) over a learn window of T
 *   rows of B sequences, q / q_target (T, B, A): a*_t = argmax_a q[t] (first maximum) and v_t = q_target[t, a*_t] for t = 1 .. T-1;
 *   r_t = clip(reward, +-max_abs_reward), d_t = gamma (1 - done) (truncation does not cut the return, as in the reference), for
 *   t < T-1.  Over seq = T - 1: targets_t = v[min(t + n - 1, seq - 1)], then for i = n-1 .. 0: targets_t = h(r_{t+i} + d_{t+i}
 *   h^-1(targets_t)) with r = 0 and d = 1 past the window; td_t = targets_t - q[t, action_t].  h(x) = sign(x)(sqrt(|x|+1) - 1) + eps x,
 *   h^-1(x) = sign(x)(z^2 - 1), z = (sqrt(1 + 4 eps (eps + 1 + |x|)) - 1) / (2 eps), both evaluated without cancellation near 0
 *   (stx_r2d2_value_transform exposes them).  loss_b = 0.5 sum_t td^2; w_b = (1 / (prob_b + 1e-6))^beta / max_b', beta =
 *   optax.linear_schedule(beta0 -> 1 over beta_steps) at *count.  d_q (T, B, A) = -w_b td_t / B at (t, action_t) for t < T-1, 0
 *   elsewhere; priorities_b = eta max_t |td| + (1 - eta) mean_t |td|; metrics[0..6) += weight (mean_b w_b loss_b, mean q, max_b
 *   priority, mean_b priority, mean_b max_t |td|, mean_b mean_t |td|); td (seq, B, nullable) receives the TD errors.  One launch;
 *   the batch sums are fp64 in sequence order.  scratch: stx_r2d2_loss_scratch_bytes(B), zeroed once.
 * stx_dueling_q: q = v + (adv - mean_a adv) (rec_r2d2's DuelingQNetwork order) with v = *value, the value branch's final LayerNorm
 *   bias: that LayerNorm normalises a single element, so its output is exactly its bias.  stx_dueling_q_backward: d_adv = dq - mean_a dq;
 *   *d_value = weight sum dq (overwrite) or += (rows then threads in a fixed order). */
#define STX_R2D2_METRICS 6
typedef struct StxR2d2Ring {
  float* obs;                 /* (L, E, obs_dim) */
  int32_t* action;            /* (L, E) */
  float* reward;
  uint8_t* done;
  uint8_t* truncated;
  uint8_t* reset;             /* reset_hidden_state */
  float* carry;               /* (L // period, E, carry_dim) */
  float* tree;                /* stx_r2d2_tree_floats() floats, zero-initialised */
  int64_t* state;             /* {write index, min(rows written, L)} */
  float* max_priority;        /* 1.0 initially */
  int32_t* owner;             /* (E (L // period)) int32, -1 between calls */
  int64_t length;             /* L */
  int32_t envs, obs_dim, carry_dim, seq_len, period;
  float priority_exponent;
} StxR2d2Ring;
typedef struct StxR2d2Loss {
  int32_t T, B, A, n;         /* learn rows, sequences, actions, n-step */
  const float* q;             /* (T, B, A) online Q */
  const float* q_target;      /* (T, B, A) target Q */
  const int32_t* action;      /* (T, B) */
  const float* reward;        /* (T, B) */
  const uint8_t* done;        /* (T, B) */
  const float* prob;          /* (B) */
  const int32_t* count;       /* Adam count word, nullable = 0 */
  float* d_q;                 /* (T, B, A) */
  float* priorities;          /* (B) */
  float* metrics;             /* STX_R2D2_METRICS */
  float* td;                  /* (T - 1, B), nullable */
  float gamma, max_abs_reward, eta, tx_eps;
  float beta0, beta_steps, weight;
  int32_t reserved;
} StxR2d2Loss;
int64_t stx_r2d2_tree_floats(const StxR2d2Ring* rb);
int stx_r2d2_ring_add(const StxR2d2Ring* rb, const float* obs, const int32_t* action, const float* reward, const uint8_t* done,
                      const uint8_t* truncated, const uint8_t* reset, const float* carry, int T, void* stream);
int stx_r2d2_ring_sample(const StxR2d2Ring* rb, int B, uint64_t seed, uint64_t offset, const uint64_t* dev_counter, const float* u_in, float* obs,
                         int32_t* action, float* reward, uint8_t* done, uint8_t* reset, float* carry0, int32_t* idx_out, float* prob_out, void* stream);
int stx_r2d2_ring_set_priorities(const StxR2d2Ring* rb, const int32_t* idx, const float* priorities, int64_t M, void* stream);
int stx_r2d2_value_transform(const float* x, int64_t n, int inverse, float eps, float* out, void* stream);
size_t stx_r2d2_loss_scratch_bytes(int B);
int stx_r2d2_loss_grads(const StxR2d2Loss* loss, void* scratch, void* stream);
int stx_dueling_q(const float* adv, const float* value, int64_t M, int A, float* q, void* stream);
int stx_dueling_q_backward(const float* d_q, int64_t M, int A, float* d_adv, float* d_value, float weight, int overwrite, void* stream);

/* ------------------------------------------------------------------ IMPALA: V-trace (fp32) ----------------------------
 * The learner step of stoix/systems/impala/sebulba/ff_impala.py:358-566 on one learner batch of T + 1 time rows and E env columns.
 *
 * stx_reward_stats: mean and population std (jnp.mean / jnp.std) of the rewards r[t * ld + e], t < T, e < E, in fp64 in a fixed
 *   order, written as float32 stats[0] = mean, stats[1] = std (ff_impala.py:389-395).  One launch.
 * stx_clip_rmsprop_step: stx_clip_adam_step with optax.rmsprop(lr) at its defaults (ff_impala.py:754-766): no centring, no momentum,
 *   no bias correction, initial_scale 0, eps inside the square root:
 *     nu = (1 - decay) g^2 + decay nu ;  p = p - lr g / sqrt(nu + eps)
 *   with decay = hyper->b2 (hyper->b1 is not read) and the clip, learning-rate schedule and per-segment counts of stx_clip_adam_step.
 *   Reads and writes nu only.  hyper->prenorm must be 0.
 * stx_vtrace_loss_grads: one minibatch = one column block of Em envs, in one launch.  Per column, time-major (row t * Em + j):
 *     logp = log_softmax(logits);  rho = exp(logp[a] - log_prob_b);  H = -sum p logp
 *     r = reward (or reward_scale (reward - mean) / (std + reward_eps) with reward_stats);  d = gamma (1 - done)  (truncation ends the
 *     trace like termination, as the reference does)
 *   rlax.vtrace_td_error_and_advantage with v_tm1 = values[t], v_t = values[t + 1]:
 *     c = lambda min(1, rho);  delta = min(clip_rho, rho) (r + d v_t - v_tm1);  acc_t = delta_t + d_t c_t acc_{t+1} (acc_T = 0)
 *     vs = acc + v_tm1;  errors = vs - v_tm1
 *     q_t = r_t + d_t (lambda vs_{t+1} + (1 - lambda) v_tm1_{t+1})  (t < T - 1),  q_{T-1} = r + d v_t
 *     pg_adv = min(clip_pg_rho, rho) (q - v_tm1)
 *   losses (sums, not means): value_loss = 0.5 sum errors^2 (the critic loss is vf_coef value_loss, gradient only through v_tm1),
 *   actor_loss = -sum pg_adv logp[a] (pg_adv constant), entropy = sum H (the actor loss subtracts ent_coef entropy):
 *     d_logits_k = -pg_adv (1[k = a] - p_k) + ent_coef p_k (logp_k + H);  d_value[t] = -vf_coef errors_t, d_value[T] = 0
 *   metrics (STX_VTRACE_METRICS, overwritten): actor_loss, entropy, value_loss, mean q_estimate, mean pg_advantage.
 *   Any T >= 1, Em >= 1, A >= 1.  action / log_prob_b / reward / done: element (t, j) at [t * ld + j] (a column block of the learner
 *   batch).  scratch: stx_vtrace_loss_scratch_bytes(), zeroed once. */
#define STX_VTRACE_METRICS 5
typedef struct StxVtraceLoss {
  const float* logits;        /* (T * Em, A) */
  const float* values;        /* ((T + 1) * Em) */
  const int32_t* action;      /* [t * ld + j], t < T */
  const float* log_prob_b;    /* behaviour log-probabilities, [t * ld + j] */
  const float* reward;        /* [t * ld + j] */
  const uint8_t* done;        /* [t * ld + j] */
  const float* reward_stats;  /* nullable: {mean, std} of stx_reward_stats, applied to the rewards as they are loaded */
  float* d_logits;            /* (T * Em, A) */
  float* d_value;             /* ((T + 1) * Em) */
  float* metrics;             /* STX_VTRACE_METRICS */
  int64_t ld;                 /* row stride of action / log_prob_b / reward / done, >= Em */
  int32_t T, Em, A;
  float gamma, lambda_, clip_rho, clip_pg_rho, ent_coef, vf_coef, reward_scale, reward_eps;
} StxVtraceLoss;
int stx_reward_stats(const float* reward, int T, int E, int64_t ld, float* stats, void* stream);
int stx_clip_rmsprop_step(float* param_arena, const float* grad_arena, float* nu, int32_t* counts, const StxAdamSeg* segs, int nseg,
                          const StxAdamHyper* hyper, void* params_bf16, float* gnorm_out, void* scratch, void* stream);
size_t stx_vtrace_loss_scratch_bytes(void);
int stx_vtrace_loss_grads(const StxVtraceLoss* loss, void* scratch, void* stream);

/* Utility casts used by the bf16 path (obs / weight shadows). */
int stx_cast_f32_to_bf16(const float* src, void* dst, int64_t n, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* STX_H_ */
