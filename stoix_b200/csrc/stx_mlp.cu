// K1 (fp32 path) MLP forward / backward, the categorical sampler, and the networks of the fp32 PPO minibatch (whose losses live
// in stx_ppo_fp32.cu).  The bf16 wgmma implementations live in stx_tc_mlp.cu and are dispatched from here by precision.
#include "stx_common.cuh"
#include "stx_ppo_halves.cuh"
#include "stx_simt_gemm.cuh"

namespace stx {

// implemented in stx_tc_mlp.cu
size_t tc_mlp_forward_workspace_bytes(const StxMlp* mlp, int64_t M);
int tc_mlp_forward(const StxMlp* mlp, const void* x, int64_t ldx, const int32_t* row_idx, int64_t M,
                   float* out, void* ws, size_t ws_bytes, cudaStream_t st);
size_t tc_ppo_workspace_bytes(const StxMlp* actor, const StxMlp* critic, int64_t mb);

namespace {

inline size_t align_up(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }

int check_mlp(const StxMlp* m, const char* who) {
  STX_REQUIRE(m != nullptr, STX_E_ARG, "%s: null StxMlp", who);
  STX_REQUIRE(m->n_layers >= 1 && m->n_layers <= STX_MAX_LAYERS, STX_E_SHAPE, "%s: n_layers=%d", who, m->n_layers);
  for (int i = 0; i <= m->n_layers; ++i)
    STX_REQUIRE(m->sizes[i] > 0, STX_E_SHAPE, "%s: sizes[%d]=%d", who, i, m->sizes[i]);
  STX_REQUIRE(m->params != nullptr, STX_E_ARG, "%s: null params", who);
  STX_REQUIRE(m->activation >= STX_ACT_RELU && m->activation <= STX_ACT_IDENTITY, STX_E_ARG, "%s: activation=%d", who, m->activation);
  if (m->use_layer_norm)
    for (int i = 1; i < m->n_layers; ++i)
      STX_REQUIRE(m->sizes[i] <= 32 * simt::kLnMaxCols, STX_E_SHAPE, "%s: LayerNorm width %d > %d", who, m->sizes[i], 32 * simt::kLnMaxCols);
  return STX_OK;
}

inline bool layer_has_ln(const StxMlp* m, int i) { return m->use_layer_norm && i < m->n_layers - 1; }

int max_width(const StxMlp* m) {
  int w = 0;
  for (int i = 1; i <= m->n_layers; ++i) w = m->sizes[i] > w ? m->sizes[i] : w;
  return w;
}

// offsets of W_i and b_i inside a network arena; LayerNorm torso layers: boff = LayerNorm scale, +sizes[i+1] = LayerNorm bias
void layer_offsets(const StxMlp* m, int64_t* woff, int64_t* boff) {
  int64_t o = 0;
  for (int i = 0; i < m->n_layers; ++i) {
    woff[i] = o;
    o += (int64_t)m->sizes[i] * m->sizes[i + 1];
    boff[i] = o;
    o += (layer_has_ln(m, i) ? 2 : 1) * (int64_t)m->sizes[i + 1];
  }
}

// Forward through all layers.  For the torso layers i = 1..n-1: acts[i] (nullable: inference) receive the PRE-activation Dense
// outputs U_i (M x sizes[i]), hacts[i] the layer outputs H_i = f(U_i) / f(LN(U_i)) the next layer multiplies, stats[i] (nullable)
// the LayerNorm (mean, rstd); the head output goes to `out`.  x may be gathered through row_idx.
int simt_forward(const StxMlp* m, const float* x, int64_t ldx, const int32_t* row_idx, int64_t M,
                 float* const* acts, float* const* hacts, float* const* stats, float* out, cudaStream_t st) {
  int64_t woff[STX_MAX_LAYERS], boff[STX_MAX_LAYERS];
  layer_offsets(m, woff, boff);
  const float* in = x;
  int64_t ld = ldx;
  const int32_t* ridx = row_idx;
  for (int i = 0; i < m->n_layers; ++i) {
    const bool last = (i == m->n_layers - 1), ln = layer_has_ln(m, i);
    simt::GemmArgs g{};
    g.A = in, g.lda = ld, g.rowidx = ridx;
    g.mask_act = -1;
    g.B = m->params + woff[i];
    g.bias = ln ? nullptr : m->params + boff[i];  // torso.py:26: use_bias = not use_layer_norm
    g.M = M, g.N = m->sizes[i + 1], g.K = m->sizes[i];
    if (last) {
      g.C = out;
    } else if (ln) {   // U now; H = f(LN(U)) by ln_apply_kernel (inference: in place on the H buffer)
      g.C = acts[i + 1] ? acts[i + 1] : hacts[i + 1];
    } else {           // MLPTorso activate_final=True: the head sees f(.) too
      g.C = acts[i + 1];
      g.C_act = hacts[i + 1], g.c_act = m->activation;
    }
    STX_CUDA_OK(simt::launch_gemm<simt::FWD>(g, 1, st));
    if (ln) {
      const float* gamma = m->params + boff[i];
      simt::ln_apply_kernel<<<(unsigned)((M + 7) / 8), 256, 0, st>>>(g.C, M, g.N, gamma, gamma + g.N, m->activation, stats ? stats[i + 1] : nullptr,
                                                                     hacts[i + 1]);
      STX_LAUNCH_OK();
    }
    in = last ? out : hacts[i + 1], ld = g.N, ridx = nullptr;
  }
  return STX_OK;
}

// ---- categorical head --------------------------------------------------------------------
__global__ void categorical_kernel(const float* __restrict__ logits, int64_t E, int A, int sample,
                                   uint64_t seed, uint64_t offset, const uint64_t* __restrict__ dev_counter,
                                   int32_t* __restrict__ action,
                                   float* __restrict__ log_prob, float* __restrict__ entropy) {
  const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (e >= E) return;
  const float* z = logits + e * A;
  float zmax = -INFINITY;
  for (int j = 0; j < A; ++j) zmax = fmaxf(zmax, z[j]);
  float se = 0.f;
  for (int j = 0; j < A; ++j) se += expf(z[j] - zmax);
  const float lse = zmax + logf(se);
  int a;
  if (sample) {
    // Gumbel-max (jax.random.categorical): argmax_j z_j - log(-log u_j)
    const uint64_t call = offset + (dev_counter ? *dev_counter : 0ull);
    const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
    const uint32_t c2 = (uint32_t)(call >> 32) ^ ((uint32_t)((uint64_t)e >> 32) << 16);
    float best = -INFINITY;
    a = 0;
    for (int j0 = 0; j0 < A; j0 += 4) {
      const uint4 r = Philox::rand4(make_uint4((uint32_t)e, (uint32_t)call, c2 ^ ((uint32_t)(j0 >> 2) << 24), 0x43415447u), key);
      const uint32_t w[4] = {r.x, r.y, r.z, r.w};
      for (int k = 0; k < 4 && j0 + k < A; ++k) {
        const float gmb = -logf(-logf(u01(w[k])));
        const float s = z[j0 + k] + gmb;
        if (s > best) best = s, a = j0 + k;
      }
    }
    action[e] = a;
  } else {
    a = action[e];
  }
  log_prob[e] = z[a] - lse;
  if (entropy) {
    float h = 0.f;
    for (int j = 0; j < A; ++j) {
      const float lp = z[j] - lse;
      h -= expf(lp) * lp;
    }
    entropy[e] = h;
  }
}

// ---- epsilon-greedy head (PQN) -------------------------------------------------------------
// distrax.EpsilonGreedy(preferences=q, epsilon): (1 - eps) uniform over the argmax set + eps / A.  Integer arithmetic on two
// Philox words, so an oracle reproduces every action bit for bit (layout in include/stx.h).  The schedule is evaluated with
// explicitly rounded fp32 operations (no contraction), so it equals a literal fp32 evaluation.
__device__ __forceinline__ float epsilon_at(const StxEpsilonSchedule& s, int32_t update_no) {
  if (!s.decay) return s.end_value;
  if (!(s.transition_steps > 0.f)) return s.init_value;   // optax.polynomial_schedule with transition_steps <= 0
  const float c = fminf(fmaxf((float)update_no, 0.f), s.transition_steps);
  const float frac = __fsub_rn(1.0f, __fdiv_rn(c, s.transition_steps));
  return __fadd_rn(__fmul_rn(__fsub_rn(s.init_value, s.end_value), frac), s.end_value);
}

__global__ void epsilon_greedy_kernel(const float* __restrict__ q, int64_t E, int A, int mode, uint64_t seed, uint64_t offset,
                                      const uint64_t* __restrict__ dev_counter, const int32_t* __restrict__ count, StxEpsilonSchedule sched,
                                      int32_t* __restrict__ action, float* __restrict__ eps_out, int32_t* __restrict__ upd_out) {
  const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (e >= E) return;
  const float* z = q + e * A;
  float zmax = -INFINITY;
  int first = 0, n_ties = 0;
  for (int j = 0; j < A; ++j) {
    const float v = z[j];
    if (v > zmax) zmax = v, first = j, n_ties = 1;
    else if (v == zmax) ++n_ties;
  }
  const int32_t upd = (count ? *count : 0) / sched.steps_per_update;   // ff_pqn.py:72: count // (epochs * num_minibatches)
  const float eps = epsilon_at(sched, upd);
  if (eps_out) eps_out[e] = eps;
  if (upd_out) upd_out[e] = upd;
  if (mode) {
    action[e] = first;
    return;
  }
  const uint64_t call = offset + (dev_counter ? *dev_counter : 0ull);
  const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
  const uint32_t c2 = (uint32_t)(call >> 32) ^ ((uint32_t)((uint64_t)e >> 32) << 16);
  const uint4 r = Philox::rand4(make_uint4((uint32_t)e, (uint32_t)call, c2, 0x45475259u), key);
  // (w0 >> 8) * 2^-24 is exact and below 1: eps = 1 always explores, eps = 0 never does
  if ((float)(r.x >> 8) * (1.0f / 16777216.0f) < eps) {
    action[e] = (int32_t)(((uint64_t)r.y * (uint64_t)A) >> 32);
    return;
  }
  const int pick = (int)(((uint64_t)r.y * (uint64_t)n_ties) >> 32);   // the pick-th maximal index
  int a = first;
  for (int j = first, seen = 0; j < A; ++j)
    if (z[j] == zmax && seen++ == pick) {
      a = j;
      break;
    }
  action[e] = a;
}

// ---- fp32 PPO minibatch: workspace carving -------------------------------------------------
struct SimtPpoWs {
  float* acts[STX_MAX_LAYERS + 1];  // pre-activation Dense outputs U_i of the torso layers, index 1..n-1
  float* hacts[STX_MAX_LAYERS + 1]; // layer outputs H_i = f(U_i) / f(LN(U_i)): the operand of the next layer's GEMMs
  float* stats[STX_MAX_LAYERS + 1]; // LayerNorm torsos: per-row (mean, rstd) of acts[i]
  float* ln_part;                   // LayerNorm backward: [blocks][2 * width] column-sum partials
  int ln_blocks, ln_rows;
  float* head;                      // logits or value (mb x head)
  float* dhead;                     // d logits / d value
  float* dbuf[2];                   // ping-pong d(hidden)
  float* partials;                  // [splits][net params]
  double* loss_partials;
  unsigned int* counter;
  int splits;
  size_t bytes;
};

// Split-M factor of the weight-gradient GEMMs.  512 rows per split (at most 32) suits wide layers; a network whose thinnest layer
// has only a few 64x64 output tiles (the 32 -> 128 -> 384 pre-torso of the recurrent nets: 2 tiles) would leave most SMs idle and
// make every CTA walk thousands of rows, so such networks get as many splits as it takes to fill the GPU twice (>= 256 rows each).
int pick_splits(const StxMlp* m, int64_t mb) {
  int64_t s = mb / 512;
  if (s < 1) s = 1;
  if (s > 32) s = 32;
  int64_t min_tiles = 1 << 30;
  for (int i = 0; i < m->n_layers; ++i) {
    const int64_t tiles = (int64_t)((m->sizes[i] + 63) / 64) * ((m->sizes[i + 1] + 63) / 64);
    if (tiles < min_tiles) min_tiles = tiles;
  }
  int64_t want = (2 * kNumSMs + min_tiles - 1) / min_tiles;
  if (want > mb / 256) want = mb / 256;
  if (want > 128) want = 128;
  return (int)(s > want ? s : want);
}

SimtPpoWs carve(const StxMlp* m, int64_t mb, char* base) {
  SimtPpoWs w{};
  size_t o = 0;
  auto take = [&](size_t bytes) {
    char* p = base ? base + o : nullptr;
    o += align_up(bytes);
    return p;
  };
  // counter must stay zero between calls: lives first so callers can zero the head of the workspace once
  w.counter = reinterpret_cast<unsigned int*>(take(256));
  const int mw = max_width(m);
  for (int i = 1; i < m->n_layers; ++i) w.acts[i] = reinterpret_cast<float*>(take((size_t)mb * m->sizes[i] * 4));
  for (int i = 1; i < m->n_layers; ++i) w.hacts[i] = reinterpret_cast<float*>(take((size_t)mb * m->sizes[i] * 4));
  for (int i = 1; i < m->n_layers; ++i) w.stats[i] = m->use_layer_norm ? reinterpret_cast<float*>(take((size_t)mb * 2 * 4)) : nullptr;
  // rows per block of ln_backward_kernel: about two blocks per SM, a whole number of rows per warp
  w.ln_rows = (int)(((mb + 295) / 296 + simt::kLnWarps - 1) / simt::kLnWarps * simt::kLnWarps);
  if (w.ln_rows > 128) w.ln_rows = 128;
  w.ln_blocks = (int)((mb + w.ln_rows - 1) / w.ln_rows);
  w.ln_part = m->use_layer_norm ? reinterpret_cast<float*>(take((size_t)w.ln_blocks * 2 * mw * 4)) : nullptr;
  w.head = reinterpret_cast<float*>(take((size_t)mb * m->sizes[m->n_layers] * 4));
  w.dhead = reinterpret_cast<float*>(take((size_t)mb * m->sizes[m->n_layers] * 4));
  w.dbuf[0] = reinterpret_cast<float*>(take((size_t)mb * mw * 4));
  w.dbuf[1] = reinterpret_cast<float*>(take((size_t)mb * mw * 4));
  w.splits = pick_splits(m, mb);
  w.partials = reinterpret_cast<float*>(take((size_t)w.splits * stx_mlp_param_count(m) * 4));
  w.loss_partials = reinterpret_cast<double*>(take(((size_t)(mb + 255) / 256) * 6 * 8));
  w.bytes = o;
  return w;
}

// backward of one network given d(head) in ws.dhead; accumulates grad_weight * grads into net_grad (nullptr: parameter
// gradients are not wanted); dx (nullable, mb x sizes[0], dense): receives d(loss)/d(input).
int simt_backward(const StxMlp* m, const float* x, int64_t ldx, const int32_t* row_idx, int64_t mb,
                  const SimtPpoWs& ws, float grad_weight, float* net_grad, int overwrite, cudaStream_t st, float* dx = nullptr) {
  int64_t woff[STX_MAX_LAYERS], boff[STX_MAX_LAYERS];
  layer_offsets(m, woff, boff);
  const int64_t np = stx_mlp_param_count(m);
  const int64_t rows_per_split = (mb + ws.splits - 1) / ws.splits;
  const float* dY = ws.dhead;
  int pp = 0;
  for (int i = m->n_layers - 1; i >= 0; --i) {
    const int nin = m->sizes[i], nout = m->sizes[i + 1];
    // dW_i, db_i partials: input of layer i is x (gathered) for i == 0, else the stored layer output H_i
    simt::GemmArgs g{};
    g.A = (i == 0) ? x : ws.hacts[i];
    g.lda = (i == 0) ? ldx : nin;
    g.rowidx = (i == 0) ? row_idx : nullptr;
    g.mask_act = -1;
    g.B = dY;
    g.C = ws.partials + woff[i];
    g.dbias = layer_has_ln(m, i) ? nullptr : ws.partials + boff[i];  // LayerNorm layers: Dense has no bias (scale / bias below)
    g.M = mb, g.N = nout, g.K = nin;
    g.rows_per_split = rows_per_split;
    g.part_stride = np, g.dbias_stride = np;
    if (net_grad != nullptr) STX_CUDA_OK(simt::launch_gemm<simt::DW>(g, ws.splits, st));
    if (i == 0 && dx != nullptr) {  // d(input) = dY @ W_0^T (no activation in front of the first Dense)
      simt::GemmArgs d{};
      d.A = dY, d.lda = nout, d.mask_act = -1;
      d.B = m->params + woff[0];
      d.C = dx;
      d.M = mb, d.N = nin, d.K = nout;
      STX_CUDA_OK(simt::launch_gemm<simt::DX>(d, 1, st));
    }
    if (i > 0) {
      // d(U_{i-1}) from dY: through the Dense (dY @ W_i^T), the activation and, for LayerNorm torsos, the normalisation
      const bool ln = layer_has_ln(m, i - 1);
      simt::GemmArgs d{};
      d.A = dY, d.lda = nout;
      d.B = m->params + woff[i];
      d.C = ws.dbuf[pp];
      d.mask = ln ? nullptr : ws.acts[i];
      d.mask_act = ln ? -1 : m->activation;
      d.M = mb, d.N = nin, d.K = nout;
      STX_CUDA_OK(simt::launch_gemm<simt::DX>(d, 1, st));
      if (ln) {
        const float* gamma = m->params + boff[i - 1];
        STX_CUDA_OK(simt::launch_ln_backward(ws.dbuf[pp], ws.acts[i], ws.stats[i], gamma, gamma + nin, m->activation, mb, nin, ws.ln_rows,
                                             ws.ln_blocks, ws.ln_part, st));
        STX_LAUNCH_OK();
        // d(scale | bias) of layer i-1: fixed-order sum over the blocks, straight into the gradient arena
        if (net_grad != nullptr)
          simt::reduce_partials_kernel<<<(unsigned)((2 * nin + 255) / 256), 256, 0, st>>>(ws.ln_part, ws.ln_blocks, 2 * (int64_t)nin, 2 * (int64_t)nin,
                                                                                        grad_weight, net_grad + boff[i - 1], overwrite);
        STX_LAUNCH_OK();
      }
      dY = ws.dbuf[pp];
      pp ^= 1;
    }
  }
  // fixed-order sum of the split-M partials: W_i and, for layers with a Dense bias, b_i (LayerNorm scale / bias were reduced above)
  for (int i = 0; i < m->n_layers && net_grad != nullptr; ++i) {
    const int64_t n = (int64_t)m->sizes[i] * m->sizes[i + 1] + (layer_has_ln(m, i) ? 0 : m->sizes[i + 1]);
    simt::reduce_partials_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(ws.partials + woff[i], ws.splits, np, n, grad_weight,
                                                                              net_grad + woff[i], overwrite);
    STX_LAUNCH_OK();
  }
  return STX_OK;
}

}  // namespace

// ---- the networks of the fp32 PPO minibatch (stx_ppo_fp32.cu) ----
// Both carve `workspace` the same way, so one stx_ppo_workspace_bytes() workspace serves either net.
int simt_check_mlp(const StxMlp* m, const char* who) { return check_mlp(m, who); }

int simt_net_forward(const StxMlp* m, const float* x, int64_t ldx, const int32_t* idx, int64_t mb, void* workspace, SimtHeadBufs* out,
                     cudaStream_t st) {
  SimtPpoWs ws = carve(m, mb, reinterpret_cast<char*>(workspace));
  out->head = ws.head, out->dhead = ws.dhead, out->loss_partials = ws.loss_partials, out->counter = ws.counter;
  return simt_forward(m, x, ldx, idx, mb, ws.acts, ws.hacts, ws.stats, ws.head, st);
}

int simt_net_backward(const StxMlp* m, const float* x, int64_t ldx, const int32_t* idx, int64_t mb, void* workspace, float grad_weight,
                      float* net_grad, int overwrite, cudaStream_t st) {
  SimtPpoWs ws = carve(m, mb, reinterpret_cast<char*>(workspace));
  return simt_backward(m, x, ldx, idx, mb, ws, grad_weight, net_grad, overwrite, st);
}

}  // namespace stx

using namespace stx;

extern "C" int64_t stx_mlp_param_count(const StxMlp* m) {
  if (!m) return 0;
  int64_t o = 0;
  for (int i = 0; i < m->n_layers; ++i)
    o += (int64_t)m->sizes[i] * m->sizes[i + 1] + ((m->use_layer_norm && i < m->n_layers - 1) ? 2 : 1) * (int64_t)m->sizes[i + 1];
  return o;
}

extern "C" size_t stx_mlp_forward_workspace_bytes(const StxMlp* m, int64_t M, int precision) {
  if (!m || M <= 0) return 0;
  if (precision == STX_PREC_BF16) return tc_mlp_forward_workspace_bytes(m, M);
  size_t o = 0;
  for (int i = 1; i < m->n_layers; ++i) o += align_up((size_t)M * m->sizes[i] * 4);
  return o > 0 ? o : 256;
}

extern "C" int stx_mlp_forward(const StxMlp* m, const void* x, int64_t ldx, const int32_t* row_idx,
                               int64_t M, float* out, int precision, void* workspace,
                               size_t workspace_bytes, void* stream) {
  if (int rc = check_mlp(m, "stx_mlp_forward")) return rc;
  STX_REQUIRE(x && out && M > 0, STX_E_ARG, "stx_mlp_forward: null x/out or M=%lld", (long long)M);
  STX_REQUIRE(ldx >= m->sizes[0], STX_E_SHAPE, "stx_mlp_forward: ldx=%lld < in dim %d", (long long)ldx, m->sizes[0]);
  STX_REQUIRE(workspace_bytes >= stx_mlp_forward_workspace_bytes(m, M, precision) && workspace, STX_E_WORKSPACE,
              "stx_mlp_forward: workspace %zu < %zu", workspace_bytes, stx_mlp_forward_workspace_bytes(m, M, precision));
  if (precision == STX_PREC_BF16)
    return tc_mlp_forward(m, x, ldx, row_idx, M, out, workspace, workspace_bytes, (cudaStream_t)stream);
  STX_REQUIRE(precision == STX_PREC_F32, STX_E_UNSUPPORTED, "stx_mlp_forward: precision=%d", precision);
  float* acts[STX_MAX_LAYERS + 1] = {nullptr};   // inference: pre-activations are not kept
  float* hacts[STX_MAX_LAYERS + 1] = {nullptr};
  char* p = reinterpret_cast<char*>(workspace);
  for (int i = 1; i < m->n_layers; ++i) {
    hacts[i] = reinterpret_cast<float*>(p);
    p += align_up((size_t)M * m->sizes[i] * 4);
  }
  return simt_forward(m, reinterpret_cast<const float*>(x), ldx, row_idx, M, acts, hacts, nullptr, out, (cudaStream_t)stream);
}

// ---- generic train-mode MLP: forward keeping what the backward needs, backward to parameters and / or the input ----
extern "C" size_t stx_mlp_train_workspace_bytes(const StxMlp* m, int64_t M) {
  if (!m || M <= 0) return 0;
  return carve(m, M, nullptr).bytes;
}

extern "C" int stx_mlp_forward_train(const StxMlp* m, const float* x, int64_t ldx, const int32_t* row_idx, int64_t M, float* out,
                                     void* workspace, size_t workspace_bytes, void* stream) {
  if (int rc = check_mlp(m, "stx_mlp_forward_train")) return rc;
  STX_REQUIRE(x && out && workspace && M > 0, STX_E_ARG, "stx_mlp_forward_train: null pointer or M=%lld", (long long)M);
  STX_REQUIRE(ldx >= m->sizes[0], STX_E_SHAPE, "stx_mlp_forward_train: ldx=%lld < in dim %d", (long long)ldx, m->sizes[0]);
  STX_REQUIRE(workspace_bytes >= stx_mlp_train_workspace_bytes(m, M), STX_E_WORKSPACE, "stx_mlp_forward_train: workspace %zu < %zu",
              workspace_bytes, stx_mlp_train_workspace_bytes(m, M));
  SimtPpoWs ws = carve(m, M, reinterpret_cast<char*>(workspace));
  return simt_forward(m, x, ldx, row_idx, M, ws.acts, ws.hacts, ws.stats, out, (cudaStream_t)stream);
}

extern "C" int stx_mlp_backward(const StxMlp* m, const float* x, int64_t ldx, const int32_t* row_idx, int64_t M, const float* d_out,
                                void* workspace, size_t workspace_bytes, float grad_weight, float* net_grad, int overwrite, float* d_input,
                                void* stream) {
  if (int rc = check_mlp(m, "stx_mlp_backward")) return rc;
  STX_REQUIRE(x && d_out && workspace && M > 0 && (net_grad || d_input), STX_E_ARG, "stx_mlp_backward: null pointer or nothing to compute");
  STX_REQUIRE(workspace_bytes >= stx_mlp_train_workspace_bytes(m, M), STX_E_WORKSPACE, "stx_mlp_backward: workspace %zu < %zu", workspace_bytes,
              stx_mlp_train_workspace_bytes(m, M));
  SimtPpoWs ws = carve(m, M, reinterpret_cast<char*>(workspace));
  cudaStream_t st = (cudaStream_t)stream;
  STX_CUDA_OK(cudaMemcpyAsync(ws.dhead, d_out, sizeof(float) * (size_t)M * m->sizes[m->n_layers], cudaMemcpyDeviceToDevice, st));
  return simt_backward(m, x, ldx, row_idx, M, ws, grad_weight, net_grad, overwrite, st, d_input);
}

extern "C" int stx_epsilon_greedy(const float* q, int64_t E, int A, int mode, uint64_t seed, uint64_t offset, const uint64_t* dev_counter,
                                  const int32_t* count, const StxEpsilonSchedule* sched, int32_t* action, float* epsilon_out,
                                  int32_t* update_no_out, void* stream) {
  STX_REQUIRE(q && sched && action, STX_E_ARG, "stx_epsilon_greedy: null pointer");
  STX_REQUIRE(E > 0 && A > 0, STX_E_SHAPE, "stx_epsilon_greedy: E=%lld A=%d", (long long)E, A);
  STX_REQUIRE(sched->steps_per_update > 0, STX_E_ARG, "stx_epsilon_greedy: steps_per_update=%d must be positive", sched->steps_per_update);
  epsilon_greedy_kernel<<<(unsigned)((E + 255) / 256), 256, 0, (cudaStream_t)stream>>>(q, E, A, mode, seed, offset, dev_counter, count, *sched,
                                                                                         action, epsilon_out, update_no_out);
  STX_LAUNCH_OK();
  return STX_OK;
}

extern "C" int stx_categorical(const float* logits, int64_t E, int A, int sample, uint64_t seed,
                               uint64_t offset, const uint64_t* dev_counter, int32_t* action,
                               float* log_prob, float* entropy, void* stream) {
  STX_REQUIRE(logits && action && log_prob, STX_E_ARG, "stx_categorical: null pointer");
  STX_REQUIRE(E > 0 && A > 0, STX_E_SHAPE, "stx_categorical: E=%lld A=%d", (long long)E, A);
  categorical_kernel<<<(unsigned)((E + 255) / 256), 256, 0, (cudaStream_t)stream>>>(logits, E, A, sample, seed, offset, dev_counter, action, log_prob, entropy);
  STX_LAUNCH_OK();
  return STX_OK;
}

extern "C" void stx_ppo_arena_offsets(const StxMlp* actor, const StxMlp* critic, int64_t* actor_off,
                                      int64_t* critic_off, int64_t* total) {
  const int64_t na = stx_mlp_param_count(actor), nc = stx_mlp_param_count(critic);
  const int64_t coff = (na + 7) / 8 * 8;  // 8 floats: the bf16 shadow of each network stays 16-byte aligned (TMA)
  if (actor_off) *actor_off = 0;
  if (critic_off) *critic_off = coff;
  if (total) *total = coff + (nc + 7) / 8 * 8;
}

extern "C" size_t stx_ppo_workspace_bytes(const StxMlp* actor, const StxMlp* critic, int64_t mb, int precision) {
  if (!actor || !critic || mb <= 0) return 0;
  if (precision == STX_PREC_BF16) return tc_ppo_workspace_bytes(actor, critic, mb);
  const size_t a = carve(actor, mb, nullptr).bytes, c = carve(critic, mb, nullptr).bytes;
  return (a > c ? a : c);
}
