// Recurrent layer of rec_ppo and rec_r2d2 (fp32): ScannedRNN(cell_type="gru" | "lstm") over a (T, E) sequence with episode
// resets, forward and backward-through-time.
//
// Reference: stoix/networks/base.py:124-159 (ScannedRNN: the carry is replaced by zeros where `resets` is set, THEN the cell
// runs; nn.scan over the leading axis) as used by RecurrentActor / RecurrentCritic (:162-222) in
// stoix/systems/ppo/anakin/rec_ppo.py:90-101 (one step per env step) and :216-247 (whole chunk inside the loss, under jax.grad).
// flax.linen.GRUCell / LSTMCell are not vendored in the reference; their published definitions are restated:
//     GRU:  r = sigmoid(gi_r + gh_r)   z = sigmoid(gi_z + gh_z)   n = tanh(gi_n + r * (gh_n + b_hn))   h' = (1 - z) n + z h
//     LSTM: i, f, o = sigmoid(gi + gh), g = tanh(gi_g + gh_g)    c' = f c + i g   h' = o tanh(c')   carry = (c | h)
// with gi = W_i x + b_i (all input projections carry a bias), gh = W_h h (only the GRU's n part carries a bias, b_hn).
//
// The input projections of ALL timesteps are one GEMM outside (they are the "head" of the pre-torso MLP); what is sequential is
// h @ W_h + the gate arithmetic, T times.  GruCell / LstmCell hold that arithmetic once per cell (gate count G, saved
// activations, forward and backward of one (row, hidden unit) item); every launch form runs it:
//   * cluster (T >= kPersistentMinT, both cells): a 2-CTA thread-block cluster per tile of R sequences; CTA q owns the hidden
//     units [q H/2, (q+1) H/2), i.e. G H/2 columns of W_h resident in its shared memory, and pushes its half of every new h to
//     the peer through distributed shared memory.  No per-step launch, no global synchronisation.
//   * persistent (T >= kPersistentMinT, GRU only, when the cluster form is off or does not fit: odd H, E >= 1024 rows): one CTA
//     per tile with the whole W_h (H x 3H) in shared memory.  The LSTM's W_h (H x 4H, 262 KB at H = 128) does not fit one SM.
//   * per-step (every other shape, e.g. the rollout's T = 1): one SIMT GEMM (stx_simt_gemm.cuh) + one gate kernel per step,
//     issued by a host loop inside the entry point.
// STX_GRU_CLUSTER=0, STX_GRU_PERSISTENT=0 and STX_LSTM_CLUSTER=0 switch a form off (read once per process).
// Backward: the gate backward of step t turns d(h_t) into d(gi_t), d(gh_t); d(h_{t-1}) = d(gh_t) W_h^T + the direct term
// (masked by reset_t); d(W_h) = sum_t hp_t^T d(gh_t) is ONE split GEMM over the stored sequences after the loop (fixed
// summation order: deterministic), in every form.
#include <cooperative_groups.h>

#include "stx_common.cuh"
#include "stx_simt_gemm.cuh"

namespace stx {
namespace {

namespace cg = cooperative_groups;

inline size_t ralign(size_t x) { return (x + 255) / 256 * 256; }

// a form switch: on unless the variable is set to 0
inline bool env_on(const char* name) {
  const char* e = getenv(name);
  return !(e && e[0] == '0');
}

__device__ __forceinline__ float sigm(float x) { return 1.f / (1.f + expf(-x)); }

// ---- cells ------------------------------------------------------------------------------------------------------------------
// fwd: x = gi, y = h W_h (no bias) of the G gates of one item, bhn = b_hn of its unit (GRU), hp = h entering the step; c: the
// LSTM's c entering the step, replaced by the new c.  Returns h' and the activations the backward needs in s.
// bwd: dh = d(h') as the form assembled it, dc = d(c') arriving from step t + 1 (LSTM), p = the carry entering the step (GRU:
// hp, LSTM: cp).  Writes d(gi) (dx) and d(gh) (dy) and returns the direct part of d(carry entering): GRU d(hp) = dh z, LSTM
// d(cp) = dc f (the LSTM's d(hp) is all W_h^T).
struct GruCell {
  static constexpr int G = 3;               // gates r, z, n
  static constexpr int S = 4;               // saved: r, z, n, gh_n + b_hn
  static constexpr bool kC = false;         // the carry is h alone
  static constexpr bool kBhn = true;        // b_hn inside r (...): d(gh) differs from d(gi); d(b_hn) = column sums of d(gh_n)
  static constexpr bool kPersistent = true;
  static constexpr const char* kClusterEnv = "STX_GRU_CLUSTER";
  static bool cluster_rows_ok(int64_t E) { return E < 1024; }   // from 1024 rows on the persistent seq<8,1> form runs
  __device__ __forceinline__ static float bias(const float* __restrict__ b_hn, int j) { return __ldg(b_hn + j); }

  __device__ __forceinline__ static float fwd(const float (&x)[G], const float (&y)[G], float bhn, float hp, float& c, float (&s)[S]) {
    const float r = sigm(x[0] + y[0]);
    const float z = sigm(x[1] + y[1]);
    const float ghn = y[2] + bhn;
    const float n = tanhf(x[2] + r * ghn);
    s[0] = r, s[1] = z, s[2] = n, s[3] = ghn;
    return __fmaf_rn(1.f - z, n, __fmul_rn(z, hp));   // (1 - z) n + z h, with the product that is rounded first fixed
  }
  __device__ __forceinline__ static float bwd(float dh, float dc, float p, const float (&s)[S], float (&dx)[G], float (&dy)[G]) {
    const float r = s[0], z = s[1], n = s[2], ghn = s[3];
    const float dn = dh * (1.f - z), dz = dh * (p - n);
    const float dpn = dn * (1.f - n * n);
    const float dpr = dpn * ghn * r * (1.f - r);
    const float dpz = dz * z * (1.f - z);
    dx[0] = dpr, dx[1] = dpz, dx[2] = dpn;
    dy[0] = dpr, dy[1] = dpz, dy[2] = dpn * r;
    return dh * z;
  }
};

struct LstmCell {
  static constexpr int G = 4;               // gates i, f, g, o
  static constexpr int S = 5;               // saved: i, f, g, o, tanh(c')
  static constexpr bool kC = true;          // the carry is (c | h)
  static constexpr bool kBhn = false;       // d(gh) = d(gi) = d(z): one buffer
  static constexpr bool kPersistent = false;
  static constexpr const char* kClusterEnv = "STX_LSTM_CLUSTER";
  static bool cluster_rows_ok(int64_t) { return true; }
  __device__ __forceinline__ static float bias(const float* __restrict__, int) { return 0.f; }

  __device__ __forceinline__ static float fwd(const float (&x)[G], const float (&y)[G], float, float, float& c, float (&s)[S]) {
    const float ig = sigm(x[0] + y[0]), fg = sigm(x[1] + y[1]), gg = tanhf(x[2] + y[2]), og = sigm(x[3] + y[3]);
    c = __fmaf_rn(ig, gg, __fmul_rn(fg, c));   // f c + i g, with the product that is rounded first fixed
    const float tc = tanhf(c);
    s[0] = ig, s[1] = fg, s[2] = gg, s[3] = og, s[4] = tc;
    return og * tc;
  }
  __device__ __forceinline__ static float bwd(float dh, float dc, float p, const float (&s)[S], float (&dx)[G], float (&dy)[G]) {
    const float ig = s[0], fg = s[1], gg = s[2], og = s[3], tc = s[4];
    dc += dh * og * (1.f - tc * tc);
    dx[0] = dc * gg * ig * (1.f - ig);
    dx[1] = dc * p * fg * (1.f - fg);
    dx[2] = dc * ig * (1.f - gg * gg);
    dx[3] = dh * tc * og * (1.f - og);
#pragma unroll
    for (int g = 0; g < G; ++g) dy[g] = dx[g];
    return dc * fg;
  }
};

// the saved activations of every step, [S][T][E][H]
template <int S>
struct Saved {
  float* p[S];
  Saved at(size_t offset) const {   // the activations of one step
    Saved r;
    for (int g = 0; g < S; ++g) r.p[g] = p[g] + offset;
    return r;
  }
};

// ---- workspace ----------------------------------------------------------------------------------------------------------
template <class Cell>
struct SeqWs {
  float* hp_seq;              // [T + 1][E][H]  h entering step t (after the reset)
  float* cp_seq;              // [T + 1][E][H]  c entering step t (LSTM)
  Saved<Cell::S> act;         // [T][E][H] each
  float* gh;                  // [E][G H]       per-step h W_h
  float* d_gh_seq;            // [T][E][G H]    d(gh) (GRU; the LSTM's is d_gi)
  float* dhp_gemm;            // [E][H]         per-step d(gh) W_h^T
  float* direct[2];           // [E][H]         per-step direct part of d(carry entering), alternating
  float* partials;            // [splits][H G H (+ G H d(b_hn) column sums)]
  int splits;
  size_t bytes;
};

int dw_splits(int64_t rows) {   // d(W_h) GEMM: (H/64) x (G H/64) output tiles; 512 rows per split fill the GPU from 32k rows on
  int64_t s = rows / 512;
  if (s < 1) s = 1;
  if (s > 64) s = 64;
  return (int)s;
}

template <class Cell>
SeqWs<Cell> carve(int T, int64_t E, int H, char* base) {
  constexpr int G = Cell::G;
  SeqWs<Cell> w{};
  size_t o = 0;
  auto take = [&](size_t floats) {
    float* p = base ? reinterpret_cast<float*>(base + o) : nullptr;
    o += ralign(floats * 4);
    return p;
  };
  const size_t eh = (size_t)E * H;
  w.hp_seq = take((size_t)(T + 1) * eh);
  if (Cell::kC) w.cp_seq = take((size_t)(T + 1) * eh);
  for (int s = 0; s < Cell::S; ++s) w.act.p[s] = take((size_t)T * eh);
  w.gh = take(G * eh);
  if (Cell::kBhn) w.d_gh_seq = take((size_t)T * G * eh);
  w.dhp_gemm = take(eh);
  w.direct[0] = take(eh), w.direct[1] = take(eh);
  w.splits = dw_splits((int64_t)T * E);
  w.partials = take((size_t)w.splits * ((size_t)H * G * H + (Cell::kBhn ? G * H : 0)));
  w.bytes = o;
  return w;
}

// ---- per-step form ------------------------------------------------------------------------------------------------------
// hp_0 = where(reset_0, 0, h0) (and cp_0 alike); carry0 is (E, H) h0 (GRU) or (E, 2H) = (c | h) (LSTM)
template <class Cell>
__global__ void step_init_kernel(const float* __restrict__ carry0, const uint8_t* __restrict__ reset0, int64_t E, int H, float* __restrict__ hp0,
                                 float* __restrict__ cp0) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= E * H) return;
  const int64_t e = i / H;
  const int k = (int)(i % H);
  const bool cut = reset0[e] != 0;
  if constexpr (Cell::kC) cp0[i] = cut ? 0.f : carry0[e * 2 * H + k];
  hp0[i] = cut ? 0.f : carry0[Cell::kC ? e * 2 * H + H + k : i];
}

// step t: gates from gi_t and gh = hp_t W_h; writes h_t, the saved activations and the carry entering step t + 1 (reset_next:
// null at the last step); pointers are those of step t
template <class Cell>
__global__ void step_fwd_kernel(const float* __restrict__ gi, const float* __restrict__ gh, const float* __restrict__ b_hn, const float* __restrict__ hp,
                                const float* __restrict__ cp, const uint8_t* __restrict__ reset_next, int64_t E, int H, float* __restrict__ h_out,
                                float* __restrict__ hp_next, float* __restrict__ cp_next, Saved<Cell::S> act, float* __restrict__ carry_last) {
  constexpr int G = Cell::G;
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= E * H) return;
  const int64_t e = i / H;
  const int k = (int)(i % H);
  const float* a = gi + e * G * H + k;
  const float* b = gh + e * G * H + k;
  float x[G], y[G], s[Cell::S], c = 0.f;
#pragma unroll
  for (int g = 0; g < G; ++g) x[g] = a[g * H], y[g] = b[g * H];
  if constexpr (Cell::kC) c = cp[i];
  const float h = Cell::fwd(x, y, Cell::bias(b_hn, k), hp[i], c, s);
  h_out[i] = h;
#pragma unroll
  for (int g = 0; g < Cell::S; ++g) act.p[g][i] = s[g];
  const bool cut = reset_next && reset_next[e];
  hp_next[i] = cut ? 0.f : h;
  if constexpr (Cell::kC) {
    cp_next[i] = cut ? 0.f : c;
    if (carry_last) carry_last[e * 2 * H + k] = c, carry_last[e * 2 * H + H + k] = h;
  }
}

// step t: d(h_t) (from the layers above + from step t + 1; dhp_gemm_next null at the last step) -> d(gi_t), d(gh_t) (GRU) and
// the direct part of d(carry entering step t); pointers are those of step t
template <class Cell>
__global__ void step_bwd_kernel(const float* __restrict__ d_h_out, const float* __restrict__ dhp_gemm_next, const float* __restrict__ direct_next,
                                const uint8_t* __restrict__ reset_next, Saved<Cell::S> act, const float* __restrict__ carry, int64_t E, int H,
                                float* __restrict__ d_gi, float* __restrict__ d_gh, float* __restrict__ direct) {
  constexpr int G = Cell::G;
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= E * H) return;
  const int64_t e = i / H;
  const int k = (int)(i % H);
  float dh = d_h_out[i], dc = 0.f;
  if (dhp_gemm_next && !reset_next[e]) {   // base.py:139-148: the reset cuts the chain (both halves of the LSTM carry)
    if constexpr (Cell::kC) dh += dhp_gemm_next[i], dc = direct_next[i];
    else dh += dhp_gemm_next[i] + direct_next[i];
  }
  float s[Cell::S], dx[G], dy[G];
#pragma unroll
  for (int g = 0; g < Cell::S; ++g) s[g] = act.p[g][i];
  direct[i] = Cell::bwd(dh, dc, carry[i], s, dx, dy);
#pragma unroll
  for (int g = 0; g < G; ++g) d_gi[e * G * H + g * H + k] = dx[g];
  if constexpr (Cell::kBhn) {
#pragma unroll
    for (int g = 0; g < G; ++g) d_gh[e * G * H + g * H + k] = dy[g];
  }
}

// d(carry0) = where(reset_0, 0, d(carry entering step 0))
template <class Cell>
__global__ void step_dcarry0_kernel(const float* __restrict__ dhp_gemm, const float* __restrict__ direct, const uint8_t* __restrict__ reset0, int64_t E,
                                    int H, float* __restrict__ d_carry0) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= E * H) return;
  const int64_t e = i / H;
  const int k = (int)(i % H);
  const bool cut = reset0[e] != 0;
  if constexpr (Cell::kC) {
    d_carry0[e * 2 * H + k] = cut ? 0.f : direct[i];
    d_carry0[e * 2 * H + H + k] = cut ? 0.f : dhp_gemm[i];
  } else {
    d_carry0[i] = cut ? 0.f : dhp_gemm[i] + direct[i];
  }
}

// G column blocks of Hq columns of W_h (H x G H), starting at column q Hq of each block, into Ws [H][G Hq + 1] (rows padded by one
// float so that both the forward walk (lanes along columns) and the transposed walk of the backward (lanes along k) are free of
// bank conflicts): local column g Hq + jl <-> global column g H + q Hq + jl.  The persistent kernels load all of W_h (Hq = H, q = 0).
__device__ __forceinline__ void load_w(float* __restrict__ Ws, const float* __restrict__ w_h, int H, int Hq, int q, int G) {
  const int nl = G * Hq, total = H * nl;
  constexpr int U = 8;
  for (int base = threadIdx.x; base < total; base += blockDim.x * U) {
    float v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int i = base + u * blockDim.x;
      if (i < total) {
        const int k = i / nl, c = i % nl;
        v[u] = __ldg(w_h + i + (size_t)k * (G * H - nl) + (c / Hq) * (H - Hq) + q * Hq);   // k G H + (c / Hq) H + q Hq + c % Hq
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int i = base + u * blockDim.x;
      if (i < total) Ws[(i / nl) * (nl + 1) + i % nl] = v[u];
    }
  }
}

// ---- persistent GRU sequence kernels -------------------------------------------------------------------------------------
// One CTA owns R sequences (rows) for ALL T steps with the whole recurrent matrix W_h (H x 3H fp32, 196 KB at H = 128) resident in
// shared memory, so the recurrence needs no global synchronisation and no per-step launch: per step the CTA streams gi_t in,
// does the (R x H) @ (H x 3H) product out of shared memory (thread n owns gate column n for the R rows), applies the gates
// (thread j owns hidden unit j) and writes h_t plus what the backward needs.  The step time is set by reading W_h once from
// shared memory (3H * H * 4 B / 128 B per clock ~ 1.5k cycles at H = 128), not by launches.
// Backward: same residency, reverse time; d(gh_t) is kept for the ONE GEMM that forms d(W_h) afterwards.
template <int R, int KS>
struct GruSmem {
  __host__ __device__ static size_t w_floats(int H) { return ((size_t)H * (3 * H + 1) + 3) / 4 * 4; }   // keeps the float4 arrays behind it 16-byte aligned
  static size_t fwd_bytes(int H) { return (w_floats(H) + (size_t)H * R + (size_t)KS * R * 3 * H) * 4; }
  static size_t bwd_bytes(int H) { return (w_floats(H) + (size_t)3 * H * R + 3 * (size_t)KS * R * H + (size_t)R * H) * 4; }
};
constexpr int kGruItems = 3;   // gate items (row, hidden unit) per thread: H * R <= kGruItems * blockDim for every launch shape

// KS thread groups split the reduction of the per-step product (partials added in a fixed order); what the gate phase of a step
// needs from global memory (gi_t, reset_{t+1}; backward: the saved gates of step t - 1) is requested BEFORE the product of the
// step, so its latency hides behind the shared-memory walk instead of sitting in front of the gate arithmetic.
template <int R, int KS>
__global__ void __launch_bounds__(1024, 1)
    gru_seq_fwd_kernel(const float* __restrict__ gi, const uint8_t* __restrict__ reset, const float* __restrict__ h0, const float* __restrict__ w_h,
                       const float* __restrict__ b_hn, int T, int64_t E, int H, float* __restrict__ h_seq, float* __restrict__ hp_seq,
                       Saved<GruCell::S> act) {
  extern __shared__ __align__(16) float gsm[];
  const int n3 = 3 * H;
  float* Ws = gsm;                               // [H][3H + 1]
  float* hs = Ws + GruSmem<R, KS>::w_floats(H);  // [H][R]   state entering the step, k-major
  float* ghp = hs + (size_t)H * R;               // [KS][R][3H] partial products
  const int kh = threadIdx.x / n3, n = threadIdx.x % n3;   // reduction group, gate column
  const int kper = (H + KS - 1) / KS;
  const int k_begin = kh * kper, k_end = (k_begin + kper < H) ? k_begin + kper : H;
  const int64_t row0 = (int64_t)blockIdx.x * R;
  const int items = H * R;
  load_w(Ws, w_h, H, H, 0, 3);
  for (int i = threadIdx.x; i < items; i += blockDim.x) {
    const int r = i / H, j = i % H;
    const int64_t row = row0 + r;
    float v = 0.f;
    if (row < E) {
      v = reset[row] ? 0.f : h0[row * H + j];
      hp_seq[row * H + j] = v;
    }
    hs[j * R + r] = v;
  }
  __syncthreads();
  const int64_t eh = E * (int64_t)H;
  for (int t = 0; t < T; ++t) {
    // ---- requests for the gate phase ----
    float x[kGruItems][3], bh[kGruItems];
    bool cut[kGruItems];
#pragma unroll
    for (int q = 0; q < kGruItems; ++q) {
      const int i = threadIdx.x + q * blockDim.x;
      x[q][0] = x[q][1] = x[q][2] = bh[q] = 0.f, cut[q] = false;
      if (i < items) {
        const int r = i / H, j = i % H;
        const int64_t row = row0 + r;
        if (row < E) {
          const float* a = gi + ((int64_t)t * E + row) * n3;
          x[q][0] = __ldg(a + j), x[q][1] = __ldg(a + H + j), x[q][2] = __ldg(a + 2 * H + j), bh[q] = GruCell::bias(b_hn, j);
          cut[q] = (t + 1 < T) && reset[(int64_t)(t + 1) * E + row] != 0;
        }
      }
    }
    // ---- (R x H) @ (H x 3H), this group's share of k ----
    if (kh < KS) {
      float2 acc[R / 2];
#pragma unroll
      for (int r = 0; r < R / 2; ++r) acc[r] = make_float2(0.f, 0.f);
      const float* wcol = Ws + n;
#pragma unroll 4
      for (int k = k_begin; k < k_end; ++k) {
        const float w = wcol[(size_t)k * (n3 + 1)];
        const float* hk = hs + k * R;
#pragma unroll
        for (int r4 = 0; r4 < R; r4 += 4) {
          const float4 hv = *reinterpret_cast<const float4*>(hk + r4);
          fma2(acc[r4 / 2], w, make_float2(hv.x, hv.y)), fma2(acc[r4 / 2 + 1], w, make_float2(hv.z, hv.w));
        }
      }
#pragma unroll
      for (int r = 0; r < R / 2; ++r) ghp[((size_t)kh * R + 2 * r) * n3 + n] = acc[r].x, ghp[((size_t)kh * R + 2 * r + 1) * n3 + n] = acc[r].y;
    }
    __syncthreads();
    // ---- gates: consecutive threads -> consecutive hidden units of one row ----
#pragma unroll
    for (int q = 0; q < kGruItems; ++q) {
      const int i = threadIdx.x + q * blockDim.x;
      if (i >= items) continue;
      const int r = i / H, j = i % H;
      const int64_t row = row0 + r;
      if (row >= E) continue;
      float y[3] = {0.f, 0.f, 0.f};
#pragma unroll
      for (int g = 0; g < KS; ++g) {   // fixed order over the reduction groups
        const float* b = ghp + ((size_t)g * R + r) * n3;
        y[0] += b[j], y[1] += b[H + j], y[2] += b[2 * H + j];
      }
      float s[GruCell::S], c;
      const float h = GruCell::fwd(x[q], y, bh[q], hs[j * R + r], c, s);
      const int64_t o = (int64_t)t * eh + row * H + j;
      h_seq[o] = h;
#pragma unroll
      for (int g = 0; g < GruCell::S; ++g) act.p[g][o] = s[g];
      const float hn = cut[q] ? 0.f : h;
      hp_seq[o + eh] = hn;
      hs[j * R + r] = hn;   // only this thread touches (j, r) in this phase; the product above is behind the barrier
    }
    __syncthreads();
  }
}

template <int R, int KS>
__global__ void __launch_bounds__(1024, 1)
    gru_seq_bwd_kernel(const float* __restrict__ d_h_seq, const uint8_t* __restrict__ reset, const float* __restrict__ w_h, int T, int64_t E, int H,
                       const float* __restrict__ hp_seq, Saved<GruCell::S> act, float* __restrict__ d_gi, float* __restrict__ d_gh_seq,
                       float* __restrict__ d_h0) {
  extern __shared__ __align__(16) float gsm[];
  const int n3 = 3 * H;
  constexpr int NB = 3 * KS;                       // column blocks of the transposed product
  float* Ws = gsm;                                 // [H][3H + 1]
  float* dgT = Ws + GruSmem<R, KS>::w_floats(H);   // [3H][R]  d(gh_t), n-major
  float* part = dgT + (size_t)n3 * R;              // [NB][R][H] partial sums of d(gh) W_h^T over the column blocks
  float* dh_rec = part + (size_t)NB * R * H;       // [R][H]   gradient arriving from step t + 1 (already masked by its reset)
  const int64_t row0 = (int64_t)blockIdx.x * R;
  const int64_t eh = E * (int64_t)H;
  const int items = H * R;
  load_w(Ws, w_h, H, H, 0, 3);
  for (int i = threadIdx.x; i < items; i += blockDim.x) dh_rec[i] = 0.f;
  // saved values of the step the gate phase will process next (requested one step ahead)
  float v_dh[kGruItems], v_s[kGruItems][GruCell::S], v_hp[kGruItems];
  bool v_cut[kGruItems];
  auto request = [&](int t) {
#pragma unroll
    for (int q = 0; q < kGruItems; ++q) {
      const int i = threadIdx.x + q * blockDim.x;
      v_dh[q] = v_s[q][0] = v_s[q][1] = v_s[q][2] = v_s[q][3] = v_hp[q] = 0.f, v_cut[q] = false;
      if (i < items && t >= 0) {
        const int r = i / H, j = i % H;
        const int64_t row = row0 + r;
        if (row < E) {
          const int64_t o = (int64_t)t * eh + row * H + j;
          v_dh[q] = __ldg(d_h_seq + o);
#pragma unroll
          for (int g = 0; g < GruCell::S; ++g) v_s[q][g] = __ldg(act.p[g] + o);
          v_hp[q] = __ldg(hp_seq + o);
          v_cut[q] = reset[(int64_t)t * E + row] != 0;
        }
      }
    }
  };
  request(T - 1);
  __syncthreads();
  const int kcol = (H + KS - 1) / KS;               // columns per block of the transposed product
  for (int t = T - 1; t >= 0; --t) {
    bool cut_t[kGruItems];
#pragma unroll
    for (int q = 0; q < kGruItems; ++q) {            // gate gradients of step t from the values requested earlier
      const int i = threadIdx.x + q * blockDim.x;
      cut_t[q] = v_cut[q];
      if (i >= items) continue;
      const int r = i / H, j = i % H;
      const int64_t row = row0 + r;
      float dy[3] = {0.f, 0.f, 0.f}, direct = 0.f;
      if (row < E) {
        float dx[3];
        direct = GruCell::bwd(v_dh[q] + dh_rec[r * H + j], 0.f, v_hp[q], v_s[q], dx, dy);
        float* a = d_gi + ((int64_t)t * E + row) * n3;
        float* b = d_gh_seq + ((int64_t)t * E + row) * n3;
        a[j] = dx[0], a[H + j] = dx[1], a[2 * H + j] = dx[2];
        b[j] = dy[0], b[H + j] = dy[1], b[2 * H + j] = dy[2];
      }
      dgT[j * R + r] = dy[0], dgT[(H + j) * R + r] = dy[1], dgT[(2 * H + j) * R + r] = dy[2];
      dh_rec[r * H + j] = direct;   // the direct part of d(hp_t); the W_h^T part is added below
    }
    request(t - 1);                 // in flight under the product
    __syncthreads();
    if ((int)threadIdx.x < NB * H) {   // d(gh_t) W_h^T: thread (k, block) sums the columns of its block
      const int k = threadIdx.x % H, blk = threadIdx.x / H;
      const int gate = blk / KS, sub = blk % KS;                 // block = (gate, sub-range of its H columns)
      const int c0 = gate * H + sub * kcol, c1 = (sub * kcol + kcol < H) ? c0 + kcol : gate * H + H;
      float2 acc[R / 2];
#pragma unroll
      for (int r = 0; r < R / 2; ++r) acc[r] = make_float2(0.f, 0.f);
      const float* wrow = Ws + (size_t)k * (n3 + 1);
#pragma unroll 4
      for (int nn = c0; nn < c1; ++nn) {
        const float w = wrow[nn];
#pragma unroll
        for (int r4 = 0; r4 < R; r4 += 4) {
          const float4 dv = *reinterpret_cast<const float4*>(dgT + (size_t)nn * R + r4);
          fma2(acc[r4 / 2], w, make_float2(dv.x, dv.y)), fma2(acc[r4 / 2 + 1], w, make_float2(dv.z, dv.w));
        }
      }
#pragma unroll
      for (int r = 0; r < R / 2; ++r) part[((size_t)blk * R + 2 * r) * H + k] = acc[r].x, part[((size_t)blk * R + 2 * r + 1) * H + k] = acc[r].y;
    }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < kGruItems; ++q) {
      const int i = threadIdx.x + q * blockDim.x;
      if (i >= items) continue;
      const int r = i / H, j = i % H;
      const int64_t row = row0 + r;
      float dhp = dh_rec[i];
#pragma unroll
      for (int blk = 0; blk < NB; ++blk) dhp += part[((size_t)blk * R + r) * H + j];   // fixed order
      dh_rec[i] = (row < E && !cut_t[q]) ? dhp : 0.f;   // base.py:139-148: the reset of step t cuts the chain into step t - 1
    }
    __syncthreads();
  }
  if (d_h0)
    for (int i = threadIdx.x; i < items; i += blockDim.x) {
      const int r = i / H, j = i % H;
      if (row0 + r < E) d_h0[(row0 + r) * H + j] = dh_rec[i];
    }
}

// ---- cluster form: 2-CTA thread-block clusters, either cell ------------------------------------------------------------------
// CTA q of a cluster owns the hidden units [q H/2, (q+1) H/2) of a tile of R sequences -- the G gate columns of those units, G H/2
// columns of W_h (99 KB for the GRU, 131 KB for the LSTM at H = 128) -- computes their gates and cell update, and after every step
// pushes its half of the new h into the PEER's shared memory (distributed shared memory) next to its own, into the buffer the
// next step reads (two h buffers alternate, so a fast CTA never overwrites what its peer still reads); one cluster barrier per
// step replaces the block barrier.  Backward: each CTA forms d(gh) of its units, multiplies with its G H/2 columns of W_h^T for
// ALL H outputs and sends the half that belongs to the peer's units across; the two partial sums are added in rank order
// (deterministic).  Against the persistent GRU form it halves the issue-bound per-step product.
constexpr int kClusterR = 4, kClusterKS = 2;   // rows per tile, thread groups splitting the reduction of the forward product

template <class Cell>
struct ClusterSmem {
  static constexpr int R = kClusterR, KS = kClusterKS, G = Cell::G, NC = Cell::kC ? 2 : 1;
  __host__ __device__ static size_t w_floats(int H) { return ((size_t)H * (G * (H / 2) + 1) + 3) / 4 * 4; }
  static size_t fwd_bytes(int H) { return (w_floats(H) + 2 * (size_t)H * R + (Cell::kC ? (size_t)(H / 2) * R : 0) + (size_t)KS * R * G * (H / 2)) * 4; }
  static size_t bwd_bytes(int H) { return (w_floats(H) + (size_t)G * (H / 2) * R + (size_t)G * R * H + (size_t)(2 + NC) * R * (H / 2)) * 4; }
};

template <class Cell>
__global__ void __launch_bounds__(1024, 1)
    cluster_fwd_kernel(const float* __restrict__ gi, const uint8_t* __restrict__ reset, const float* __restrict__ carry0, const float* __restrict__ w_h,
                       const float* __restrict__ b_hn, int T, int64_t E, int H, float* __restrict__ h_seq, float* __restrict__ carry_last,
                       float* __restrict__ hp_seq, float* __restrict__ cp_seq, Saved<Cell::S> act) {
  constexpr int R = kClusterR, KS = kClusterKS, G = Cell::G, NC = Cell::kC ? 2 : 1;
  cg::cluster_group cluster = cg::this_cluster();
  const int q = (int)cluster.block_rank();
  extern __shared__ __align__(16) float gsm[];
  const int Hq = H / 2, nl = G * Hq;
  float* Ws = gsm;                                        // [H][nl + 1]
  float* hs = Ws + ClusterSmem<Cell>::w_floats(H);        // [2][H][R]  full h entering the step (k-major), two alternating buffers
  float* cs = hs + 2 * (size_t)H * R;                     // [Hq][R]    c of this CTA's units (LSTM)
  float* ghp = cs + (Cell::kC ? (size_t)Hq * R : 0);      // [KS][R][nl] partial products
  float* hs_peer = cluster.map_shared_rank(hs, q ^ 1);
  const int kh = threadIdx.x / nl, n = threadIdx.x % nl;
  const int kper = (H + KS - 1) / KS;
  const int k_begin = kh * kper, k_end = (k_begin + kper < H) ? k_begin + kper : H;
  const int64_t row0 = (int64_t)(blockIdx.x / 2) * R;
  const int items = Hq * R;
  const int64_t eh = E * (int64_t)H;
  load_w(Ws, w_h, H, Hq, q, G);
  for (int i = threadIdx.x; i < H * R; i += blockDim.x) {     // every CTA initialises the FULL h of buffer 0 itself
    const int r = i / H, j = i % H;
    const int64_t row = row0 + r;
    float hv = 0.f;
    if (row < E && !reset[row]) hv = carry0[row * NC * H + (NC - 1) * H + j];
    hs[j * R + r] = hv;
    if (j / Hq == q) {
      if (row < E) hp_seq[row * H + j] = hv;
      if constexpr (Cell::kC) {
        const float cv = (row < E && !reset[row]) ? carry0[row * 2 * H + j] : 0.f;
        cs[(j - q * Hq) * R + r] = cv;
        if (row < E) cp_seq[row * H + j] = cv;
      }
    }
  }
  cluster.sync();
  const int i0 = threadIdx.x;                // one gate item per thread: Hq * R <= blockDim
  const int r0 = i0 / Hq, jl0 = i0 % Hq;
  const int64_t rowg = row0 + r0;
  const int j0 = q * Hq + jl0;
  for (int t = 0; t < T; ++t) {
    const float* hcur = hs + (size_t)(t & 1) * H * R;
    const size_t nxt = (size_t)((t + 1) & 1) * H * R;
    // requests for the gate phase
    float x[G] = {}, bh = 0.f;
    bool cut = false;
    if (i0 < items && rowg < E) {
      const float* a = gi + ((int64_t)t * E + rowg) * G * H + j0;
#pragma unroll
      for (int g = 0; g < G; ++g) x[g] = __ldg(a + g * H);
      bh = Cell::bias(b_hn, j0);
      cut = (t + 1 < T) && reset[(int64_t)(t + 1) * E + rowg] != 0;
    }
    if (kh < KS) {
      float2 a01 = make_float2(0.f, 0.f), a23 = make_float2(0.f, 0.f);
      const float* wcol = Ws + n;
#pragma unroll 4
      for (int k = k_begin; k < k_end; ++k) {
        const float w = wcol[(size_t)k * (nl + 1)];
        const float4 hv = *reinterpret_cast<const float4*>(hcur + k * R);
        fma2(a01, w, make_float2(hv.x, hv.y)), fma2(a23, w, make_float2(hv.z, hv.w));
      }
      const float acc[R] = {a01.x, a01.y, a23.x, a23.y};
#pragma unroll
      for (int r = 0; r < R; ++r) ghp[((size_t)kh * R + r) * nl + n] = acc[r];
    }
    __syncthreads();
    if (i0 < items) {
      float hn = 0.f;
      if (rowg < E) {
        float y[G];
#pragma unroll
        for (int g = 0; g < G; ++g) {
          float v = 0.f;
#pragma unroll
          for (int kk = 0; kk < KS; ++kk) v += ghp[((size_t)kk * R + r0) * nl + g * Hq + jl0];   // fixed order
          y[g] = v;
        }
        float s[Cell::S], c = 0.f;
        if constexpr (Cell::kC) c = cs[jl0 * R + r0];
        const float h = Cell::fwd(x, y, bh, hcur[j0 * R + r0], c, s);
        const int64_t o = (int64_t)t * eh + rowg * H + j0;
        h_seq[o] = h;
#pragma unroll
        for (int g = 0; g < Cell::S; ++g) act.p[g][o] = s[g];
        hn = cut ? 0.f : h;
        hp_seq[o + eh] = hn;
        if constexpr (Cell::kC) {
          const float cn = cut ? 0.f : c;
          cp_seq[o + eh] = cn;
          cs[jl0 * R + r0] = cn;
          if (t == T - 1 && carry_last) carry_last[rowg * 2 * H + j0] = c, carry_last[rowg * 2 * H + H + j0] = h;
        }
      }
      hs[nxt + (size_t)j0 * R + r0] = hn;         // my half of the next step's h: here ...
      hs_peer[nxt + (size_t)j0 * R + r0] = hn;    // ... and in the peer's shared memory
    }
    cluster.sync();   // both halves of h_{t+1} are in place in both CTAs; also this block's barrier
  }
}

// carry_seq: the carry the cell's backward reads (GRU: hp_seq, LSTM: cp_seq)
template <class Cell>
__global__ void __launch_bounds__(1024, 1)
    cluster_bwd_kernel(const float* __restrict__ d_h_seq, const uint8_t* __restrict__ reset, const float* __restrict__ w_h, int T, int64_t E, int H,
                       const float* __restrict__ carry_seq, Saved<Cell::S> act, float* __restrict__ d_gi, float* __restrict__ d_gh_seq,
                       float* __restrict__ d_carry0) {
  constexpr int R = kClusterR, G = Cell::G, NC = Cell::kC ? 2 : 1;
  constexpr int NB = G;                             // column blocks of this CTA's G Hq columns (one gate each)
  cg::cluster_group cluster = cg::this_cluster();
  const int q = (int)cluster.block_rank();
  extern __shared__ __align__(16) float gsm[];
  const int Hq = H / 2, nl = G * Hq;
  float* Ws = gsm;                                  // [H][nl + 1]  (this CTA's columns)
  float* dgT = Ws + ClusterSmem<Cell>::w_floats(H); // [nl][R]     d(gh_t) of this CTA's units, column-major
  float* part = dgT + (size_t)nl * R;               // [NB][R][H]  partial d(gh) W_h^T over this CTA's column blocks
  float* inbox = part + (size_t)NB * R * H;         // [2][R][Hq]  the peer's partial sums for MY units (two alternating buffers)
  float* dh_rec = inbox + 2 * (size_t)R * Hq;       // [R][Hq]     d(hp) arriving from step t + 1 (already masked by its reset)
  float* dc_rec = dh_rec + (size_t)R * Hq;          // [R][Hq]     d(cp) alike (LSTM)
  float* inbox_peer = cluster.map_shared_rank(inbox, q ^ 1);
  const int64_t row0 = (int64_t)(blockIdx.x / 2) * R;
  const int64_t eh = E * (int64_t)H;
  const int items = Hq * R;
  load_w(Ws, w_h, H, Hq, q, G);
  for (int i = threadIdx.x; i < items; i += blockDim.x) {
    dh_rec[i] = 0.f;
    if constexpr (Cell::kC) dc_rec[i] = 0.f;
  }
  const int i0 = threadIdx.x;
  const int r0 = i0 / Hq, jl0 = i0 % Hq;
  const int64_t rowg = row0 + r0;
  const int j0 = q * Hq + jl0;
  float v_dh = 0.f, v_s[Cell::S], v_p = 0.f;
  bool v_cut = false;
  auto request = [&](int t) {
    v_dh = v_p = 0.f, v_cut = false;
#pragma unroll
    for (int g = 0; g < Cell::S; ++g) v_s[g] = 0.f;
    if (i0 < items && rowg < E && t >= 0) {
      const int64_t o = (int64_t)t * eh + rowg * H + j0;
      v_dh = __ldg(d_h_seq + o);
#pragma unroll
      for (int g = 0; g < Cell::S; ++g) v_s[g] = __ldg(act.p[g] + o);
      v_p = __ldg(carry_seq + o);
      v_cut = reset[(int64_t)t * E + rowg] != 0;
    }
  };
  request(T - 1);
  cluster.sync();
  for (int t = T - 1; t >= 0; --t) {
    const bool cut_t = v_cut;
    float direct = 0.f;
    if (i0 < items) {
      float dy[G] = {};
      if (rowg < E) {
        float dx[G], dc = 0.f;
        if constexpr (Cell::kC) dc = dc_rec[r0 * Hq + jl0];
        direct = Cell::bwd(v_dh + dh_rec[r0 * Hq + jl0], dc, v_p, v_s, dx, dy);
        float* a = d_gi + ((int64_t)t * E + rowg) * G * H + j0;
#pragma unroll
        for (int g = 0; g < G; ++g) a[g * H] = dx[g];
        if constexpr (Cell::kBhn) {
          float* b = d_gh_seq + ((int64_t)t * E + rowg) * G * H + j0;
#pragma unroll
          for (int g = 0; g < G; ++g) b[g * H] = dy[g];
        }
      }
#pragma unroll
      for (int g = 0; g < G; ++g) dgT[(size_t)(g * Hq + jl0) * R + r0] = dy[g];
    }
    request(t - 1);
    __syncthreads();
    if ((int)threadIdx.x < NB * H) {           // partial d(gh) W_h^T over this CTA's columns, for ALL H outputs k
      const int k = threadIdx.x % H, blk = threadIdx.x / H;
      const int kcol = (nl + NB - 1) / NB;     // = Hq; in this form the LSTM backward runs faster than with c0 + Hq
      const int c0 = blk * kcol, c1 = (c0 + kcol < nl) ? c0 + kcol : nl;
      float2 a01 = make_float2(0.f, 0.f), a23 = make_float2(0.f, 0.f);
      const float* wrow = Ws + (size_t)k * (nl + 1);
#pragma unroll 4
      for (int nn = c0; nn < c1; ++nn) {
        const float w = wrow[nn];
        const float4 dv = *reinterpret_cast<const float4*>(dgT + (size_t)nn * R);
        fma2(a01, w, make_float2(dv.x, dv.y)), fma2(a23, w, make_float2(dv.z, dv.w));
      }
      const float acc[R] = {a01.x, a01.y, a23.x, a23.y};
#pragma unroll
      for (int r = 0; r < R; ++r) part[((size_t)blk * R + r) * H + k] = acc[r];
    }
    __syncthreads();
    // my partial for the PEER's units goes into its inbox; my partial for my own units stays in a register
    float mine = 0.f;
    float* box = inbox + (size_t)(t & 1) * R * Hq;
    if (i0 < items) {
      float other = 0.f;
      const int jp = (q ^ 1) * Hq + jl0;
#pragma unroll
      for (int blk = 0; blk < NB; ++blk) {   // fixed order
        mine += part[((size_t)blk * R + r0) * H + j0];
        other += part[((size_t)blk * R + r0) * H + jp];
      }
      inbox_peer[(size_t)(t & 1) * R * Hq + r0 * Hq + jl0] = other;
    }
    cluster.sync();
    if (i0 < items) {
      const float theirs = box[r0 * Hq + jl0];
      float dhp = (q == 0) ? (mine + theirs) : (theirs + mine);   // rank-0 partial first on both CTAs
      const bool keep = rowg < E && !cut_t;                       // base.py:139-148: the reset of step t cuts the chain
      if constexpr (Cell::kC) dc_rec[r0 * Hq + jl0] = keep ? direct : 0.f;
      else dhp = direct + dhp;
      dh_rec[r0 * Hq + jl0] = keep ? dhp : 0.f;
    }
    __syncthreads();
  }
  if (d_carry0 && i0 < items && rowg < E) {
    if constexpr (Cell::kC) d_carry0[rowg * 2 * H + j0] = dc_rec[r0 * Hq + jl0];
    d_carry0[rowg * NC * H + (NC - 1) * H + j0] = dh_rec[r0 * Hq + jl0];
  }
  cluster.sync();   // no CTA exits while its peer may still write into its shared memory
}

// ---- form selection -----------------------------------------------------------------------------------------------------
constexpr size_t kSmemLimit = 227 * 1024;
constexpr int kPersistentMinT = 4;   // below: short sequences (the rollout's T = 1 step) do not amortise filling shared memory with W_h

template <class Cell>
inline int cluster_threads(int H) { return ((kClusterKS * Cell::G * (H / 2) + 31) / 32) * 32; }

template <class Cell>
inline bool cluster_ok(int H, int64_t E) {
  static const bool enabled = env_on(Cell::kClusterEnv);
  const int th = cluster_threads<Cell>(H);
  return enabled && Cell::cluster_rows_ok(E) && H >= 2 && H % 2 == 0 && th <= 1024 && (H / 2) * kClusterR <= th && Cell::G * H <= th &&
         ClusterSmem<Cell>::fwd_bytes(H) <= kSmemLimit && ClusterSmem<Cell>::bwd_bytes(H) <= kSmemLimit;
}

// launch shape: R = 8 rows per CTA from 1024 sequences up (the rollout step), else 4 with the reduction split over two thread groups
inline int gru_threads(int H, int ks) { return ((ks * 3 * H + 31) / 32) * 32; }
inline bool gru_persistent_ok(int H) {
  static const bool enabled = env_on("STX_GRU_PERSISTENT");
  return enabled && H >= 2 && gru_threads(H, 2) <= 1024 && GruSmem<8, 1>::fwd_bytes(H) <= kSmemLimit && GruSmem<8, 1>::bwd_bytes(H) <= kSmemLimit &&
         GruSmem<4, 2>::fwd_bytes(H) <= kSmemLimit && GruSmem<4, 2>::bwd_bytes(H) <= kSmemLimit;
}

enum class Form { kCluster, kPersistent, kPerStep };

template <class Cell>
Form form_of(int T, int64_t E, int H) {
  if (T < kPersistentMinT) return Form::kPerStep;
  if (cluster_ok<Cell>(H, E)) return Form::kCluster;
  if (Cell::kPersistent && gru_persistent_ok(H)) return Form::kPersistent;
  return Form::kPerStep;
}

template <typename... KArgs, typename... Args>
inline cudaError_t launch_cluster2(void (*kernel)(KArgs...), unsigned clusters, int threads, size_t smem, cudaStream_t st, Args... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(2 * clusters), cfg.blockDim = dim3(threads), cfg.dynamicSmemBytes = smem, cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 2, attr[0].val.clusterDim.y = 1, attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr, cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, args...);
}

// ---- drivers ------------------------------------------------------------------------------------------------------------
template <class Cell>
size_t workspace_bytes(int T, int64_t E, int H) {
  if (T <= 0 || E <= 0 || H <= 0) return 0;
  return carve<Cell>(T, E, H, nullptr).bytes;
}

// carry0: (E, H) h0 (GRU) or (E, 2H) = (c | h) (LSTM); b_hn and carry_last: GRU / LSTM only
template <class Cell>
int sequence_forward(const char* fn, const float* gi, const uint8_t* reset, const float* carry0, const float* w_h, const float* b_hn, int T, int64_t E,
                     int H, float* h_seq, float* carry_last, void* workspace, size_t workspace_bytes_, cudaStream_t st) {
  constexpr int G = Cell::G;
  STX_REQUIRE(T > 0 && E > 0 && H > 0, STX_E_SHAPE, "%s: T=%d E=%lld H=%d", fn, T, (long long)E, H);
  STX_REQUIRE(workspace_bytes_ >= workspace_bytes<Cell>(T, E, H), STX_E_WORKSPACE, "%s: workspace %zu < %zu", fn, workspace_bytes_,
              workspace_bytes<Cell>(T, E, H));
  const SeqWs<Cell> ws = carve<Cell>(T, E, H, reinterpret_cast<char*>(workspace));
  const size_t eh = (size_t)E * H;
  const unsigned blocks = (unsigned)((eh + 255) / 256);
  switch (form_of<Cell>(T, E, H)) {
    case Form::kCluster:
      STX_CUDA_OK(opt_in_smem<cluster_fwd_kernel<Cell>>(kSmemLimit));
      STX_CUDA_OK(launch_cluster2(cluster_fwd_kernel<Cell>, (unsigned)((E + kClusterR - 1) / kClusterR), cluster_threads<Cell>(H),
                                  ClusterSmem<Cell>::fwd_bytes(H), st, gi, reset, carry0, w_h, b_hn, T, E, H, h_seq, carry_last, ws.hp_seq, ws.cp_seq,
                                  ws.act));
      STX_LAUNCH_OK();
      return STX_OK;
    case Form::kPersistent:
      if constexpr (Cell::kPersistent) {
        if (E >= 1024) {
          STX_CUDA_OK(opt_in_smem<gru_seq_fwd_kernel<8, 1>>(kSmemLimit));
          gru_seq_fwd_kernel<8, 1><<<(unsigned)((E + 7) / 8), gru_threads(H, 1), GruSmem<8, 1>::fwd_bytes(H), st>>>(gi, reset, carry0, w_h, b_hn, T, E, H,
                                                                                                                      h_seq, ws.hp_seq, ws.act);
        } else {
          STX_CUDA_OK(opt_in_smem<gru_seq_fwd_kernel<4, 2>>(kSmemLimit));
          gru_seq_fwd_kernel<4, 2><<<(unsigned)((E + 3) / 4), gru_threads(H, 2), GruSmem<4, 2>::fwd_bytes(H), st>>>(gi, reset, carry0, w_h, b_hn, T, E, H,
                                                                                                                      h_seq, ws.hp_seq, ws.act);
        }
        STX_LAUNCH_OK();
        return STX_OK;
      }
      [[fallthrough]];   // form_of picks the persistent form only for a cell that has one
    case Form::kPerStep:
      break;
  }
  step_init_kernel<Cell><<<blocks, 256, 0, st>>>(carry0, reset, E, H, ws.hp_seq, ws.cp_seq);
  STX_LAUNCH_OK();
  for (int t = 0; t < T; ++t) {
    simt::GemmArgs g{};
    g.A = ws.hp_seq + (size_t)t * eh, g.lda = H, g.B = w_h, g.C = ws.gh, g.mask_act = -1;
    g.M = E, g.N = G * H, g.K = H;
    STX_CUDA_OK(simt::launch_gemm<simt::FWD>(g, 1, st));
    const size_t o = (size_t)t * eh;
    float* cp = Cell::kC ? ws.cp_seq + o : nullptr;
    step_fwd_kernel<Cell><<<blocks, 256, 0, st>>>(gi + o * G, ws.gh, b_hn, ws.hp_seq + o, cp, t + 1 < T ? reset + (size_t)(t + 1) * E : nullptr, E, H,
                                                  h_seq + o, ws.hp_seq + o + eh, Cell::kC ? cp + eh : nullptr, ws.act.at(o),
                                                  t == T - 1 ? carry_last : nullptr);
    STX_LAUNCH_OK();
  }
  return STX_OK;
}

// d_b_hn: GRU only, with d_w_h; d_carry0 shaped like carry0
template <class Cell>
int sequence_backward(const char* fn, const float* d_h_seq, const uint8_t* reset, const float* w_h, int T, int64_t E, int H, void* workspace,
                      size_t workspace_bytes_, float* d_gi, float* d_w_h, float* d_b_hn, float grad_weight, int overwrite, float* d_carry0,
                      cudaStream_t st) {
  constexpr int G = Cell::G;
  STX_REQUIRE(T > 0 && E > 0 && H > 0, STX_E_SHAPE, "%s: T=%d E=%lld H=%d", fn, T, (long long)E, H);
  STX_REQUIRE(workspace_bytes_ >= workspace_bytes<Cell>(T, E, H), STX_E_WORKSPACE, "%s: workspace %zu < %zu", fn, workspace_bytes_,
              workspace_bytes<Cell>(T, E, H));
  const SeqWs<Cell> ws = carve<Cell>(T, E, H, reinterpret_cast<char*>(workspace));
  const size_t eh = (size_t)E * H;
  const unsigned blocks = (unsigned)((eh + 255) / 256);
  float* dgh_seq = Cell::kBhn ? ws.d_gh_seq : d_gi;              // d(gh) of every step: the operand of the DX and d(W_h) GEMMs
  const float* carry_seq = Cell::kC ? ws.cp_seq : ws.hp_seq;     // the carry the cell's backward reads
  switch (form_of<Cell>(T, E, H)) {
    case Form::kCluster:
      STX_CUDA_OK(opt_in_smem<cluster_bwd_kernel<Cell>>(kSmemLimit));
      STX_CUDA_OK(launch_cluster2(cluster_bwd_kernel<Cell>, (unsigned)((E + kClusterR - 1) / kClusterR), cluster_threads<Cell>(H),
                                  ClusterSmem<Cell>::bwd_bytes(H), st, d_h_seq, reset, w_h, T, E, H, carry_seq, ws.act, d_gi, ws.d_gh_seq, d_carry0));
      STX_LAUNCH_OK();
      break;
    case Form::kPersistent:
      if constexpr (Cell::kPersistent) {
        if (E >= 1024) {
          STX_CUDA_OK(opt_in_smem<gru_seq_bwd_kernel<8, 1>>(kSmemLimit));
          gru_seq_bwd_kernel<8, 1><<<(unsigned)((E + 7) / 8), gru_threads(H, 1), GruSmem<8, 1>::bwd_bytes(H), st>>>(d_h_seq, reset, w_h, T, E, H, ws.hp_seq,
                                                                                                                      ws.act, d_gi, ws.d_gh_seq, d_carry0);
        } else {
          STX_CUDA_OK(opt_in_smem<gru_seq_bwd_kernel<4, 2>>(kSmemLimit));
          gru_seq_bwd_kernel<4, 2><<<(unsigned)((E + 3) / 4), gru_threads(H, 2), GruSmem<4, 2>::bwd_bytes(H), st>>>(d_h_seq, reset, w_h, T, E, H, ws.hp_seq,
                                                                                                                      ws.act, d_gi, ws.d_gh_seq, d_carry0);
        }
        STX_LAUNCH_OK();
        break;
      }
      [[fallthrough]];   // form_of picks the persistent form only for a cell that has one
    case Form::kPerStep:
      for (int t = T - 1; t >= 0; --t) {
        const bool last = (t == T - 1);
        const size_t o = (size_t)t * eh;
        step_bwd_kernel<Cell><<<blocks, 256, 0, st>>>(d_h_seq + o, last ? nullptr : ws.dhp_gemm, ws.direct[(t + 1) & 1],
                                                      last ? nullptr : reset + (size_t)(t + 1) * E, ws.act.at(o), carry_seq + o, E, H, d_gi + o * G,
                                                      Cell::kBhn ? ws.d_gh_seq + o * G : nullptr, ws.direct[t & 1]);
        STX_LAUNCH_OK();
        if (t > 0 || d_carry0) {  // d(hp_t) through W_h: dX form, W_h is (H x G H) "Kout x Nr"
          simt::GemmArgs d{};
          d.A = dgh_seq + (size_t)t * G * eh, d.lda = G * H, d.B = w_h, d.C = ws.dhp_gemm, d.mask_act = -1;
          d.M = E, d.N = H, d.K = G * H;
          STX_CUDA_OK(simt::launch_gemm<simt::DX>(d, 1, st));
        }
      }
      if (d_carry0) {
        step_dcarry0_kernel<Cell><<<blocks, 256, 0, st>>>(ws.dhp_gemm, ws.direct[0], reset, E, H, d_carry0);
        STX_LAUNCH_OK();
      }
      break;
  }
  if (d_w_h) {
    // d(W_h) = hp_seq^T d(gh)_seq over all (t, e) rows; GRU: column sums of the n part = d(b_hn)
    const int64_t rows = (int64_t)T * E;
    const int64_t nw = (int64_t)H * G * H;
    const int64_t np = nw + (Cell::kBhn ? G * H : 0);
    simt::GemmArgs g{};
    g.A = ws.hp_seq, g.lda = H, g.B = dgh_seq, g.C = ws.partials, g.dbias = Cell::kBhn ? ws.partials + nw : nullptr, g.mask_act = -1;
    g.M = rows, g.N = G * H, g.K = H;
    g.rows_per_split = (rows + ws.splits - 1) / ws.splits;
    g.part_stride = np, g.dbias_stride = np;
    STX_CUDA_OK(simt::launch_gemm<simt::DW>(g, ws.splits, st));
    simt::reduce_partials_kernel<<<(unsigned)((nw + 255) / 256), 256, 0, st>>>(ws.partials, ws.splits, np, nw, grad_weight, d_w_h, overwrite);
    STX_LAUNCH_OK();
    if (Cell::kBhn) {
      simt::reduce_partials_kernel<<<(unsigned)((H + 255) / 256), 256, 0, st>>>(ws.partials + nw + 2 * H, ws.splits, np, H, grad_weight, d_b_hn, overwrite);
      STX_LAUNCH_OK();
    }
  }
  return STX_OK;
}

}  // namespace
}  // namespace stx

using namespace stx;

extern "C" size_t stx_gru_workspace_bytes(int T, int64_t E, int H) { return workspace_bytes<GruCell>(T, E, H); }

extern "C" int stx_gru_sequence_forward(const float* gi, const uint8_t* reset, const float* h0, const float* w_h, const float* b_hn, int T, int64_t E,
                                        int H, float* h_seq, void* workspace, size_t workspace_bytes, void* stream) {
  STX_REQUIRE(gi && reset && h0 && w_h && b_hn && h_seq && workspace, STX_E_ARG, "stx_gru_sequence_forward: null pointer");
  return sequence_forward<GruCell>("stx_gru_sequence_forward", gi, reset, h0, w_h, b_hn, T, E, H, h_seq, nullptr, workspace, workspace_bytes,
                                   (cudaStream_t)stream);
}

extern "C" int stx_gru_sequence_backward(const float* d_h_seq, const uint8_t* reset, const float* w_h, int T, int64_t E, int H, void* workspace,
                                         size_t workspace_bytes, float* d_gi, float* d_w_h, float* d_b_hn, float grad_weight, int overwrite,
                                         float* d_h0, void* stream) {
  STX_REQUIRE(d_h_seq && reset && w_h && workspace && d_gi, STX_E_ARG, "stx_gru_sequence_backward: null pointer");
  STX_REQUIRE((d_w_h == nullptr) == (d_b_hn == nullptr), STX_E_ARG, "stx_gru_sequence_backward: d_w_h and d_b_hn go together");
  return sequence_backward<GruCell>("stx_gru_sequence_backward", d_h_seq, reset, w_h, T, E, H, workspace, workspace_bytes, d_gi, d_w_h, d_b_hn,
                                    grad_weight, overwrite, d_h0, (cudaStream_t)stream);
}

extern "C" size_t stx_lstm_workspace_bytes(int T, int64_t E, int H) { return workspace_bytes<LstmCell>(T, E, H); }

extern "C" int stx_lstm_sequence_forward(const float* gi, const uint8_t* reset, const float* carry0, const float* w_h, int T, int64_t E, int H,
                                         float* h_seq, float* carry_last, void* workspace, size_t workspace_bytes, void* stream) {
  STX_REQUIRE(gi && reset && carry0 && w_h && h_seq && workspace, STX_E_ARG, "stx_lstm_sequence_forward: null pointer");
  return sequence_forward<LstmCell>("stx_lstm_sequence_forward", gi, reset, carry0, w_h, nullptr, T, E, H, h_seq, carry_last, workspace,
                                    workspace_bytes, (cudaStream_t)stream);
}

extern "C" int stx_lstm_sequence_backward(const float* d_h_seq, const uint8_t* reset, const float* w_h, int T, int64_t E, int H, void* workspace,
                                          size_t workspace_bytes, float* d_gi, float* d_w_h, float grad_weight, int overwrite, float* d_carry0,
                                          void* stream) {
  STX_REQUIRE(d_h_seq && reset && w_h && workspace && d_gi, STX_E_ARG, "stx_lstm_sequence_backward: null pointer");
  return sequence_backward<LstmCell>("stx_lstm_sequence_backward", d_h_seq, reset, w_h, T, E, H, workspace, workspace_bytes, d_gi, d_w_h, nullptr,
                                     grad_weight, overwrite, d_carry0, (cudaStream_t)stream);
}
