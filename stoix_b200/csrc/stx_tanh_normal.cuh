// Device arithmetic of the tanh-Normal policy head (NormalAffineTanhDistributionHead, stoix/networks/heads.py:44-65, on
// AffineTanhTransformedDistribution, stoix/networks/distributions.py:19-89), shared by the SAC kernels (stx_sac.cu) and the
// fp32 PPO loss kernels (stx_ppo_loss.cuh, stx_ppo_fp32.cu).  tfp pieces restated from their published definitions: Normal.log_prob,
// log_cdf / log_survival_function, bijectors.Tanh.forward_log_det_jacobian(x) = 2 (log 2 - x - softplus(-2x)).
#pragma once
#include "stx_common.cuh"

namespace stx {

constexpr float kLogSqrt2Pi = 0.9189385332046727f;
constexpr float kTanhNormalEpsilon = 1e-3f;  // the clip band of AffineTanhTransformedDistribution (distributions.py:28)

__device__ __forceinline__ float softplusf(float x) { return fmaxf(x, 0.f) + log1pf(expf(-fabsf(x))); }
__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }
// log Phi(z) = log(0.5 erfc(-z / sqrt 2)); erfcx keeps the far tail finite
__device__ __forceinline__ float log_ndtrf(float z) {
  const float t = -z * 0.70710678118654752f;
  if (t < 3.f) return logf(0.5f * erfcf(t));
  return logf(0.5f * erfcxf(t)) - t * t;
}
// phi(z) / Phi(z).  Far in the left tail it is sqrt(2/pi) / erfcx(t), t = -z / sqrt 2, exactly.  The exp form below cancels
// -z^2/2 against the -t^2 of log_ndtrf, so the rounding of t leaves a relative error that grows as 2^-24 z^2 (about 5e-5 at
// z = -50, 5e-4 at z = -200, 6e-2 at z = -1500).  The switch sits at t = 64 (z = -90.5); below it the exp form is kept, so
// every gradient whose z stays above -90.5 is unchanged bit for bit.
constexpr float kMillsErfcxFrom = 64.f;
__device__ __forceinline__ float mills(float z) {
  const float t = -z * 0.70710678118654752f;
  if (t < kMillsErfcxFrom) return expf(-0.5f * z * z - kLogSqrt2Pi - log_ndtrf(z));
  return 0.7978845608028654f / erfcxf(t);
}
// forward log-det-Jacobian of tanh at x
__device__ __forceinline__ float tanh_fldj(float x) { return 2.f * (0.6931471805599453f - x - softplusf(-2.f * x)); }

struct HeadGeom {
  float s, sh, lo, hi, u_lo, u_hi, log_s, log_eps;
};
__device__ __forceinline__ HeadGeom head_geom(float minimum, float maximum, float epsilon) {
  HeadGeom g;
  g.s = 0.5f * (maximum - minimum), g.sh = 0.5f * (minimum + maximum);
  g.lo = minimum + epsilon, g.hi = maximum - epsilon;
  g.u_lo = atanhf((g.lo - g.sh) / g.s), g.u_hi = atanhf((g.hi - g.sh) / g.s);
  g.log_s = logf(g.s), g.log_eps = logf(epsilon);
  return g;
}

// One action dimension of log_prob(a) for a GIVEN event a (the inverse path, distributions.py:56-80) and its derivatives
// with respect to loc and sigma (the event held fixed).  The event is clipped to [lo, hi]:
//   a <= lo:  log Phi((u_lo - loc) / sigma) - log eps            d/dloc = -m / sigma, d/dsigma = -m z / sigma
//   a >= hi:  log Phi(-(u_hi - loc) / sigma) - log eps           d/dloc =  m / sigma, d/dsigma = -m z / sigma
//   else:     u = atanh((a - shift) / s), z = (u - loc) / sigma,
//             -z^2/2 - log sigma - log sqrt(2 pi) - fldj(u) - log s    d/dloc = z / sigma, d/dsigma = (z^2 - 1) / sigma
// with m = phi(z) / Phi(z) at the tail's own z.  Callers that only need the value let the compiler drop the rest.
struct TanhNormalDim {
  float lp, d_loc, d_sigma;
};
__device__ __forceinline__ TanhNormalDim tanh_normal_log_prob_given(float loc, float sigma, float a, const HeadGeom& g) {
  TanhNormalDim r;
  const float ev = fminf(fmaxf(a, g.lo), g.hi);
  if (ev <= g.lo) {
    const float z = (g.u_lo - loc) / sigma, m = mills(z);
    r.lp = log_ndtrf(z) - g.log_eps, r.d_loc = -m / sigma, r.d_sigma = -m * z / sigma;
  } else if (ev >= g.hi) {
    const float z = -(g.u_hi - loc) / sigma, m = mills(z);
    r.lp = log_ndtrf(z) - g.log_eps, r.d_loc = m / sigma, r.d_sigma = -m * z / sigma;
  } else {
    const float u = atanhf((ev - g.sh) / g.s), z = (u - loc) / sigma;
    r.lp = -0.5f * z * z - logf(sigma) - kLogSqrt2Pi - tanh_fldj(u) - g.log_s;
    r.d_loc = z / sigma, r.d_sigma = (z * z - 1.f) / sigma;
  }
  return r;
}

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

// ---- the seeded entropy estimate of the PPO losses (stx_ppo_loss.cuh) ----
constexpr uint32_t kTagPpoEntropy = 0x50504f45u;  // "PPOE"

// Entropy noise eps' of row m, dims j0..j0+3 (layout in include/stx.h); eps_in (nullable, (rows, A)) replaces the draw.
__device__ __forceinline__ void entropy_noise(const float* __restrict__ eps_in, int A, uint64_t seed, int64_t m, uint64_t call, int j0, float e[4]) {
  if (eps_in) {
#pragma unroll
    for (int k = 0; k < 4; ++k) e[k] = j0 + k < A ? eps_in[m * A + j0 + k] : 0.f;
    return;
  }
  const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
  const uint4 w = Philox::rand4(make_uint4((uint32_t)m, (uint32_t)call,
                                           (uint32_t)(call >> 32) ^ ((uint32_t)(j0 >> 2) << 20) ^ ((uint32_t)((uint64_t)m >> 32) << 8),
                                           kTagPpoEntropy), key);
  const float2 n0 = normal2(w.x, w.y), n1 = normal2(w.z, w.w);
  e[0] = n0.x, e[1] = n0.y, e[2] = n1.x, e[3] = n1.y;
}

// One dimension of the entropy estimate: Normal entropy + fldj of the Shift / Scale / Tanh chain at the Normal sample.
__device__ __forceinline__ float tanh_normal_entropy_dim(float loc, float sigma, float e, const HeadGeom& g) {
  return 0.5f + kLogSqrt2Pi + logf(sigma) + g.log_s + tanh_fldj(loc + sigma * e);
}

}  // namespace stx
