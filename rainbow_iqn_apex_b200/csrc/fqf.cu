// FQF (Yang et al., NeurIPS 2019): the fraction proposal's softmax / cumsum, the backward of its 1-Wasserstein fraction
// loss, the fraction layer's weight gradient and the Delta-tau weighted argmax.  The logits product itself runs on the
// fp32 SIMT GEMM (riqn_linear_fwd_ld); see include/riqn_b200.h for the statements.
//
// Every per-sample sum runs in double in a fixed order (one warp per sample, sequential loops on lane 0 where the order
// is part of the contract), so the results are bitwise reproducible and independent of the launch shape.
#include <math.h>

#include "common.cuh"
#include "../../include/riqn_b200.h"

namespace riqn {

constexpr int FQF_MAX_N = 256;
constexpr int FQF_WARPS = 4;      // samples per CTA

// e[k] = exp(logit_k - max) in double for one sample, lanes strided over k; returns max (exact: a max has no order).
__device__ __forceinline__ float fqf_exp_shift(int n, const float* __restrict__ lg, double* __restrict__ e, int lane) {
  float m = -INFINITY;
  for (int k = lane; k < n; k += 32) m = fmaxf(m, lg[k]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  for (int k = lane; k < n; k += 32) e[k] = exp((double)lg[k] - (double)m);
  __syncwarp();
  return m;
}

// ------------------------------------------------------------------------------------------------
// Fractions: P = softmax(logits), tau_i = sum_{k<i} P_k, tau_hat, dtau, H(P)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(32 * FQF_WARPS)
fqf_fractions_kernel(int B, int n, const float* __restrict__ logits, float* __restrict__ tau, float* __restrict__ tau_hat,
                     float* __restrict__ dtau, float* __restrict__ entropy) {
  __shared__ double s_e[FQF_WARPS][FQF_MAX_N];
  __shared__ double s_c[FQF_WARPS][FQF_MAX_N + 1];
  __shared__ float s_t[FQF_WARPS][FQF_MAX_N + 1];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.x * FQF_WARPS + w;
  if (b >= B) return;
  const float* lg = logits + (long)b * n;
  double* e = s_e[w];
  double* c = s_c[w];
  float* t = s_t[w];
  const float m = fqf_exp_shift(n, lg, e, lane);
  if (lane == 0) {
    // c_i = sum_{k<i} e_k, k ascending; S = c_n.  Every term is >= 0, so c is non-decreasing and c_i <= S.
    double acc = 0.0, ed = 0.0;
    c[0] = 0.0;
    for (int k = 0; k < n; ++k) {
      acc += e[k];
      c[k + 1] = acc;
      ed += e[k] * ((double)lg[k] - (double)m);
    }
    // H = -sum P_k log P_k = log S - sum_k P_k (l_k - max): no log of an underflowed P_k
    if (entropy != nullptr) entropy[b] = (float)(log(acc) - ed / acc);
  }
  __syncwarp();
  const double S = c[n];
  for (int i = lane; i <= n; i += 32) {
    // rounded once; c_i / S is monotone in c_i, and c_n / S == 1 exactly
    const float v = i == 0 ? 0.f : (i == n ? 1.f : (float)(c[i] / S));
    t[i] = v;
    tau[(long)b * (n + 1) + i] = v;
  }
  __syncwarp();
  for (int i = lane; i < n; i += 32) {
    const float lo = t[i], hi = t[i + 1];
    tau_hat[(long)i * B + b] = 0.5f * (lo + hi);
    dtau[(long)i * B + b] = hi - lo;            // >= 0: lo <= hi
  }
}

// ------------------------------------------------------------------------------------------------
// Fraction-loss backward (W1 gradient, suffix sums, softmax / entropy Jacobian)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(32 * FQF_WARPS)
fqf_fraction_bwd_kernel(int B, int n, int A, const float* __restrict__ logits, const float* __restrict__ tau,
                        const float* __restrict__ q_hat, const float* __restrict__ q_bnd, const int64_t* __restrict__ actions,
                        const float* __restrict__ gscale, float gscale_mul, float entropy_coef, float* __restrict__ dlogits,
                        float* __restrict__ loss_out) {
  __shared__ double s_e[FQF_WARPS][FQF_MAX_N];
  __shared__ double s_g[FQF_WARPS][FQF_MAX_N];     // g_i, then G_k = sum_{i>k} g_i
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.x * FQF_WARPS + w;
  if (b >= B) return;
  const float* lg = logits + (long)b * n;
  const float* tb = tau + (long)b * (n + 1);
  double* e = s_e[w];
  double* g = s_g[w];
  const int a = (int)actions[b];
  const float m = fqf_exp_shift(n, lg, e, lane);
  // g_i = 2 F(tau_i) - F(tau_hat_i) - F(tau_hat_{i-1}), i = 1..n-1, each in double from the fp32 quantile values
  for (int i = lane; i < n; i += 32) {
    double gi = 0.0;
    if (i > 0)
      gi = 2.0 * (double)q_bnd[((long)(i - 1) * B + b) * A + a] - (double)q_hat[((long)i * B + b) * A + a] -
           (double)q_hat[((long)(i - 1) * B + b) * A + a];
    g[i] = gi;
  }
  __syncwarp();
  __shared__ double s_red[FQF_WARPS][4];
  if (lane == 0) {
    double S = 0.0, ed = 0.0, surr = 0.0;
    for (int k = 0; k < n; ++k) {
      S += e[k];
      ed += e[k] * ((double)lg[k] - (double)m);
    }
    for (int i = 1; i < n; ++i) surr += g[i] * (double)tb[i];
    // suffix sums, k descending: G_{n-1} = 0, G_k = G_{k+1} + g_{k+1}
    double run = 0.0;
    for (int k = n - 1; k >= 0; --k) {
      const double gk = g[k];
      g[k] = run;
      run += gk;
    }
    double pg = 0.0;                                  // sum_m P_m G_m, m ascending
    for (int k = 0; k < n; ++k) pg += (e[k] / S) * g[k];
    const double H = log(S) - ed / S;
    s_red[w][0] = S;
    s_red[w][1] = pg;
    s_red[w][2] = H;
    s_red[w][3] = log(S);
    if (loss_out != nullptr) loss_out[b] = (float)(surr - (double)entropy_coef * H);
  }
  __syncwarp();
  const double S = s_red[w][0], pg = s_red[w][1], H = s_red[w][2], logS = s_red[w][3];
  const double wt = (double)(gscale != nullptr ? gscale[b] : 1.f) * (double)gscale_mul;
  for (int k = lane; k < n; k += 32) {
    const double P = e[k] / S;
    const double logP = ((double)lg[k] - (double)m) - logS;
    const double d = P * (g[k] - pg) + (double)entropy_coef * P * (logP + H);
    dlogits[(long)b * n + k] = (float)(wt * d);
  }
}

// ------------------------------------------------------------------------------------------------
// Fraction-layer weight gradient: grad_w[k, j] += sum_b dl[b, k] feat[b, j], grad_b[k] += sum_b dl[b, k]  (b ascending)
// ------------------------------------------------------------------------------------------------
constexpr int WG_KT = 16, WG_JT = 128;

__global__ void __launch_bounds__(WG_JT)
fqf_wgrad_kernel(int B, int n, int F, const float* __restrict__ dl, const float* __restrict__ feat, float* __restrict__ grad_w,
                 float* __restrict__ grad_b) {
  const int j = blockIdx.x * WG_JT + threadIdx.x;
  const int k0 = blockIdx.y * WG_KT;
  float acc[WG_KT];
#pragma unroll
  for (int kk = 0; kk < WG_KT; ++kk) acc[kk] = 0.f;
  if (j < F) {
    for (int b = 0; b < B; ++b) {
      const float f = __ldg(&feat[(long)b * F + j]);
      const float* d = dl + (long)b * n + k0;
#pragma unroll
      for (int kk = 0; kk < WG_KT; ++kk)
        if (k0 + kk < n) acc[kk] = fmaf(__ldg(&d[kk]), f, acc[kk]);
    }
#pragma unroll
    for (int kk = 0; kk < WG_KT; ++kk)
      if (k0 + kk < n) grad_w[(long)(k0 + kk) * F + j] += acc[kk];
  }
  if (blockIdx.x == 0 && threadIdx.x < WG_KT && k0 + (int)threadIdx.x < n) {
    const int k = k0 + threadIdx.x;
    float s = 0.f;
    for (int b = 0; b < B; ++b) s += dl[(long)b * n + k];
    grad_b[k] += s;
  }
}

// ------------------------------------------------------------------------------------------------
// a*[b] = argmax_a sum_k w[k*B+b] q[k*B+b, a]   (k ascending, fmaf; first maximal index wins)
// ------------------------------------------------------------------------------------------------
__global__ void argmax_weighted_kernel(int B, int K, int A, const float* __restrict__ q, const float* __restrict__ wk,
                                       int64_t* __restrict__ a_star) {
  const int b = (int)(((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (b >= B) return;
  float s = -INFINITY;
  if (lane < A) {
    s = 0.f;
    for (int k = 0; k < K; ++k) s = fmaf(wk[(long)k * B + b], q[((long)k * B + b) * A + lane], s);
  }
  float best = s;
  int arg = lane;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oa = __shfl_xor_sync(0xffffffffu, arg, o);
    if (ob > best || (ob == best && oa < arg)) { best = ob; arg = oa; }
  }
  if (lane == 0) a_star[b] = arg;
}

static inline bool fqf_n_ok(int n) { return n >= 2 && n <= FQF_MAX_N; }

}  // namespace riqn

using namespace riqn;

RIQN_API int riqn_fqf_fractions(int batch, int n, const float* logits, float* tau, float* tau_hat, float* dtau,
                                float* entropy, void* stream) {
  if (batch < 1 || !fqf_n_ok(n)) return (int)cudaErrorInvalidValue;
  riqn::note_launches(1);
  fqf_fractions_kernel<<<riqn_cdiv(batch, FQF_WARPS), 32 * FQF_WARPS, 0, (cudaStream_t)stream>>>(batch, n, logits, tau,
                                                                                                 tau_hat, dtau, entropy);
  return (int)cudaGetLastError();
}

RIQN_API int riqn_fqf_fraction_bwd(int batch, int n, int action_space, const float* logits, const float* tau,
                                   const float* q_hat, const float* q_bnd, const long long* actions, const float* gscale,
                                   float gscale_mul, float entropy_coef, float* dlogits, float* loss_out, void* stream) {
  if (batch < 1 || !fqf_n_ok(n) || action_space < 1 || action_space > 32 || !isfinite(gscale_mul) ||
      !isfinite(entropy_coef) || !(entropy_coef >= 0.f))
    return (int)cudaErrorInvalidValue;
  riqn::note_launches(1);
  fqf_fraction_bwd_kernel<<<riqn_cdiv(batch, FQF_WARPS), 32 * FQF_WARPS, 0, (cudaStream_t)stream>>>(
      batch, n, action_space, logits, tau, q_hat, q_bnd, (const int64_t*)actions, gscale, gscale_mul, entropy_coef, dlogits,
      loss_out);
  return (int)cudaGetLastError();
}

RIQN_API int riqn_fqf_fraction_wgrad(int batch, int n, int feat_dim, const float* dlogits, const float* feat, float* grad_w,
                                     float* grad_b, void* stream) {
  if (batch < 1 || !fqf_n_ok(n) || feat_dim < 1) return (int)cudaErrorInvalidValue;
  riqn::note_launches(1);
  dim3 grid(riqn_cdiv(feat_dim, WG_JT), riqn_cdiv(n, WG_KT));
  fqf_wgrad_kernel<<<grid, WG_JT, 0, (cudaStream_t)stream>>>(batch, n, feat_dim, dlogits, feat, grad_w, grad_b);
  return (int)cudaGetLastError();
}

RIQN_API int riqn_linear_wgrad(int batch, int n, int feat_dim, const float* dy, const float* x, float* grad_w,
                               float* grad_b, void* stream) {
  if (batch < 1 || n < 1 || feat_dim < 1 || !dy || !x || !grad_w || !grad_b) return (int)cudaErrorInvalidValue;
  riqn::note_launches(1);
  dim3 grid(riqn_cdiv(feat_dim, WG_JT), riqn_cdiv(n, WG_KT));
  fqf_wgrad_kernel<<<grid, WG_JT, 0, (cudaStream_t)stream>>>(batch, n, feat_dim, dy, x, grad_w, grad_b);
  return (int)cudaGetLastError();
}

RIQN_API int riqn_argmax_weighted(int batch, int n, int action_space, const float* q, const float* w, long long* a_star,
                                  void* stream) {
  if (batch < 1 || !fqf_n_ok(n) || action_space < 1 || action_space > 32) return (int)cudaErrorInvalidValue;
  riqn::note_launches(1);
  argmax_weighted_kernel<<<riqn_cdiv((long)batch * 32, 128), 128, 0, (cudaStream_t)stream>>>(batch, n, action_space, q, w,
                                                                                              (int64_t*)a_star);
  return (int)cudaGetLastError();
}
