// MMDQN loss (Nguyen-Tang, Gupta & Venkatesh, "Distributional Reinforcement Learning via Moment Matching", AAAI 2021; no
// counterpart in the reference): the squared maximum mean discrepancy between the n online particles and the n
// Bellman-target particles of a transition under a mixture of Gaussian kernels, and its gradient in the particles.
//   th[b,i]  = q_on[(i*B+b), act[b]]
//   T[b,j]   = R[b] + fl(gamma^n*nt[b]) * q_tgt[(j*B+b), a*[b]]        (RESCALE: fl(h(R + g*h^-1(q_tgt))), as the IQN loss)
//   k(x, y)  = sum_h exp(-(x-y)^2 / h) ,  k1(x, y) = -sum_h (2(x-y)/h) exp(-(x-y)^2 / h)
//   loss[b]  = max(0, (1/n^2) sum_i sum_j [k(th_i, th_j) + k(T_i, T_j) - 2 k(th_i, T_j)])
//   dth[i*B+b] = (2/n^2) sum_j [k1(th_i, th_j) - k1(th_i, T_j)]          (gradient of the unclamped sum; T detached)
// One CTA per transition.  The particles and targets are staged in shared memory; thread i owns th_i and T_i and walks
// j = 0..n-1 ascending; the loss is reduced over i in the fixed warp-and-slot order of the quantile-Huber loss.  No
// atomics, so a step is bitwise reproducible.
//
// Arithmetic, with every operation explicitly rounded (nvcc contracts nothing):
//   c_h = fl(-log2(e) / h), w_h = fl(2 / h)       (host, in double, rounded once to float)
//   for a pair (x, y):  d = fl(x - y) ;  s = fl(d * d) ;  e_h = exp2f(fl(s * c_h))
//   kxy = sum_h e_h ,  G = sum_h fl(w_h * e_h)      (fp32 adds, h ascending, starting from 0)
//   bracket_ij = fl(fl(k_thth + k_TT) - fl(2 k_thT)) ;  g_ij = fl(fl(d_thT * G_thT) - fl(d_thth * G_thth))
//   acc_i = sum_j bracket_ij, gacc_i = sum_j g_ij   (fp32, j ascending, from 0)
//   loss = max(0, fl(S / n^2)), S the warp-and-slot sum of acc_i ;  dth_i = fl(fl(2 gacc_i) / n^2)
// Per-term error model (u = 2^-24): with a = s * log2(e) / h the exact exponent, d carries one rounding, s three, the
// argument fl(s * c_h) five (relative), and exp2f at most 2 ulp, so
//   |e_h - exp(-(x-y)^2/h)| <= exp(-(x-y)^2/h) * (4u + 5u * ln2 * a) + 2^-126     (the last term: an underflowed result)
// and fl(w_h * e_h) adds 2u.  Every sum above then adds at most (its length) * u * (sum of the |terms| it adds).
// T_j = th_j for every j (same values in the same order) gives brackets and g_ij of exactly 0, hence loss and dth 0.
#include "common.cuh"
#include "value_rescaling.cuh"
#include "../../include/riqn_b200.h"

#include <cmath>

namespace riqn {
constexpr int MMD_MAX_N = 256;
constexpr int MMD_MAX_H = 16;

struct MmdBandwidths {     // by value: a captured graph holds the constants
  int H;
  float c[MMD_MAX_H];      // fl(-log2(e) / h)
  float w[MMD_MAX_H];      // fl(2 / h)
};

template <bool RESCALE>
__global__ void mmd_loss_kernel(int B, int n, int A, const float* __restrict__ q_on, const float* __restrict__ q_tgt,
                                const int64_t* __restrict__ actions, const int64_t* __restrict__ a_star,
                                const float* __restrict__ returns, const float* __restrict__ nonterminals, float gamma_n,
                                const MmdBandwidths bw, float* __restrict__ loss, float* __restrict__ dtheta,
                                float* __restrict__ theta_out, float* __restrict__ target_out, float eps) {
  extern __shared__ float sm[];  // n particles | n targets | 32 reduction slots
  float* sth = sm;
  float* sT = sm + n;
  float* red = sT + n;
  const int b = blockIdx.x, tid = threadIdx.x;
  const int as = (int)a_star[b], ac = (int)actions[b];
  const float g = __fmul_rn(gamma_n, nonterminals[b]);
  for (int j = tid; j < n; j += blockDim.x) {
    float t;
    if constexpr (RESCALE) {
      const double z = vr_h_inv((double)q_tgt[((long)j * B + b) * A + as], (double)eps);
      t = __double2float_rn(vr_h(__dadd_rn((double)returns[b], __dmul_rn((double)g, z)), (double)eps));
    } else {
      t = __fadd_rn(returns[b], __fmul_rn(g, q_tgt[((long)j * B + b) * A + as]));
    }
    sT[j] = t;
    if (target_out) target_out[(long)b * n + j] = t;
    const float th = q_on[((long)j * B + b) * A + ac];
    sth[j] = th;
    if (theta_out) theta_out[(long)b * n + j] = th;
  }
  __syncthreads();
  const float nn = (float)(n * n);
  float part = 0.f;
  if (tid < n) {
    const float th = sth[tid], ti = sT[tid];
    float acc = 0.f, gacc = 0.f;
    for (int j = 0; j < n; ++j) {
      const float thj = sth[j], tj = sT[j];
      const float d1 = __fsub_rn(th, thj), d2 = __fsub_rn(ti, tj), d3 = __fsub_rn(th, tj);
      const float s1 = __fmul_rn(d1, d1), s2 = __fmul_rn(d2, d2), s3 = __fmul_rn(d3, d3);
      float k1 = 0.f, k2 = 0.f, k3 = 0.f, g1 = 0.f, g3 = 0.f;
      for (int h = 0; h < bw.H; ++h) {
        const float c = bw.c[h], w = bw.w[h];
        const float e1 = exp2f(__fmul_rn(s1, c)), e2 = exp2f(__fmul_rn(s2, c)), e3 = exp2f(__fmul_rn(s3, c));
        k1 = __fadd_rn(k1, e1);
        k2 = __fadd_rn(k2, e2);
        k3 = __fadd_rn(k3, e3);
        g1 = __fadd_rn(g1, __fmul_rn(w, e1));
        g3 = __fadd_rn(g3, __fmul_rn(w, e3));
      }
      acc = __fadd_rn(acc, __fsub_rn(__fadd_rn(k1, k2), __fmul_rn(2.f, k3)));
      gacc = __fadd_rn(gacc, __fsub_rn(__fmul_rn(d3, g3), __fmul_rn(d1, g1)));
    }
    part = acc;
    dtheta[(long)tid * B + b] = __fdiv_rn(__fmul_rn(2.f, gacc), nn);
  }
  part = warp_sum(part);
  if ((tid & 31) == 0) red[tid >> 5] = part;
  __syncthreads();
  if (tid < 32) {
    float v = tid < (blockDim.x >> 5) ? red[tid] : 0.f;
    v = warp_sum(v);
    if (tid == 0) {
      const float l = __fdiv_rn(v, nn);
      loss[b] = l < 0.f ? 0.f : l;          // a NaN stays visible
    }
  }
}

// The bandwidths as the kernel takes them; false (nothing to launch) unless 1 <= H <= 16 and every h is finite and > 0
// with finite constants c_h and w_h.
static bool mmd_bandwidths(int H, const float* h, MmdBandwidths* out) {
  if (H < 1 || H > MMD_MAX_H || h == nullptr) return false;
  out->H = H;
  for (int k = 0; k < MMD_MAX_H; ++k) out->c[k] = out->w[k] = 0.f;
  for (int k = 0; k < H; ++k) {
    if (!(h[k] > 0.f) || !std::isfinite(h[k])) return false;
    out->c[k] = (float)(-1.4426950408889634 / (double)h[k]);
    out->w[k] = (float)(2.0 / (double)h[k]);
    if (!std::isfinite(out->c[k]) || !std::isfinite(out->w[k])) return false;
  }
  return true;
}

template <bool RESCALE>
static int mmd_launch(int batch, int n, int action_space, const float* q_online, const float* q_target,
                      const long long* actions, const long long* a_star, const float* returns,
                      const float* nonterminals, float gamma_n, int n_bandwidths, const float* bandwidths, float eps,
                      float* loss, float* dtheta, float* theta_out, float* target_out, void* stream) {
  MmdBandwidths bw;
  if (batch < 1 || n < 1 || n > MMD_MAX_N || action_space < 1 || action_space > 32 ||
      !mmd_bandwidths(n_bandwidths, bandwidths, &bw) || (RESCALE && !vr_eps_ok(eps)))
    return (int)cudaErrorInvalidValue;
  riqn::note_launches(1);
  const int threads = (n + 31) / 32 * 32;
  const size_t smem = sizeof(float) * (2 * (size_t)n + 32);
  mmd_loss_kernel<RESCALE><<<batch, threads, smem, (cudaStream_t)stream>>>(
      batch, n, action_space, q_online, q_target, (const int64_t*)actions, (const int64_t*)a_star, returns,
      nonterminals, gamma_n, bw, loss, dtheta, theta_out, target_out, eps);
  return (int)cudaGetLastError();
}

}  // namespace riqn

using namespace riqn;

RIQN_API int riqn_mmd_loss_fwd_bwd(int batch, int n, int action_space, const float* q_online, const float* q_target,
                                   const long long* actions, const long long* a_star, const float* returns,
                                   const float* nonterminals, float gamma_n, int n_bandwidths, const float* bandwidths,
                                   float* loss, float* dtheta, float* theta_out, float* target_out, void* stream) {
  return mmd_launch<false>(batch, n, action_space, q_online, q_target, actions, a_star, returns, nonterminals, gamma_n,
                           n_bandwidths, bandwidths, 0.f, loss, dtheta, theta_out, target_out, stream);
}

RIQN_API int riqn_mmd_loss_fwd_bwd_h(int batch, int n, int action_space, const float* q_online, const float* q_target,
                                     const long long* actions, const long long* a_star, const float* returns,
                                     const float* nonterminals, float gamma_n, int n_bandwidths,
                                     const float* bandwidths, float eps, float* loss, float* dtheta, float* theta_out,
                                     float* target_out, void* stream) {
  return mmd_launch<true>(batch, n, action_space, q_online, q_target, actions, a_star, returns, nonterminals, gamma_n,
                          n_bandwidths, bandwidths, eps, loss, dtheta, theta_out, target_out, stream);
}
