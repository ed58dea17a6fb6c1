// HL-Gauss loss (Farebrother et al., "Stop Regressing: Training Value Functions via Classification for Scalable Deep RL",
// ICML 2024; the histogram loss of Imani & White, ICML 2018; no counterpart in the reference) on the C51 head: the
// cross-entropy of the online categorical output against the mass that a Gaussian N(y, sigma^2) centred on the scalar
// double-DQN target y puts in each bin of the support.
//   g    = fl32(nt[b] * gamma_n)
//   Q'   = sum_j p_tgt[b, a*, j] * s_j        s_j = support[j], RESCALE: h^-1(support[j])        (double, j ascending)
//   y    = clamp(R[b] + g * Q', v_min, v_max)                    RESCALE: clamp(h(R[b] + g * Q'), v_min, v_max)
//   e_i  = v_min + (i - 1/2) * D,  D = (v_max - v_min) / (atoms - 1),  i = 0..atoms     (atom j centres [e_j, e_j+1])
//   u_i  = (e_i - y) / s,  s = (r * D) * sqrt(2) ;  c_i = erfc(|u_i|) / 2   (the Gaussian's tail beyond e_i, away from y)
//   mass_j = c_j - c_j+1 (u_j >= 0) | c_j+1 - c_j (u_j+1 <= 0) | (1/2 - c_j) + (1/2 - c_j+1) (the bin holding y)
//   m_j  = fl32(mass_j / Z),  Z = (1/2 - c_0) + (1/2 - c_atoms)
//   loss[b] = -sum_j m_j logp[b, act, j] ,  dq[b, j] = -(m_j - p_j * sum_k m_k),  p_j = fl32(exp(logp[b, act, j]))
// Every double operation is an explicitly rounded intrinsic (nvcc contracts nothing), so target_out = fl32(y) is the value
// numpy float64 computes with the same operations in the same order; only erfc is not a basic operation (CUDA's double
// erfc and libm's are a few double ulps apart).  Each mass is a difference of one-sided tails, never of two numbers
// near 1, and the clamp keeps y inside [e_0, e_atoms], so Z > 0.  1 - c_j - c_j+1 is formed as
// (1/2 - c_j) + (1/2 - c_j+1): each difference is exact where c >= 1/4, so at a wide sigma (c -> 1/2, small bin masses
// and Z) no digit is lost to a rounded 1 - c, and sum_j m_j = 1 to a few double ulps up to sigma = 1000 bin widths.
//
// The cross-entropy tail is c51_loss_kernel's (one thread per atom, the two-warp reduction, loss = -tot) written out with
// explicitly rounded fp32 operations and a correctly rounded p_j, not shared with it: that kernel lets nvcc contract
// m - p * mt into an FMA and takes expf's 2-ulp exponential, which would leave dq without a numpy statement, and
// rewriting it would change the pinned SASS of its existing instantiations.  dq stays the gradient riqn_c51_head_bwd takes.
//
// One CTA of 64 threads per transition (atoms <= 64: one thread per atom and per edge, thread 0 also takes edge 64),
// no atomics, so a step is bitwise reproducible.
#include "common.cuh"
#include "value_rescaling.cuh"
#include "../../include/riqn_b200.h"

#include <cmath>

namespace riqn {
constexpr int HLG_THREADS = 64;
constexpr double HLG_SQRT2 = 1.4142135623730951;   // fl64(sqrt(2))

template <bool RESCALE>
__global__ void __launch_bounds__(HLG_THREADS)
hl_gauss_loss_kernel(int A, int atoms, const float* __restrict__ logp_online, const float* __restrict__ p_target,
                     const int64_t* __restrict__ actions, const int64_t* __restrict__ a_star,
                     const float* __restrict__ returns, const float* __restrict__ nonterminals,
                     const float* __restrict__ support, float gamma_n, float vmin, float vmax, float sigma_ratio,
                     float eps, float* __restrict__ loss, float* __restrict__ dq, float* __restrict__ m_out,
                     float* __restrict__ target_out) {
  __shared__ double sc[HLG_THREADS + 1];     // c_i
  __shared__ double su[HLG_THREADS + 1];     // u_i
  __shared__ double sprod[HLG_THREADS];      // p_tgt[b, a*, j] * s_j
  __shared__ double sy;
  __shared__ float red[2][2];
  const int b = blockIdx.x, tid = threadIdx.x;
  const double lo = (double)vmin, hi = (double)vmax;
  if (tid < atoms) {
    const float* pa = p_target + ((long)b * A + (int)a_star[b]) * atoms;
    const double s = RESCALE ? vr_h_inv((double)support[tid], (double)eps) : (double)support[tid];
    sprod[tid] = __dmul_rn((double)pa[tid], s);
  }
  __syncthreads();
  if (tid == 0) {
    const float g = __fmul_rn(nonterminals[b], gamma_n);
    double q = 0.0;
    for (int j = 0; j < atoms; ++j) q = __dadd_rn(q, sprod[j]);
    double y = __dadd_rn((double)returns[b], __dmul_rn((double)g, q));
    if constexpr (RESCALE) y = vr_h(y, (double)eps);
    y = y < lo ? lo : (y > hi ? hi : y);        // a NaN stays visible
    sy = y;
    if (target_out) target_out[b] = __double2float_rn(y);
  }
  __syncthreads();
  const double y = sy;
  const double D = __ddiv_rn(__dsub_rn(hi, lo), (double)(atoms - 1));
  const double s = __dmul_rn(__dmul_rn((double)sigma_ratio, D), HLG_SQRT2);
  for (int i = tid; i <= atoms; i += HLG_THREADS) {
    const double e = __dadd_rn(lo, __dmul_rn(__dsub_rn((double)i, 0.5), D));
    const double u = __ddiv_rn(__dsub_rn(e, y), s);
    su[i] = u;
    sc[i] = __dmul_rn(0.5, erfc(fabs(u)));
  }
  __syncthreads();
  float m = 0.f, part = 0.f;
  const float* lp = logp_online + ((long)b * A + (int)actions[b]) * atoms;
  if (tid < atoms) {
    const double cj = sc[tid], ck = sc[tid + 1];
    double mass;
    if (su[tid] >= 0.0) mass = __dsub_rn(cj, ck);             // the bin lies wholly above y
    else if (su[tid + 1] <= 0.0) mass = __dsub_rn(ck, cj);    // wholly below y
    else mass = __dadd_rn(__dsub_rn(0.5, cj), __dsub_rn(0.5, ck));   // the bin that holds y
    const double Z = __dadd_rn(__dsub_rn(0.5, sc[0]), __dsub_rn(0.5, sc[atoms]));
    m = __double2float_rn(__ddiv_rn(mass, Z));
    part = __fmul_rn(m, lp[tid]);
  }
  part = warp_sum(part);
  const float msum = warp_sum(m);
  if ((tid & 31) == 0) { red[0][tid >> 5] = part; red[1][tid >> 5] = msum; }
  __syncthreads();
  const float tot = __fadd_rn(__fadd_rn(0.f, red[0][0]), red[0][1]);
  const float mt = __fadd_rn(__fadd_rn(0.f, red[1][0]), red[1][1]);
  if (tid == 0) loss[b] = -tot;
  if (tid < atoms) {
    const float p = __double2float_rn(exp((double)lp[tid]));
    dq[(long)b * atoms + tid] = -__fsub_rn(m, __fmul_rn(p, mt));
    if (m_out) m_out[(long)b * atoms + tid] = m;
  }
}

template <bool RESCALE>
static int hl_gauss_launch(int batch, int action_space, int atoms, const float* logp_online, const float* p_target,
                           const long long* actions, const long long* a_star, const float* returns,
                           const float* nonterminals, const float* support, float gamma_n, float v_min, float v_max,
                           float sigma_ratio, float eps, float* loss, float* dq, float* m_out, float* target_out,
                           void* stream) {
  if (batch < 1 || action_space < 1 || atoms < 2 || atoms > HLG_THREADS || !std::isfinite(v_min) ||
      !std::isfinite(v_max) || !(v_min < v_max) || !std::isfinite(sigma_ratio) || !(sigma_ratio > 0.f) ||
      sigma_ratio > 1000.f || (RESCALE && !vr_eps_ok(eps)))
    return (int)cudaErrorInvalidValue;
  riqn::note_launches(1);
  hl_gauss_loss_kernel<RESCALE><<<batch, HLG_THREADS, 0, (cudaStream_t)stream>>>(
      action_space, atoms, logp_online, p_target, (const int64_t*)actions, (const int64_t*)a_star, returns,
      nonterminals, support, gamma_n, v_min, v_max, sigma_ratio, eps, loss, dq, m_out, target_out);
  return (int)cudaGetLastError();
}

}  // namespace riqn

using namespace riqn;

RIQN_API int riqn_hl_gauss_loss_fwd_bwd(int batch, int action_space, int atoms, const float* logp_online,
                                        const float* p_target, const long long* actions, const long long* a_star,
                                        const float* returns, const float* nonterminals, const float* support,
                                        float gamma_n, float v_min, float v_max, float sigma_ratio, float* loss,
                                        float* dq, float* m_out, float* target_out, void* stream) {
  return hl_gauss_launch<false>(batch, action_space, atoms, logp_online, p_target, actions, a_star, returns,
                                nonterminals, support, gamma_n, v_min, v_max, sigma_ratio, 0.f, loss, dq, m_out,
                                target_out, stream);
}

RIQN_API int riqn_hl_gauss_loss_fwd_bwd_h(int batch, int action_space, int atoms, const float* logp_online,
                                          const float* p_target, const long long* actions, const long long* a_star,
                                          const float* returns, const float* nonterminals, const float* support,
                                          float gamma_n, float v_min, float v_max, float sigma_ratio, float eps,
                                          float* loss, float* dq, float* m_out, float* target_out, void* stream) {
  return hl_gauss_launch<true>(batch, action_space, atoms, logp_online, p_target, actions, a_star, returns,
                               nonterminals, support, gamma_n, v_min, v_max, sigma_ratio, eps, loss, dq, m_out,
                               target_out, stream);
}
