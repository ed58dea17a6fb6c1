// Rainbow-only (C51) head and loss: reference rainbowiqn/model.py:120-129 and rainbowiqn/agent.py:77-141.
// The heavy part (conv trunk + hidden NoisyLinear layers) is shared with the IQN path; here are the categorical
// pieces: dueling over atoms + (log-)softmax, expected-value argmax, the Bellman projection with its l == u fix,
// the cross-entropy and its gradient, plus small strided linear-layer helpers for the (B, 512) x (51 | 918) z-layers.
#include "common.cuh"
#include "gemm.h"
#include "../../include/riqn_b200.h"

namespace riqn {
int colsum_add(long M, int N, const float* X, float* out, cudaStream_t s);

// One block per sample.  q[a,j] = v[j] + a[a,j] - mean_a a[.,j]; p = softmax_j q, logp = log_softmax_j q.
// Optionally the double-DQN action argmax_a sum_j support[j] p[a,j]  (agent.py:92-99).
__global__ void c51_head_fwd_kernel(int A, int atoms, const float* __restrict__ zv, const float* __restrict__ za,
                                    const float* __restrict__ support, float* __restrict__ p, float* __restrict__ logp,
                                    int64_t* __restrict__ a_star) {
  extern __shared__ float sm[];      // amean[atoms] | ev[A]
  float* amean = sm;
  float* ev = sm + atoms;
  const int b = blockIdx.x;
  const float* zab = za + (long)b * A * atoms;
  for (int j = threadIdx.x; j < atoms; j += blockDim.x) {
    float s = 0.f;
    for (int a = 0; a < A; ++a) s += zab[a * atoms + j];
    amean[j] = s / (float)A;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int a = warp; a < A; a += nw) {
    float q0 = -INFINITY, q1 = -INFINITY;          // atoms <= 64: lane owns j = lane and lane + 32
    if (lane < atoms) q0 = zv[(long)b * atoms + lane] + zab[a * atoms + lane] - amean[lane];
    if (lane + 32 < atoms) q1 = zv[(long)b * atoms + lane + 32] + zab[a * atoms + lane + 32] - amean[lane + 32];
    float mx = fmaxf(q0, q1);
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    const float e0 = lane < atoms ? expf(q0 - mx) : 0.f, e1 = lane + 32 < atoms ? expf(q1 - mx) : 0.f;
    const float sum = warp_sum(e0 + e1);
    const float lse = logf(sum);
    const long o = ((long)b * A + a) * atoms;
    float evp = 0.f;
    if (lane < atoms) {
      if (p) p[o + lane] = e0 / sum;
      if (logp) logp[o + lane] = q0 - mx - lse;
      evp += support[lane] * (e0 / sum);
    }
    if (lane + 32 < atoms) {
      if (p) p[o + lane + 32] = e1 / sum;
      if (logp) logp[o + lane + 32] = q1 - mx - lse;
      evp += support[lane + 32] * (e1 / sum);
    }
    evp = warp_sum(evp);
    if (lane == 0) ev[a] = evp;
  }
  __syncthreads();
  if (a_star && threadIdx.x == 0) {
    int arg = 0;
    float best = ev[0];
    for (int a = 1; a < A; ++a)
      if (ev[a] > best) { best = ev[a]; arg = a; }
    a_star[b] = arg;
  }
}

// One block per sample: categorical projection (agent.py:104-133), loss = -sum_j m_j logp[b, act, j] (agent.py:141)
// and dq[b, j] = d loss / d q[b, act, j] = -(m_j - p_j sum_k m_k).
__global__ void c51_loss_kernel(int A, int atoms, const float* __restrict__ logp_online, const float* __restrict__ p_target,
                                const int64_t* __restrict__ actions, const int64_t* __restrict__ a_star,
                                const float* __restrict__ returns, const float* __restrict__ nonterminals,
                                const float* __restrict__ support, float gamma_n, float vmin, float vmax, float delta_z,
                                float* __restrict__ loss, float* __restrict__ dq, float* __restrict__ m_out) {
  extern __shared__ float sm[];      // m[atoms] | lo[atoms] | up[atoms] | wl[atoms] | wu[atoms]
  float* m = sm;
  int* lo = reinterpret_cast<int*>(sm + atoms);
  int* up = lo + atoms;
  float* wl = reinterpret_cast<float*>(up + atoms);
  float* wu = wl + atoms;
  const int b = blockIdx.x;
  const int act = (int)actions[b], as = (int)a_star[b];
  const float* pa = p_target + ((long)b * A + as) * atoms;
  const float g = __fmul_rn(nonterminals[b], gamma_n);
  for (int j = threadIdx.x; j < atoms; j += blockDim.x) {
    float tz = __fadd_rn(returns[b], __fmul_rn(g, support[j]));
    tz = fminf(fmaxf(tz, vmin), vmax);
    // The clamp of tz does not bound the index: fp32 rounding of the division can take bj just above atoms - 1
    // (v_min = -1, v_max = 1, 62 atoms: tz = v_max gives 61.0000038), and u = atoms would add wu past m.  Every
    // bj <= atoms - 1 is unchanged.  (The reference's index_add_ lands on the next sample's atom 0 instead.)
    const float bj = fminf(__fdiv_rn(__fsub_rn(tz, vmin), delta_z), (float)(atoms - 1));
    int l = (int)floorf(bj), u = (int)ceilf(bj);
    if (u > 0 && l == u) l -= 1;                   // agent.py:119
    if (l < atoms - 1 && l == u) u += 1;           // agent.py:120
    lo[j] = l; up[j] = u;
    wl[j] = __fmul_rn(pa[j], __fsub_rn((float)u, bj));
    wu[j] = __fmul_rn(pa[j], __fsub_rn(bj, (float)l));
    m[j] = 0.f;
  }
  __syncthreads();
  if (threadIdx.x == 0) {                          // index_add_ order of the reference: all l-adds, then all u-adds
    for (int j = 0; j < atoms; ++j) m[lo[j]] += wl[j];
    for (int j = 0; j < atoms; ++j) m[up[j]] += wu[j];
  }
  __syncthreads();
  const float* lp = logp_online + ((long)b * A + act) * atoms;
  float part = 0.f, msum = 0.f;
  for (int j = threadIdx.x; j < atoms; j += blockDim.x) { part += m[j] * lp[j]; msum += m[j]; }
  part = warp_sum(part);
  msum = warp_sum(msum);
  __shared__ float red[2][32];
  if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = part; red[1][threadIdx.x >> 5] = msum; }
  __syncthreads();
  float tot = 0.f, mt = 0.f;
  for (int w = 0; w < (blockDim.x >> 5); ++w) { tot += red[0][w]; mt += red[1][w]; }
  if (threadIdx.x == 0) loss[b] = -tot;
  for (int j = threadIdx.x; j < atoms; j += blockDim.x) {
    dq[(long)b * atoms + j] = -(m[j] - expf(lp[j]) * mt);
    if (m_out) m_out[(long)b * atoms + j] = m[j];
  }
}

// dzv[b,j] = g*dq[b,j] ; dza[b,a,j] = g*dq[b,j]*(1{a==act} - 1/A)
__global__ void c51_head_bwd_kernel(int B, int A, int atoms, const float* __restrict__ dq, const float* __restrict__ gscale, float gmul,
                                    const int64_t* __restrict__ actions, float* __restrict__ dzv, float* __restrict__ dza) {
  const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long)B * A * atoms) return;
  const int j = (int)(idx % atoms), a = (int)((idx / atoms) % A);
  const long b = idx / ((long)atoms * A);
  const float g = dq[b * atoms + j] * (gscale[b] * gmul);
  dza[idx] = g * ((a == (int)actions[b] ? 1.f : 0.f) - 1.f / (float)A);
  if (a == 0) dzv[b * atoms + j] = g;
}

// Dense upstream gradient G (B, A, atoms) of the head's output, one block per sample, one warp per action (atoms <= 64:
// lane owns j = lane and lane + 32).  out holds p (is_log == 0) or log p (is_log != 0):
//   log-softmax: dq = G - p * sum_j G ;  softmax: dq = p * (G - sum_j p G)
// then the dueling split over actions, per atom: dzv[j] = sum_a dq[a,j] (a ascending), dza[a,j] = dq[a,j] - dzv[j] / A.
__global__ void c51_head_bwd_dense_kernel(int A, int atoms, const float* __restrict__ out, const float* __restrict__ G,
                                          int is_log, float* __restrict__ dzv, float* __restrict__ dza) {
  extern __shared__ float sdq[];     // dq[A * atoms] | dv[atoms]
  float* dv = sdq + A * atoms;
  const int b = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int a = warp; a < A; a += nw) {
    const long o = ((long)b * A + a) * atoms;
    float p[2] = {0.f, 0.f}, g[2] = {0.f, 0.f};
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int j = lane + 32 * u;
      if (j < atoms) {
        p[u] = is_log ? expf(out[o + j]) : out[o + j];
        g[u] = G[o + j];
      }
    }
    const float s = is_log ? warp_sum(g[0] + g[1]) : warp_sum(p[0] * g[0] + p[1] * g[1]);
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int j = lane + 32 * u;
      if (j < atoms) sdq[a * atoms + j] = is_log ? g[u] - p[u] * s : p[u] * (g[u] - s);
    }
  }
  __syncthreads();
  for (int j = threadIdx.x; j < atoms; j += blockDim.x) {
    float t = 0.f;
    for (int a = 0; a < A; ++a) t += sdq[a * atoms + j];
    dv[j] = t;
    dzv[(long)b * atoms + j] = t;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < A * atoms; i += blockDim.x)
    dza[(long)b * A * atoms + i] = sdq[i] - dv[i % atoms] / (float)A;
}

// grad_mu += s ; grad_sigma += s * eps with s = the split-K partials of dy^T x added in split order
__global__ void noisy_wgrad_finish_kernel(int splits, long n, const float* __restrict__ part, const float* __restrict__ eps,
                                          float* __restrict__ grad_mu, float* __restrict__ grad_sigma) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float acc = part[i];
  for (int k = 1; k < splits; ++k) acc += part[(long)k * n + i];
  grad_mu[i] += acc;
  grad_sigma[i] += __fmul_rn(acc, eps[i]);
}

__global__ void relu_mask_kernel(long n, const float* __restrict__ act, float* __restrict__ grad) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && !(act[i] > 0.f)) grad[i] = 0.f;
}

}  // namespace riqn

using namespace riqn;

RIQN_API int riqn_c51_head_fwd(int batch, int action_space, int atoms, const float* zv, const float* za,
                               const float* support, float* p, float* logp, long long* a_star, void* stream) {
  riqn::note_launches(1);
  if (atoms > 64) return (int)cudaErrorInvalidValue;
  c51_head_fwd_kernel<<<batch, 256, sizeof(float) * (atoms + action_space), (cudaStream_t)stream>>>(
      action_space, atoms, zv, za, support, p, logp, (int64_t*)a_star);
  return (int)cudaGetLastError();
}

RIQN_API int riqn_c51_loss_fwd_bwd(int batch, int action_space, int atoms, const float* logp_online, const float* p_target,
                                   const long long* actions, const long long* a_star, const float* returns,
                                   const float* nonterminals, const float* support, float gamma_n, float v_min, float v_max,
                                   float delta_z, float* loss, float* dq, float* m_out, void* stream) {
  riqn::note_launches(1);
  c51_loss_kernel<<<batch, 64, sizeof(float) * 5 * atoms, (cudaStream_t)stream>>>(
      action_space, atoms, logp_online, p_target, (const int64_t*)actions, (const int64_t*)a_star, returns, nonterminals,
      support, gamma_n, v_min, v_max, delta_z, loss, dq, m_out);
  return (int)cudaGetLastError();
}

RIQN_API int riqn_c51_head_bwd(int batch, int action_space, int atoms, const float* dq, const float* gscale, float gscale_mul,
                               const long long* actions, float* dzv, float* dza, void* stream) {
  riqn::note_launches(1);
  const long n = (long)batch * action_space * atoms;
  c51_head_bwd_kernel<<<riqn_cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(batch, action_space, atoms, dq, gscale, gscale_mul,
                                                                          (const int64_t*)actions, dzv, dza);
  return (int)cudaGetLastError();
}

RIQN_API int riqn_c51_head_bwd_dense(int batch, int action_space, int atoms, const float* out, const float* grad_out,
                                     int is_log, float* dzv, float* dza, void* stream) {
  riqn::note_launches(1);
  if (atoms > 64) return (int)cudaErrorInvalidValue;
  const size_t smem = sizeof(float) * ((size_t)action_space * atoms + atoms);
  if (smem > 48 * 1024) return (int)cudaErrorInvalidValue;
  c51_head_bwd_dense_kernel<<<batch, 256, smem, (cudaStream_t)stream>>>(action_space, atoms, out, grad_out, is_log, dzv, dza);
  return (int)cudaGetLastError();
}

RIQN_API int riqn_relu_mask(long n, const float* act, float* grad, void* stream) {
  riqn::note_launches(1);
  relu_mask_kernel<<<riqn_cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(n, act, grad);
  return (int)cudaGetLastError();
}

// y (rows, out) [ldy] = x (rows, in) [ldx] w^T + bias, optional ReLU
RIQN_API int riqn_linear_fwd_ld(long rows, int in_features, int out_features, const float* x, long ldx, const float* w,
                                const float* bias, float* y, long ldy, int relu, void* stream) {
  riqn::note_launches(1);
  EpiArgs e;
  e.bias = bias;
  return gemm_f32((int)rows, out_features, in_features, x, ldx, 1, w, in_features, 1, y, ldy, relu ? EPI_BIAS_RELU : EPI_BIAS,
                  e, 1, (cudaStream_t)stream);
}

// dx (rows, in) [lddx] = dy (rows, out) [lddy] w
RIQN_API int riqn_linear_dgrad_ld(long rows, int in_features, int out_features, const float* dy, long lddy, const float* w,
                                  float* dx, long lddx, void* stream) {
  riqn::note_launches(1);
  EpiArgs e;
  return gemm_f32((int)rows, in_features, out_features, dy, lddy, 1, w, 1, in_features, dx, lddx, EPI_STORE, e, 1,
                  (cudaStream_t)stream);
}

// grad_mu (out, in) += dy^T x ; grad_sigma += (dy^T x) * eps_w.  Split-K over the rows (at least 64 per split) to fill
// the SMs; every split stores its partial product in its own scratch slab and noisy_wgrad_finish_kernel adds the slabs
// in split order, so the result does not depend on which split finishes first.  One split accumulates in the epilogue.
RIQN_API int riqn_noisy_wgrad_ld(long rows, int in_features, int out_features, const float* dy, long lddy, const float* x,
                                 long ldx, const float* weight_epsilon, float* grad_mu, float* grad_sigma, void* stream) {
  cudaStream_t s = (cudaStream_t)stream;
  EpiArgs e;
  const int tiles = ((out_features + 127) / 128) * ((in_features + 127) / 128);
  int split = (riqn_sms() + tiles - 1) / tiles;
  if ((long)split * 64 > rows) split = (int)((rows + 63) / 64);
  const int splits = gemm_f32_splits((int)rows, split);
  if (splits <= 1) {
    riqn::note_launches(1);
    e.out2 = grad_sigma;
    e.eps = weight_epsilon;
    return gemm_f32(out_features, in_features, (int)rows, dy, 1, lddy, x, 1, ldx, grad_mu, in_features, EPI_NOISY_WGRAD, e,
                    1, s);
  }
  riqn::note_launches(2);
  const long n = (long)out_features * in_features;
  StreamScratch part;
  RIQN_CUDA(part.alloc((size_t)splits * n, s));
  e.slab = n;
  int rc = gemm_f32(out_features, in_features, (int)rows, dy, 1, lddy, x, 1, ldx, part.p, in_features, EPI_SLAB, e, split, s);
  if (rc) return rc;
  noisy_wgrad_finish_kernel<<<riqn_cdiv(n, 256), 256, 0, s>>>(splits, n, part.p, weight_epsilon, grad_mu, grad_sigma);
  return (int)cudaGetLastError();
}
