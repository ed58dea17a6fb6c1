// QR-DQN head (Dabney, Rowland, Bellemare & Munos, AAAI 2018; no counterpart in the reference): the dueling sum taken per
// quantile on the C51-shaped z-layers, zv (B, n) and za (B, A*n), written quantile-major as the IQN head's q (n*B, A), and
// its two backwards.  The z-layers are sample-major and q is quantile-major, so every kernel moves a tile of QR_TB samples x
// QR_TI quantiles through shared memory: reads along the quantile index of a z-layer row, writes along the rows of q (and
// the reverse for the backwards).  Every element is computed by one thread in a fixed order: no atomics.
#include "common.cuh"
#include "../../include/riqn_b200.h"

namespace riqn {
constexpr int QR_TB = 8;         // samples per tile
constexpr int QR_TI = 32;        // quantiles per tile
constexpr int QR_THREADS = 256;

// q[(i*B + b)*A + a] = fl(fl(zv[b,i] + za[b, a*n+i]) - fl(s_i / A)),  s_i = sum_a za[b, a*n+i] (a ascending, fp32)
__global__ void qr_head_fwd_kernel(int B, int A, int n, const float* __restrict__ zv, const float* __restrict__ za,
                                   float* __restrict__ q) {
  extern __shared__ float sm[];    // za tile [TB][A][TI] | zv [TB][TI] | mean [TB][TI]
  float* sza = sm;
  float* szv = sza + QR_TB * A * QR_TI;
  float* smean = szv + QR_TB * QR_TI;
  const int i0 = blockIdx.x * QR_TI, b0 = blockIdx.y * QR_TB;
  const int ni = min(QR_TI, n - i0), nb = min(QR_TB, B - b0);
  for (int t = threadIdx.x; t < nb * A * QR_TI; t += blockDim.x) {       // coalesced along i within each (b, a) row
    const int il = t % QR_TI, a = (t / QR_TI) % A, bl = t / (QR_TI * A);
    if (il < ni) sza[t] = za[(long)(b0 + bl) * A * n + (long)a * n + i0 + il];
  }
  for (int t = threadIdx.x; t < nb * QR_TI; t += blockDim.x) {
    const int il = t % QR_TI, bl = t / QR_TI;
    if (il < ni) szv[t] = zv[(long)(b0 + bl) * n + i0 + il];
  }
  __syncthreads();
  for (int t = threadIdx.x; t < nb * QR_TI; t += blockDim.x) {
    const int il = t % QR_TI, bl = t / QR_TI;
    if (il < ni) {
      float s = 0.f;
      for (int a = 0; a < A; ++a) s = __fadd_rn(s, sza[(bl * A + a) * QR_TI + il]);
      smean[t] = __fdiv_rn(s, (float)A);
    }
  }
  __syncthreads();
  // quantile i's rows b0..b0+nb-1 are nb*A consecutive floats of q
  for (int il = 0; il < ni; ++il) {
    float* qi = q + ((long)(i0 + il) * B + b0) * A;
    for (int t = threadIdx.x; t < nb * A; t += blockDim.x) {
      const int a = t % A, bl = t / A;
      qi[t] = __fsub_rn(__fadd_rn(szv[bl * QR_TI + il], sza[(bl * A + a) * QR_TI + il]), smean[bl * QR_TI + il]);
    }
  }
}

// DENSE == false: the one-hot gradient of the loss kernel, dL/dq[i*B+b, a] = 1{a == actions[b]} * dtheta[i*B+b] * gscale[b]
// * gscale_mul, rounded exactly as riqn_c51_head_bwd rounds it on dq[b, i] = dtheta[i*B+b]:
//   g = fl(dtheta * fl(gscale * gscale_mul)) ;  dzv[b,i] = g ;  dza[b, a*n+i] = fl(g * fl(1{a == act} - fl(1 / A)))
// DENSE == true: a dense G = dL/dq (n*B, A):  dzv[b,i] = sum_a G[i*B+b, a] (a ascending) ;  dza = fl(G - fl(dzv / A))
template <bool DENSE>
__global__ void qr_head_bwd_kernel(int B, int A, int n, const float* __restrict__ dtheta, const float* __restrict__ gscale,
                                   float gmul, const int64_t* __restrict__ actions, const float* __restrict__ G,
                                   float* __restrict__ dzv, float* __restrict__ dza) {
  extern __shared__ float sm[];    // DENSE: G tile [TB][A][TI] ; one-hot: g tile [TB][TI] | sum / g [TB][TI]
  float* sg = sm;
  float* sv = sg + (DENSE ? QR_TB * A * QR_TI : 0);
  const int i0 = blockIdx.x * QR_TI, b0 = blockIdx.y * QR_TB;
  const int ni = min(QR_TI, n - i0), nb = min(QR_TB, B - b0);
  if constexpr (DENSE) {
    for (int il = 0; il < ni; ++il) {            // quantile i's rows b0..b0+nb-1: nb*A consecutive floats of G
      const float* gi = G + ((long)(i0 + il) * B + b0) * A;
      for (int t = threadIdx.x; t < nb * A; t += blockDim.x) {
        const int a = t % A, bl = t / A;
        sg[(bl * A + a) * QR_TI + il] = gi[t];
      }
    }
    __syncthreads();
    for (int t = threadIdx.x; t < nb * QR_TI; t += blockDim.x) {
      const int il = t % QR_TI, bl = t / QR_TI;
      if (il < ni) {
        float s = 0.f;
        for (int a = 0; a < A; ++a) s = __fadd_rn(s, sg[(bl * A + a) * QR_TI + il]);
        sv[t] = s;
        dzv[(long)(b0 + bl) * n + i0 + il] = s;
      }
    }
  } else {
    for (int t = threadIdx.x; t < QR_TB * QR_TI; t += blockDim.x) {
      const int bl = t % QR_TB, il = t / QR_TB;   // reads along b within quantile i's rows
      if (bl < nb && il < ni) {
        const int b = b0 + bl;
        const float w = gscale ? __fmul_rn(gscale[b], gmul) : gmul;
        sv[bl * QR_TI + il] = __fmul_rn(dtheta[(long)(i0 + il) * B + b], w);
      }
    }
    __syncthreads();
    for (int t = threadIdx.x; t < nb * QR_TI; t += blockDim.x) {
      const int il = t % QR_TI, bl = t / QR_TI;
      if (il < ni) dzv[(long)(b0 + bl) * n + i0 + il] = sv[t];
    }
  }
  __syncthreads();
  const float rA = __fdiv_rn(1.f, (float)A);
  for (int t = threadIdx.x; t < nb * A * QR_TI; t += blockDim.x) {       // coalesced along i within each (b, a) row
    const int il = t % QR_TI, a = (t / QR_TI) % A, bl = t / (QR_TI * A);
    if (il >= ni) continue;
    float d;
    if constexpr (DENSE) {
      d = __fsub_rn(sg[t], __fdiv_rn(sv[bl * QR_TI + il], (float)A));
    } else {
      const float one = a == (int)actions[b0 + bl] ? 1.f : 0.f;
      d = __fmul_rn(sv[bl * QR_TI + il], __fsub_rn(one, rA));
    }
    dza[(long)(b0 + bl) * A * n + (long)a * n + i0 + il] = d;
  }
}

static bool qr_shape_ok(int batch, int action_space, int n) {
  return batch >= 1 && action_space >= 1 && action_space <= 32 && n >= 2 && n <= 256;
}

static dim3 qr_grid(int batch, int n) { return dim3(riqn_cdiv(n, QR_TI), riqn_cdiv(batch, QR_TB)); }

}  // namespace riqn

using namespace riqn;

RIQN_API int riqn_qr_head_fwd(int batch, int action_space, int n, const float* zv, const float* za, float* q, void* stream) {
  if (!qr_shape_ok(batch, action_space, n)) return (int)cudaErrorInvalidValue;
  riqn::note_launches(1);
  const size_t smem = sizeof(float) * QR_TI * QR_TB * ((size_t)action_space + 2);
  qr_head_fwd_kernel<<<qr_grid(batch, n), QR_THREADS, smem, (cudaStream_t)stream>>>(batch, action_space, n, zv, za, q);
  return (int)cudaGetLastError();
}

RIQN_API int riqn_qr_head_bwd(int batch, int action_space, int n, const float* dtheta, const float* gscale,
                              float gscale_mul, const long long* actions, float* dzv, float* dza, void* stream) {
  if (!qr_shape_ok(batch, action_space, n)) return (int)cudaErrorInvalidValue;
  riqn::note_launches(1);
  const size_t smem = sizeof(float) * QR_TI * QR_TB;
  qr_head_bwd_kernel<false><<<qr_grid(batch, n), QR_THREADS, smem, (cudaStream_t)stream>>>(
      batch, action_space, n, dtheta, gscale, gscale_mul, (const int64_t*)actions, nullptr, dzv, dza);
  return (int)cudaGetLastError();
}

RIQN_API int riqn_qr_head_bwd_dense(int batch, int action_space, int n, const float* grad_q, float* dzv, float* dza,
                                    void* stream) {
  if (!qr_shape_ok(batch, action_space, n)) return (int)cudaErrorInvalidValue;
  riqn::note_launches(1);
  const size_t smem = sizeof(float) * QR_TI * QR_TB * ((size_t)action_space + 1);
  qr_head_bwd_kernel<true><<<qr_grid(batch, n), QR_THREADS, smem, (cudaStream_t)stream>>>(
      batch, action_space, n, nullptr, nullptr, 1.f, nullptr, grad_q, dzv, dza);
  return (int)cudaGetLastError();
}
