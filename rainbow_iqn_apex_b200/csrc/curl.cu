// CURL (Srinivas, Laskin & Abbeel, ICML 2020): the bilinear InfoNCE between the anchor and key projections, the row
// LayerNorm (no affine) of the projection head, the momentum (EMA) update of the key encoder and the feature-gradient
// sum.  See include/riqn_b200.h for the statements.
//
// No atomics anywhere: every sum is a sequential fp32 chain in a stated order or the warp_sum butterfly, so the results
// are bitwise reproducible and independent of the stream and of other work on the device.
#include <math.h>

#include "common.cuh"
#include "../../include/riqn_b200.h"

namespace riqn {

int colsum_add(long M, int N, const float* X, float* out, cudaStream_t s);   // conv.cu

constexpr int CURL_D = 128;          // projection width the InfoNCE kernel is specialised for
constexpr int CURL_ROWS = 8;         // anchor rows per CTA (one warp each)
constexpr int CURL_THREADS = 32 * CURL_ROWS;
constexpr int CURL_CHUNK = 32;       // key rows staged in shared memory at a time
constexpr int CURL_LD = CURL_D + 1;  // padded row stride of the staged W and key rows (conflict-free column reads)
constexpr int CURL_MAX_BATCH = 4096;

static size_t curl_smem_bytes(int batch) {
  return sizeof(float) * ((size_t)CURL_D * CURL_LD + 2 * CURL_ROWS * CURL_D + CURL_CHUNK * CURL_LD +
                          (size_t)CURL_ROWS * batch);
}

// Stage key rows [j0, j0 + CURL_CHUNK) of z_k (rows past the batch read as 0).
__device__ __forceinline__ void curl_stage_keys(int B, int j0, const float* __restrict__ z_k, float* __restrict__ ks) {
  for (int e = threadIdx.x; e < CURL_CHUNK * CURL_D; e += CURL_THREADS) {
    const int jj = e / CURL_D, q = e % CURL_D;
    ks[jj * CURL_LD + q] = (j0 + jj < B) ? z_k[(long)(j0 + jj) * CURL_D + q] : 0.f;
  }
}

// One CTA per CURL_ROWS anchor rows i:
//   v_i = W^T z_a,i ; logits_ij = v_i . z_k,j ; m_i = max_j ; s_i = sum_j exp(l_ij - m_i) ; loss_i = m_i + log s_i - l_ii
//   dl_ij = scale * (exp(l_ij - m_i) / s_i - [i == j]) ; g_i = sum_j dl_ij z_k,j ; dz_a,i = W g_i ; g -> work (for dW)
__global__ void __launch_bounds__(CURL_THREADS, 1)
curl_infonce_rows_kernel(int B, const float* __restrict__ z_a, const float* __restrict__ z_k, const float* __restrict__ w,
                         float scale, float* __restrict__ loss_rows, float* __restrict__ dz_a, float* __restrict__ work,
                         float* __restrict__ logits_out) {
  extern __shared__ float smem[];
  float* ws = smem;                                   // W (D, D), row stride CURL_LD
  float* za = ws + CURL_D * CURL_LD;                  // anchor rows (ROWS, D), later g
  float* v = za + CURL_ROWS * CURL_D;                 // v (ROWS, D)
  float* ks = v + CURL_ROWS * CURL_D;                 // staged key rows (CHUNK, D), row stride CURL_LD
  float* L = ks + CURL_CHUNK * CURL_LD;               // logits, then dl (ROWS, B)
  const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
  const int i0 = blockIdx.x * CURL_ROWS;
  for (int e = t; e < CURL_D * CURL_D; e += CURL_THREADS) ws[(e / CURL_D) * CURL_LD + e % CURL_D] = w[e];
  for (int e = t; e < CURL_ROWS * CURL_D; e += CURL_THREADS) {
    const int r = e / CURL_D;
    za[e] = (i0 + r < B) ? z_a[(long)(i0 + r) * CURL_D + e % CURL_D] : 0.f;
  }
  __syncthreads();
  // v[r][q] = sum_p z_a[r][p] W[p][q], p ascending
  const int q = t & (CURL_D - 1), rb = t >> 7;        // each thread: column q of rows rb, rb + 2, rb + 4, rb + 6
  {
    float acc[CURL_ROWS / 2] = {};
    for (int p = 0; p < CURL_D; ++p) {
      const float wq = ws[p * CURL_LD + q];
#pragma unroll
      for (int k = 0; k < CURL_ROWS / 2; ++k) acc[k] = fmaf(za[(rb + 2 * k) * CURL_D + p], wq, acc[k]);
    }
#pragma unroll
    for (int k = 0; k < CURL_ROWS / 2; ++k) v[(rb + 2 * k) * CURL_D + q] = acc[k];
  }
  // logits: warp = row, lane = key row of the chunk; q ascending
  for (int j0 = 0; j0 < B; j0 += CURL_CHUNK) {
    __syncthreads();
    curl_stage_keys(B, j0, z_k, ks);
    __syncthreads();
    float acc = 0.f;
    const float* kr = ks + lane * CURL_LD;
    const float* vr = v + warp * CURL_D;
    for (int qq = 0; qq < CURL_D; ++qq) acc = fmaf(vr[qq], kr[qq], acc);
    if (j0 + lane < B) L[(long)warp * B + j0 + lane] = acc;
  }
  __syncthreads();
  // row softmax: max, sum of exp(l - max) (lane chains over j = lane + 32k ascending, then the butterfly), loss, dl
  const int i = i0 + warp;
  if (i < B) {
    float* Lr = L + (long)warp * B;
    float m = -INFINITY;
    for (int j = lane; j < B; j += 32) m = fmaxf(m, Lr[j]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float s = 0.f;
    for (int j = lane; j < B; j += 32) s += expf(Lr[j] - m);
    s = warp_sum(s);
    if (lane == 0) loss_rows[i] = (m + logf(s)) - Lr[i];
    if (logits_out != nullptr)
      for (int j = lane; j < B; j += 32) logits_out[(long)i * B + j] = Lr[j];
    __syncwarp();
    const float rs = __frcp_rn(s);
    for (int j = lane; j < B; j += 32) Lr[j] = scale * (__fmul_rn(expf(Lr[j] - m), rs) - (j == i ? 1.f : 0.f));
  } else {
    for (int j = lane; j < B; j += 32) L[(long)warp * B + j] = 0.f;
  }
  // g[r][q] = sum_j dl[r][j] z_k[j][q], j ascending
  float g[CURL_ROWS / 2] = {};
  for (int j0 = 0; j0 < B; j0 += CURL_CHUNK) {
    __syncthreads();
    curl_stage_keys(B, j0, z_k, ks);
    __syncthreads();
    const int n = min(CURL_CHUNK, B - j0);
    for (int jj = 0; jj < n; ++jj) {
      const float kq = ks[jj * CURL_LD + q];
#pragma unroll
      for (int k = 0; k < CURL_ROWS / 2; ++k) g[k] = fmaf(L[(long)(rb + 2 * k) * B + j0 + jj], kq, g[k]);
    }
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < CURL_ROWS / 2; ++k) {
    const int r = rb + 2 * k;
    za[r * CURL_D + q] = g[k];
    if (i0 + r < B) work[(long)(i0 + r) * CURL_D + q] = g[k];
  }
  __syncthreads();
  // dz_a[r][p] = sum_q W[p][q] g[r][q], q ascending (thread: p = t mod D)
  const int p = q;
  float acc[CURL_ROWS / 2] = {};
  for (int qq = 0; qq < CURL_D; ++qq) {
    const float wp = ws[p * CURL_LD + qq];
#pragma unroll
    for (int k = 0; k < CURL_ROWS / 2; ++k) acc[k] = fmaf(wp, za[(rb + 2 * k) * CURL_D + qq], acc[k]);
  }
#pragma unroll
  for (int k = 0; k < CURL_ROWS / 2; ++k)
    if (i0 + rb + 2 * k < B) dz_a[(long)(i0 + rb + 2 * k) * CURL_D + p] = acc[k];
}

// dW[p][q] += sum_i z_a[i][p] g[i][q]: one fmaf chain over i ascending per element, added once.
__global__ void __launch_bounds__(256)
curl_infonce_dw_kernel(int B, const float* __restrict__ z_a, const float* __restrict__ g, float* __restrict__ dw) {
  const int e = blockIdx.x * 256 + threadIdx.x;
  const int p = e / CURL_D, q = e % CURL_D;
  float acc = 0.f;
  for (int i = 0; i < B; ++i) acc = fmaf(__ldg(&z_a[(long)i * CURL_D + p]), __ldg(&g[(long)i * CURL_D + q]), acc);
  dw[e] += acc;
}

// Row LayerNorm without affine parameters, one warp per row, lane l holding elements l + 32k.  The row is fl(x + bias) when bias is non-NULL.
template <int W>
__device__ __forceinline__ void ln_stats(const float* __restrict__ x, const float* __restrict__ bias, float (&d)[W / 32],
                                         float& rstd, int lane) {
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < W / 32; ++k) {
    d[k] = bias != nullptr ? __fadd_rn(x[lane + 32 * k], bias[lane + 32 * k]) : x[lane + 32 * k];
    s += d[k];
  }
  const float mean = warp_sum(s) / (float)W;
  float ss = 0.f;
#pragma unroll
  for (int k = 0; k < W / 32; ++k) {
    d[k] = d[k] - mean;
    ss = __fadd_rn(ss, __fmul_rn(d[k], d[k]));
  }
  rstd = 1.f / sqrtf(warp_sum(ss) / (float)W + 1e-5f);
#pragma unroll
  for (int k = 0; k < W / 32; ++k) d[k] = __fmul_rn(d[k], rstd);   // x_hat
}

template <int W>
__global__ void __launch_bounds__(256) layernorm_fwd_kernel(long rows, const float* __restrict__ x,
                                                            const float* __restrict__ bias, int relu,
                                                            float* __restrict__ y) {
  const long row = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  float d[W / 32], rstd;
  ln_stats<W>(x + row * W, bias, d, rstd, lane);
#pragma unroll
  for (int k = 0; k < W / 32; ++k) y[row * W + lane + 32 * k] = relu ? fmaxf(d[k], 0.f) : d[k];
}

template <int W>
__global__ void __launch_bounds__(256) layernorm_bwd_kernel(long rows, const float* __restrict__ x,
                                                            const float* __restrict__ bias, const float* __restrict__ dy, int relu, float* __restrict__ dx) {
  const long row = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  float d[W / 32], g[W / 32], rstd;
  ln_stats<W>(x + row * W, bias, d, rstd, lane);
  float sg = 0.f, sgx = 0.f;
#pragma unroll
  for (int k = 0; k < W / 32; ++k) {
    const float gy = dy[row * W + lane + 32 * k];
    g[k] = (relu && !(d[k] > 0.f)) ? 0.f : gy;
    sg += g[k];
    sgx = __fadd_rn(sgx, __fmul_rn(g[k], d[k]));
  }
  const float mg = warp_sum(sg) / (float)W, mgx = warp_sum(sgx) / (float)W;
#pragma unroll
  for (int k = 0; k < W / 32; ++k)
    dx[row * W + lane + 32 * k] = __fmul_rn(rstd, __fsub_rn(__fsub_rn(g[k], mg), __fmul_rn(d[k], mgx)));
}

__global__ void ema_f32_kernel(long n, const float* __restrict__ theta, float* __restrict__ xi, float tau) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) xi[i] = __fadd_rn(xi[i], __fmul_rn(tau, __fsub_rn(theta[i], xi[i])));
}

__global__ void add_f32_kernel(long n, const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ out) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = __fadd_rn(a[i], b[i]);
}

}  // namespace riqn

using namespace riqn;

RIQN_API int riqn_curl_infonce_fwd_bwd(int batch, int dim, const float* z_a, const float* z_k, const float* w, float coef,
                                       float* loss_rows, float* dz_a, float* dw, float* logits_out, void* stream) {
  if (batch < 2 || batch > CURL_MAX_BATCH || dim != CURL_D || !isfinite(coef) || !z_a || !z_k || !w || !loss_rows ||
      !dz_a || !dw)
    return (int)cudaErrorInvalidValue;
  cudaStream_t s = (cudaStream_t)stream;
  const size_t smem = curl_smem_bytes(batch);
  static PerDeviceOnce once;
  const int d = PerDeviceOnce::device();
  if (!once.done[d]) {
    RIQN_CUDA(cudaFuncSetAttribute(curl_infonce_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   (int)curl_smem_bytes(CURL_MAX_BATCH)));
    once.done[d] = true;
  }
  StreamScratch g;
  RIQN_CUDA(g.alloc((size_t)batch * CURL_D, s));
  riqn::note_launches(2);
  curl_infonce_rows_kernel<<<riqn_cdiv(batch, CURL_ROWS), CURL_THREADS, smem, s>>>(
      batch, z_a, z_k, w, coef / (float)batch, loss_rows, dz_a, g.p, logits_out);
  RIQN_LAUNCH_CHECK();
  curl_infonce_dw_kernel<<<CURL_D * CURL_D / 256, 256, 0, s>>>(batch, z_a, g.p, dw);
  return (int)cudaGetLastError();
}

RIQN_API int riqn_layernorm_fwd(long rows, int width, const float* x, const float* bias, int relu, float* y,
                                void* stream) {
  if (rows < 1 || (width != 128 && width != 512) || !x || !y) return (int)cudaErrorInvalidValue;
  riqn::note_launches(1);
  const int grid = riqn_cdiv(rows * 32, 256);
  if (width == 128) layernorm_fwd_kernel<128><<<grid, 256, 0, (cudaStream_t)stream>>>(rows, x, bias, relu, y);
  else layernorm_fwd_kernel<512><<<grid, 256, 0, (cudaStream_t)stream>>>(rows, x, bias, relu, y);
  return (int)cudaGetLastError();
}

RIQN_API int riqn_layernorm_bwd(long rows, int width, const float* x, const float* bias, const float* dy, int relu,
                                float* dx, void* stream) {
  if (rows < 1 || (width != 128 && width != 512) || !x || !dy || !dx) return (int)cudaErrorInvalidValue;
  riqn::note_launches(1);
  const int grid = riqn_cdiv(rows * 32, 256);
  if (width == 128) layernorm_bwd_kernel<128><<<grid, 256, 0, (cudaStream_t)stream>>>(rows, x, bias, dy, relu, dx);
  else layernorm_bwd_kernel<512><<<grid, 256, 0, (cudaStream_t)stream>>>(rows, x, bias, dy, relu, dx);
  return (int)cudaGetLastError();
}

RIQN_API int riqn_ema_f32(long n, const float* theta, float* xi, float tau, void* stream) {
  if (n < 1 || !theta || !xi || !isfinite(tau) || !(tau > 0.f) || !(tau <= 1.f)) return (int)cudaErrorInvalidValue;
  riqn::note_launches(1);
  ema_f32_kernel<<<riqn_cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(n, theta, xi, tau);
  return (int)cudaGetLastError();
}

RIQN_API int riqn_add_f32(long n, const float* a, const float* b, float* out, void* stream) {
  if (n < 1 || !a || !b || !out) return (int)cudaErrorInvalidValue;
  riqn::note_launches(1);
  add_f32_kernel<<<riqn_cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(n, a, b, out);
  return (int)cudaGetLastError();
}

RIQN_API int riqn_colsum_add(long rows, int cols, const float* x, float* out, void* stream) {
  if (rows < 1 || cols < 1 || !x || !out) return (int)cudaErrorInvalidValue;
  riqn::note_launches(2);
  return colsum_add(rows, cols, x, out, (cudaStream_t)stream);
}
