// fp32 CUDA-core GEMM with fused epilogues.  Used for the small / oddly-shaped products on the
// learner path (conv im2col products, quantile embedding K=64, z-layers, weight-gradient
// reductions) and as the fp32 cross-check for the wgmma path (gemm_tc.cu).
//
// Tile 128x128x16, 256 threads, 8x8 register micro-tile (4+4 split so shared-memory reads are
// 128-bit and conflict-free), global->register prefetch of the next k-slab overlapped with the
// FMAs of the current one.
#include "common.cuh"
#include "gemm.h"

namespace riqn {

constexpr int BM = 128, BN = 128, BK = 16, NT = 256;

template <int EPI>
__device__ __forceinline__ void epi_one(float v, int m, int n, int N, float* __restrict__ C, long ldc, const EpiArgs& e) {
  if (EPI == EPI_STORE) {
    C[(long)m * ldc + n] = e.alpha * v;
  } else if (EPI == EPI_BIAS) {
    C[(long)m * ldc + n] = v + e.bias[n];
  } else if (EPI == EPI_BIAS_RELU) {
    C[(long)m * ldc + n] = fmaxf(v + e.bias[n], 0.f);
  } else if (EPI == EPI_BIAS_RELU_NCHW) {
    const int b = m / e.ohw, p = m - b * e.ohw;
    C[((long)b * N + n) * e.ohw + p] = fmaxf(v + e.bias[n], 0.f);
  } else if (EPI == EPI_EMBED) {
    C[(long)m * ldc + n] = e.feat[(long)(m / e.batch) * N + n] * fmaxf(v + e.bias[n], 0.f);
  } else if (EPI == EPI_NOISY_WGRAD) {        // split 1 only: one block owns the element
    C[(long)m * ldc + n] += v;
    e.out2[(long)m * ldc + n] += __fmul_rn(v, e.eps[(long)m * ldc + n]);
  } else if (EPI == EPI_SLAB) {
    C[(long)m * ldc + n] = v;
  }
}

template <int EPI, bool AKC, bool BKC>
__global__ void __launch_bounds__(NT, 2)
gemm_simt_kernel(int M, int N, int K, const float* __restrict__ A, long sAm, long sAk,
                 const float* __restrict__ B, long sBn, long sBk, float* __restrict__ C, long ldc,
                 EpiArgs e, int kchunk) {
  __shared__ __align__(16) float As[2][BK][BM + 4];
  __shared__ __align__(16) float Bs[2][BK][BN + 4];
  const int tid = threadIdx.x;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const int kbeg = blockIdx.z * kchunk;
  const int kend = min(K, kbeg + kchunk);
  const int tx = tid & 15, ty = tid >> 4;

  float ra[8], rb[8];
  auto gload = [&](int kt) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int idx = tid + i * NT;
      int mm, kk;
      if (AKC) { kk = idx % BK; mm = idx / BK; } else { mm = idx % BM; kk = idx / BM; }
      const int gm = m0 + mm, gk = kt + kk;
      ra[i] = (gm < M && gk < kend) ? __ldg(&A[(long)gm * sAm + (long)gk * sAk]) : 0.f;
      int nn, kb;
      if (BKC) { kb = idx % BK; nn = idx / BK; } else { nn = idx % BN; kb = idx / BN; }
      const int gn = n0 + nn, gk2 = kt + kb;
      rb[i] = (gn < N && gk2 < kend) ? __ldg(&B[(long)gn * sBn + (long)gk2 * sBk]) : 0.f;
    }
  };
  auto sstore = [&](int buf) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int idx = tid + i * NT;
      int mm, kk;
      if (AKC) { kk = idx % BK; mm = idx / BK; } else { mm = idx % BM; kk = idx / BM; }
      As[buf][kk][mm] = ra[i];
      int nn, kb;
      if (BKC) { kb = idx % BK; nn = idx / BK; } else { nn = idx % BN; kb = idx / BN; }
      Bs[buf][kb][nn] = rb[i];
    }
  };

  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  if (kbeg < kend) {
    gload(kbeg);
    sstore(0);
  }
  __syncthreads();
  int buf = 0;
  for (int kt = kbeg; kt < kend; kt += BK) {
    const bool more = kt + BK < kend;
    if (more) gload(kt + BK);
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][k][64 + ty * 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][k][64 + tx * 4]);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (more) sstore(buf ^ 1);
    __syncthreads();
    buf ^= 1;
  }

  if (EPI == EPI_SLAB) C += (long)blockIdx.z * e.slab;
  const bool vec_ok = (EPI == EPI_STORE || EPI == EPI_BIAS_RELU || EPI == EPI_EMBED || EPI == EPI_BIAS || EPI == EPI_SLAB) &&
                      ((ldc & 3) == 0) && ((N & 3) == 0) && ((reinterpret_cast<uintptr_t>(C) & 15) == 0);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int m = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
    if (m >= M) continue;
#pragma unroll
    for (int jh = 0; jh < 2; ++jh) {
      const int n = n0 + jh * 64 + tx * 4;
      if (n >= N) continue;
      if (vec_ok && n + 3 < N) {
        float4 v = make_float4(acc[i][jh * 4 + 0], acc[i][jh * 4 + 1], acc[i][jh * 4 + 2], acc[i][jh * 4 + 3]);
        if (EPI == EPI_STORE) {
          v.x *= e.alpha; v.y *= e.alpha; v.z *= e.alpha; v.w *= e.alpha;
        } else if (EPI != EPI_SLAB) {
          const float4 bb = *reinterpret_cast<const float4*>(&e.bias[n]);
          v.x += bb.x; v.y += bb.y; v.z += bb.z; v.w += bb.w;
          if (EPI != EPI_BIAS) {
            v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
          }
          if (EPI == EPI_EMBED) {
            const float4 f = *reinterpret_cast<const float4*>(&e.feat[(long)(m / e.batch) * N + n]);
            v.x *= f.x; v.y *= f.y; v.z *= f.z; v.w *= f.w;
          }
        }
        *reinterpret_cast<float4*>(&C[(long)m * ldc + n]) = v;
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (n + j < N) epi_one<EPI>(acc[i][jh * 4 + j], m, n + j, N, C, ldc, e);
      }
    }
  }
}

template <int EPI>
static int launch_epi(int M, int N, int K, const float* A, long sAm, long sAk, const float* B, long sBn, long sBk,
                      float* C, long ldc, const EpiArgs& e, int split_k, cudaStream_t s) {
  const int kchunk = gemm_f32_kchunk(K, split_k);
  split_k = gemm_f32_splits(K, split_k);
  dim3 grid((N + BN - 1) / BN, (M + BM - 1) / BM, split_k);
  const bool akc = (sAk == 1), bkc = (sBk == 1);
#define RIQN_GEMM_GO(AK_, BK_) \
  gemm_simt_kernel<EPI, AK_, BK_><<<grid, NT, 0, s>>>(M, N, K, A, sAm, sAk, B, sBn, sBk, C, ldc, e, kchunk)
  if (akc && bkc) RIQN_GEMM_GO(true, true);
  else if (akc) RIQN_GEMM_GO(true, false);
  else if (bkc) RIQN_GEMM_GO(false, true);
  else RIQN_GEMM_GO(false, false);
#undef RIQN_GEMM_GO
  return (int)cudaGetLastError();
}

// Rows of K per split: ceil(K / split_k) rounded up to whole k-slabs, so the last split may be shorter or empty.
int gemm_f32_kchunk(int K, int split_k) {
  if (split_k < 1) split_k = 1;
  const int kchunk = (K + split_k - 1) / split_k;
  return kchunk < BK ? BK : ((kchunk + BK - 1) / BK) * BK;
}

// Non-empty splits of that cut (<= split_k).
int gemm_f32_splits(int K, int split_k) {
  const int kchunk = gemm_f32_kchunk(K, split_k);
  const int s = (K + kchunk - 1) / kchunk;
  return s < 1 ? 1 : s;
}

int gemm_f32(int M, int N, int K, const float* A, long sAm, long sAk, const float* B, long sBn, long sBk,
             float* C, long ldc, int epi, const EpiArgs& e, int split_k, cudaStream_t s) {
  if (M <= 0 || N <= 0) return 0;
  if (split_k > 1 && epi != EPI_SLAB) return (int)cudaErrorInvalidValue;
  switch (epi) {
    case EPI_STORE: return launch_epi<EPI_STORE>(M, N, K, A, sAm, sAk, B, sBn, sBk, C, ldc, e, split_k, s);
    case EPI_BIAS: return launch_epi<EPI_BIAS>(M, N, K, A, sAm, sAk, B, sBn, sBk, C, ldc, e, split_k, s);
    case EPI_BIAS_RELU: return launch_epi<EPI_BIAS_RELU>(M, N, K, A, sAm, sAk, B, sBn, sBk, C, ldc, e, split_k, s);
    case EPI_BIAS_RELU_NCHW: return launch_epi<EPI_BIAS_RELU_NCHW>(M, N, K, A, sAm, sAk, B, sBn, sBk, C, ldc, e, split_k, s);
    case EPI_EMBED: return launch_epi<EPI_EMBED>(M, N, K, A, sAm, sAk, B, sBn, sBk, C, ldc, e, split_k, s);
    case EPI_NOISY_WGRAD: return launch_epi<EPI_NOISY_WGRAD>(M, N, K, A, sAm, sAk, B, sBn, sBk, C, ldc, e, split_k, s);
    case EPI_SLAB: return launch_epi<EPI_SLAB>(M, N, K, A, sAm, sAk, B, sBn, sBk, C, ldc, e, split_k, s);
  }
  return (int)cudaErrorInvalidValue;
}

// C (M, N row-major) += A B^T with K cut as gemm_f32_kchunk does: every split stores its partial product in its own slab
// of stream scratch (EPI_SLAB) and sum_slots_add adds the slabs in split order onto C, so the sum does not depend on
// which split finishes first.  Two launches.
int gemm_f32_add(int M, int N, int K, const float* A, long sAm, long sAk, const float* B, long sBn, long sBk, float* C,
                 int split_k, cudaStream_t s) {
  if (M <= 0 || N <= 0) return 0;
  const long n = (long)M * N;
  const int splits = gemm_f32_splits(K, split_k);
  StreamScratch part;
  RIQN_CUDA(part.alloc((size_t)splits * n, s));
  EpiArgs e;
  e.slab = n;
  const int rc = gemm_f32(M, N, K, A, sAm, sAk, B, sBn, sBk, part.p, N, EPI_SLAB, e, split_k, s);
  if (rc) return rc;
  return sum_slots_add(splits, (int)n, part.p, C, s);
}

}  // namespace riqn

// Test hook (C-ABI): plain strided fp32 product, C = A * B^T in the (m,k)/(n,k) stride convention.
RIQN_API int riqn_gemm_f32(int M, int N, int K, const float* A, long sAm, long sAk, const float* B, long sBn,
                           long sBk, float* C, long ldc, void* stream) {
  riqn::note_launches(1);
  riqn::EpiArgs e;
  return riqn::gemm_f32(M, N, K, A, sAm, sAk, B, sBn, sBk, C, ldc, riqn::EPI_STORE, e, 1, (cudaStream_t)stream);
}
