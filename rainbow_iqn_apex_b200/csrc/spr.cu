// SPR (Schwarzer et al., ICLR 2021): the packing between the (B, 64, 7, 7) latent and the strip convolution's block
// matrix, its adjoint, the transition convolutions' weight images and the fused masked negative cosine.  See
// include/riqn_b200.h for the statements.
//
// No atomics: every element is written once, and every sum is a sequential fp32 chain in a stated order or the warp_sum
// butterfly, so the results are bitwise reproducible.
#include <math.h>

#include "common.cuh"
#include "../../include/riqn_b200.h"

namespace riqn {

using bf16 = __nv_bfloat16;

constexpr int SPR_CH = 64;           // latent channels
constexpr int SPR_E = 7;              // latent edge
constexpr int SPR_G = SPR_E + 2;      // zero-bordered edge (the strip grid of a 3x3 / stride 1 / pad 0 convolution)
constexpr int SPR_DIM = 128;          // projection width the cosine kernel is specialised for
constexpr int SPR_MAX_K = 12;
constexpr int SPR_MAX_ROWS = 4096;
constexpr int SPR_MAX_ACTIONS = 64;

// One thread per element of the (B*81, C) block matrix: row (b, gy, gx), column c.
__global__ void spr_pack_kernel(long n, int C, const float* __restrict__ z, const int64_t* __restrict__ actions,
                                int action_stride, int num_actions, bf16* __restrict__ hi, bf16* __restrict__ lo) {
  const long e = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const int c = (int)(e % C);
  const long row = e / C;
  const int g = (int)(row % (SPR_G * SPR_G));
  const long b = row / (SPR_G * SPR_G);
  const int y = g / SPR_G - 1, x = g % SPR_G - 1;
  float v = 0.f;
  if (y >= 0 && y < SPR_E && x >= 0 && x < SPR_E) {
    if (c < SPR_CH) v = z[((b * SPR_CH + c) * SPR_E + y) * SPR_E + x];
    else if (c - SPR_CH < num_actions) v = (actions[b * action_stride] == (int64_t)(c - SPR_CH)) ? 1.f : 0.f;
  }
  const bf16 h = __float2bfloat16_rn(v);
  hi[e] = h;
  lo[e] = __float2bfloat16_rn(v - __bfloat162float(h));
}

// out[b, c, y, x] = fl(acc[b, c, y, x] + din[b, c, y + 1, x + 1]) (or the crop alone without acc), c < 64.
__global__ void spr_unpack_grad_kernel(long n, int C, const float* __restrict__ din, const float* acc, float* out) {
  const long e = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const int x = (int)(e % SPR_E), y = (int)((e / SPR_E) % SPR_E), c = (int)((e / (SPR_E * SPR_E)) % SPR_CH);
  const long b = e / (SPR_CH * SPR_E * SPR_E);
  const float g = din[((b * C + c) * SPR_G + y + 1) * SPR_G + x + 1];
  out[e] = acc != nullptr ? __fadd_rn(acc[e], g) : g;
}

// Weight images of a 3x3 transition convolution (Cout, cin, 3, 3), zero-padded to cpad input channels: strip order
// column (dy*3 + dx)*cpad + c (hi / lo) and original order column c*9 + dy*3 + dx (hi_orig).  One thread per element.
__global__ void spr_weight_images_kernel(int cout, int cin, int cpad, const float* __restrict__ w, bf16* __restrict__ hi,
                                         bf16* __restrict__ lo, bf16* __restrict__ hi_orig) {
  const int K = cpad * 9;
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= cout * K) return;
  const int o = e / K, k = e % K;
  {
    const int c = k % cpad, s = k / cpad;
    const float v = c < cin ? w[(o * cin + c) * 9 + s] : 0.f;
    const bf16 h = __float2bfloat16_rn(v);
    hi[e] = h;
    lo[e] = __float2bfloat16_rn(v - __bfloat162float(h));
  }
  const int c = k / 9, s = k % 9;
  hi_orig[e] = __float2bfloat16_rn(c < cin ? w[(o * cin + c) * 9 + s] : 0.f);
}

// gw[o, c, s] = fl(gw[o, c, s] + gpad[o, c, s]) for c < cin (gw (cout, cin, 9), gpad (cout, cpad, 9)).
__global__ void spr_weight_grad_add_kernel(int cout, int cin, int cpad, const float* __restrict__ gpad,
                                           float* __restrict__ gw) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= cout * cin * 9) return;
  const int s = e % 9, c = (e / 9) % cin, o = e / (9 * cin);
  gw[e] = __fadd_rn(gw[e], gpad[(o * cpad + c) * 9 + s]);
}

// One CTA per sample b, warp k = step: lane l holds elements l + 32j (j = 0..3).
__global__ void __launch_bounds__(32 * SPR_MAX_K)
spr_cosine_kernel(int B, int K, const float* __restrict__ pred, const float* __restrict__ target,
                  const uint8_t* __restrict__ valid, float scale, float* __restrict__ loss_rows,
                  float* __restrict__ dpred) {
  __shared__ float terms[SPR_MAX_K];
  const int b = blockIdx.x, k = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (k < K) {
    const long r = (long)k * B + b;
    const float* p = pred + r * SPR_DIM;
    const float* t = target + r * SPR_DIM;
    float pv[SPR_DIM / 32], tv[SPR_DIM / 32];
    float spp = 0.f, stt = 0.f, spt = 0.f;
#pragma unroll
    for (int j = 0; j < SPR_DIM / 32; ++j) {
      pv[j] = p[lane + 32 * j];
      tv[j] = t[lane + 32 * j];
      spp = __fadd_rn(spp, __fmul_rn(pv[j], pv[j]));
      stt = __fadd_rn(stt, __fmul_rn(tv[j], tv[j]));
      spt = __fadd_rn(spt, __fmul_rn(pv[j], tv[j]));
    }
    spp = warp_sum(spp);
    stt = warp_sum(stt);
    spt = warp_sum(spt);
    const float lp = sqrtf(spp), np_ = fmaxf(lp, 1e-12f), nt = fmaxf(sqrtf(stt), 1e-12f);
    const float cosv = __fdiv_rn(spt, __fmul_rn(np_, nt));
    const bool v = valid[(long)b * K + k] != 0;
    if (lane == 0) terms[k] = v ? -cosv : 0.f;
    const float sv = v ? -scale : 0.f;
#pragma unroll
    for (int j = 0; j < SPR_DIM / 32; ++j) {
      const float th = __fdiv_rn(tv[j], nt);
      const float g = lp > 1e-12f ? __fsub_rn(th, __fmul_rn(cosv, __fdiv_rn(pv[j], np_))) : th;
      dpred[r * SPR_DIM + lane + 32 * j] = __fmul_rn(sv, __fdiv_rn(g, np_));
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int j = 0; j < K; ++j) s = __fadd_rn(s, terms[j]);
    loss_rows[b] = s;
  }
}

}  // namespace riqn

using namespace riqn;

RIQN_API int riqn_spr_pack(int batch, int channels, const float* latent, const long long* actions, int action_stride,
                           int num_actions, void* hi, void* lo, void* stream) {
  const bool with_a = channels == 2 * SPR_CH;
  if (batch < 1 || !latent || !hi || !lo || (channels != SPR_CH && !with_a) || (with_a != (actions != nullptr)) ||
      (with_a && (num_actions < 1 || num_actions > SPR_MAX_ACTIONS || action_stride < 1)))
    return (int)cudaErrorInvalidValue;
  riqn::note_launches(1);
  const long n = (long)batch * SPR_G * SPR_G * channels;
  spr_pack_kernel<<<riqn_cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(
      n, channels, latent, (const int64_t*)actions, action_stride, with_a ? num_actions : 0, (bf16*)hi, (bf16*)lo);
  return (int)cudaGetLastError();
}

RIQN_API int riqn_spr_unpack_grad(int batch, int channels, const float* din, const float* acc, float* out, void* stream) {
  if (batch < 1 || (channels != SPR_CH && channels != 2 * SPR_CH) || !din || !out) return (int)cudaErrorInvalidValue;
  riqn::note_launches(1);
  const long n = (long)batch * SPR_CH * SPR_E * SPR_E;
  spr_unpack_grad_kernel<<<riqn_cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(n, channels, din, acc, out);
  return (int)cudaGetLastError();
}

RIQN_API int riqn_spr_weight_images(int cout, int cin, int cpad, const float* w, void* hi, void* lo, void* hi_orig,
                                    void* stream) {
  if (cout < 1 || cout > 64 || cin < 1 || cin > cpad || cpad % 64 || !w || !hi || !lo || !hi_orig)
    return (int)cudaErrorInvalidValue;
  riqn::note_launches(1);
  spr_weight_images_kernel<<<riqn_cdiv((long)cout * cpad * 9, 256), 256, 0, (cudaStream_t)stream>>>(
      cout, cin, cpad, w, (bf16*)hi, (bf16*)lo, (bf16*)hi_orig);
  return (int)cudaGetLastError();
}

RIQN_API int riqn_spr_weight_grad_add(int cout, int cin, int cpad, const float* gpad, float* gw, void* stream) {
  if (cout < 1 || cin < 1 || cin > cpad || !gpad || !gw) return (int)cudaErrorInvalidValue;
  riqn::note_launches(1);
  spr_weight_grad_add_kernel<<<riqn_cdiv((long)cout * cin * 9, 256), 256, 0, (cudaStream_t)stream>>>(cout, cin, cpad,
                                                                                                    gpad, gw);
  return (int)cudaGetLastError();
}

RIQN_API int riqn_spr_cosine_fwd_bwd(int rows, int K, int dim, const float* pred, const float* target,
                                     const unsigned char* valid, float coef, float* loss_rows, float* dpred,
                                     void* stream) {
  if (rows < 1 || rows > SPR_MAX_ROWS || K < 1 || K > SPR_MAX_K || dim != SPR_DIM || !isfinite(coef) || !pred ||
      !target || !valid || !loss_rows || !dpred)
    return (int)cudaErrorInvalidValue;
  riqn::note_launches(1);
  spr_cosine_kernel<<<rows, 32 * K, 0, (cudaStream_t)stream>>>(rows, K, pred, target, valid, coef / (float)rows,
                                                               loss_rows, dpred);
  return (int)cudaGetLastError();
}
