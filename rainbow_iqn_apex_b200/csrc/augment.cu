// Random-shift image augmentation (DrQ: Kostrikov, Yarats & Fergus, ICLR 2021; no counterpart in the reference): the
// per-sample shift draw and the edge-replicating shift of a batch of frame stacks, as ops behind the C-ABI in
// include/riqn_b200.h.
//
// riqn_random_shift moves one (sample, channel) plane per CTA through shared memory: the plane arrives with 16-byte loads,
// every thread builds 4-byte output words from clamped source columns (an unaligned 4-pixel run of one source row is two
// aligned shared-memory words and one __byte_perm), the words go to a second shared plane, and the plane leaves with
// 16-byte stores.  Nothing is accumulated: every output element is a copy of one input element.
#include "common.cuh"
#include "../../include/riqn_b200.h"

namespace riqn {
constexpr int SHIFT_THREADS = 256;
constexpr int SHIFT_MAX_PLANE = 48 * 1024;     // bytes of one (H, W) plane; the CTA holds two

// Pairs 2*i4 and 2*i4 + 1 read the four words of Philox draw i4, the words riqn_fill_uniform(2n, seed, stream) turns into
// its values 4*i4 .. 4*i4 + 3.  m = x >> 8 is the 24-bit integer behind that uniform (m + 0.5) / 2^24, and
// (m (2p+1)) >> 24 is floor((m / 2^24) (2p+1)) in integer arithmetic: in [0, 2p] for every m < 2^24.
__global__ void fill_shifts_kernel(long n, int pad, uint64_t seed, uint64_t stream, int* __restrict__ out,
                                   const riqn_dyn_state* __restrict__ dyn) {
  if (dyn) stream += dyn->rng_offset;
  const long i4 = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const long words = 2 * n;
  if (i4 * 4 >= words) return;
  const uint4 r = Philox::draw(seed, stream, (uint64_t)i4);
  const uint32_t w[4] = {r.x, r.y, r.z, r.w};
  const uint64_t span = 2 * (uint64_t)pad + 1;
#pragma unroll
  for (int j = 0; j < 4; ++j)
    if (i4 * 4 + j < words) out[i4 * 4 + j] = (int)(((uint64_t)(w[j] >> 8) * span) >> 24) - pad;
}

__device__ __forceinline__ int clampi(int v, int hi) { return min(max(v, 0), hi); }

// Output word w of a shifted uint8 plane: pixels 4w .. 4w+3 in row-major order, pixel (y, x) = in[clamp(y + dy), clamp(x + dx)].
__device__ __forceinline__ uint32_t shifted_word(const unsigned char* __restrict__ s, int w, int H, int W, int dy, int dx) {
  const int e0 = 4 * w;
  const int y = e0 / W, x = e0 - y * W;
  if (x + 3 < W && x + dx >= 0 && x + dx + 3 < W) {       // one row, no column clamped: a funnel of two aligned words
    const int a = clampi(y + dy, H - 1) * W + x + dx;
    const uint32_t* s32 = reinterpret_cast<const uint32_t*>(s);
    const int q = a >> 2, r = a & 3;
    const uint32_t lo = s32[q];
    const uint32_t hi = r ? s32[q + 1] : lo;
    return __byte_perm(lo, hi, 0x3210u + 0x1111u * (uint32_t)r);
  }
  uint32_t v = 0;
  for (int k = 0; k < 4; ++k) {                            // a clamped column, or a word that runs into the next row(s)
    const int yy = (e0 + k) / W, xx = e0 + k - yy * W;
    v |= (uint32_t)s[clampi(yy + dy, H - 1) * W + clampi(xx + dx, W - 1)] << (8 * k);
  }
  return v;
}

__device__ __forceinline__ uint32_t shifted_word(const float* __restrict__ s, int w, int H, int W, int dy, int dx) {
  const int y = w / W, x = w - y * W;
  return __float_as_uint(s[clampi(y + dy, H - 1) * W + clampi(x + dx, W - 1)]);
}

// One CTA per (image, channel): image i < B reads in0 + i*s0, image B + i reads in1 + i*s1 (strides in elements).
template <typename T>
__global__ void __launch_bounds__(SHIFT_THREADS, 4)   // 4 CTAs of 64 registers per thread: no spills in the uint8 path
    random_shift_kernel(int B, int C, int H, int W, const T* __restrict__ in0, long s0, const T* __restrict__ in1, long s1,
                        const int* __restrict__ shifts, T* __restrict__ out) {
  extern __shared__ uint4 sm_shift[];
  const int hw = H * W;
  const int nvec = hw * (int)sizeof(T) / 16, nword = 4 * nvec;
  uint4* sin = sm_shift;
  uint4* sout = sm_shift + nvec;
  const int img = blockIdx.x / C, c = blockIdx.x - img * C;
  const T* src = (img < B ? in0 + (long)img * s0 : in1 + (long)(img - B) * s1) + (long)c * hw;
  // |dy| >= H (|dx| >= W) clamps every row (column) to the edge, as H (W) does: bounding them keeps y + dy in range
  const int dy = min(max(shifts[2 * img], -H), H), dx = min(max(shifts[2 * img + 1], -W), W);
  const uint4* src4 = reinterpret_cast<const uint4*>(src);
  for (int v = threadIdx.x; v < nvec; v += SHIFT_THREADS) sin[v] = __ldg(src4 + v);
  __syncthreads();
  const T* splane = reinterpret_cast<const T*>(sin);
  uint32_t* sw = reinterpret_cast<uint32_t*>(sout);
  for (int w = threadIdx.x; w < nword; w += SHIFT_THREADS) sw[w] = shifted_word(splane, w, H, W, dy, dx);
  __syncthreads();
  uint4* dst4 = reinterpret_cast<uint4*>(out + ((long)img * C + c) * hw);
  for (int v = threadIdx.x; v < nvec; v += SHIFT_THREADS) dst4[v] = sout[v];
}
}  // namespace riqn

using namespace riqn;

RIQN_API int riqn_fill_shifts(long n, int pad, unsigned long long seed, unsigned long long stream_id, int* out,
                              const riqn_dyn_state* dyn, void* stream) {
  if (n < 0 || pad < 0 || pad >= (1 << 30) || (n > 0 && out == nullptr)) return (int)cudaErrorInvalidValue;
  riqn::note_launches(1);
  if (n == 0) return 0;
  fill_shifts_kernel<<<riqn_cdiv((2 * n + 3) / 4, 256), 256, 0, (cudaStream_t)stream>>>(n, pad, seed, stream_id, out, dyn);
  return (int)cudaGetLastError();
}

RIQN_API int riqn_random_shift(int B, int C, int H, int W, const void* in0, long in0_bstride, const void* in1,
                               long in1_bstride, int is_u8, const int* shifts, void* out, void* stream) {
  if (B < 1 || C < 1 || H < 1 || W < 1 || in0 == nullptr || shifts == nullptr || out == nullptr || (is_u8 != 0 && is_u8 != 1))
    return (int)cudaErrorInvalidValue;
  const long esz = is_u8 ? 1 : 4;
  const long plane = (long)H * W * esz, chw = (long)C * H * W;
  const long images = in1 != nullptr ? 2L * B : (long)B;
  const auto misaligned = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) != 0; };
  if (plane % 16 || plane > SHIFT_MAX_PLANE || images * C > 0x7fffffffL || in0_bstride < chw || misaligned(in0) ||
      (in0_bstride * esz) % 16 || misaligned(out) ||
      (in1 != nullptr && (in1_bstride < chw || misaligned(in1) || (in1_bstride * esz) % 16)))
    return (int)cudaErrorInvalidValue;
  static PerDeviceOnce attr_once;
  const int attr_dev = PerDeviceOnce::device();
  if (!attr_once.done[attr_dev]) {
    RIQN_CUDA(cudaFuncSetAttribute(random_shift_kernel<unsigned char>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   2 * SHIFT_MAX_PLANE));
    RIQN_CUDA(cudaFuncSetAttribute(random_shift_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   2 * SHIFT_MAX_PLANE));
    attr_once.done[attr_dev] = true;
  }
  riqn::note_launches(1);
  const dim3 grid((unsigned)(images * C));
  const size_t smem = (size_t)(2 * plane);
  cudaStream_t s = (cudaStream_t)stream;
  if (is_u8)
    random_shift_kernel<unsigned char><<<grid, SHIFT_THREADS, smem, s>>>(
        B, C, H, W, (const unsigned char*)in0, in0_bstride, (const unsigned char*)in1, in1_bstride, shifts,
        (unsigned char*)out);
  else
    random_shift_kernel<float><<<grid, SHIFT_THREADS, smem, s>>>(B, C, H, W, (const float*)in0, in0_bstride,
                                                                  (const float*)in1, in1_bstride, shifts, (float*)out);
  return (int)cudaGetLastError();
}
