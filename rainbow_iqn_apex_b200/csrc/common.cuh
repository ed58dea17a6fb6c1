// Shared device/host helpers for the Rainbow-IQN Ape-X learner hot path (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

#define RIQN_API extern "C" __attribute__((visibility("default")))

#define RIQN_LAUNCH_CHECK()                                   \
  do {                                                        \
    cudaError_t _e = cudaGetLastError();                      \
    if (_e != cudaSuccess) return (int)_e;                    \
  } while (0)

#define RIQN_CUDA(expr)                                       \
  do {                                                        \
    cudaError_t _e = (expr);                                  \
    if (_e != cudaSuccess) return (int)_e;                    \
  } while (0)

namespace riqn {
void note_launches(int n);   // bookkeeping for riqn_launch_count()

// Deterministic cross-block sums.  A float atomicAdd makes a sum depend on which block arrives first, and the learner
// feeds its losses back into the prioritized sampler, so last-bit differences would change which transitions later
// steps draw.  Instead every contributing block writes its partial to its own slot of a scratch buffer and
// sum_slots_add() adds the slots in slot order.
// out[i] += sum_{k < slots} part[k * n + i], k ascending
int sum_slots_add(int slots, int n, const float* part, float* out, cudaStream_t s);
}  // namespace riqn

static inline int riqn_cdiv(long a, long b) { return (int)((a + b - 1) / b); }

// Scratch memory of one entry-point call: taken from the device's stream-ordered memory pool on the calling stream and
// handed back on the same stream when the call returns, i.e. after every kernel that uses it has been enqueued
// (cudaMallocAsync / cudaFreeAsync).  No host synchronisation, no state shared between calls or streams; inside a CUDA
// graph capture it becomes an allocation node of the graph.
struct StreamScratch {
  float* p = nullptr;
  cudaStream_t s = nullptr;
  cudaError_t alloc(size_t n, cudaStream_t stream) {
    s = stream;
    return cudaMallocAsync(reinterpret_cast<void**>(&p), n * sizeof(float), stream);
  }
  ~StreamScratch() {
    if (p != nullptr) cudaFreeAsync(p, s);
  }
};

// ----------------------------------------------------------------------------------------------
// Philox4x32-10 counter RNG (Salmon et al. 2011); stateless: value = f(seed, stream, index).
// ----------------------------------------------------------------------------------------------
struct Philox {
  static __device__ __forceinline__ uint4 round10(uint4 ctr, uint2 key) {
#pragma unroll
    for (int i = 0; i < 10; ++i) {
      const uint32_t hi0 = __umulhi(0xD2511F53u, ctr.x), lo0 = 0xD2511F53u * ctr.x;
      const uint32_t hi1 = __umulhi(0xCD9E8D57u, ctr.z), lo1 = 0xCD9E8D57u * ctr.z;
      ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
      key.x += 0x9E3779B9u;
      key.y += 0xBB67AE85u;
    }
    return ctr;
  }
  static __device__ __forceinline__ uint4 draw(uint64_t seed, uint64_t stream, uint64_t index) {
    uint4 ctr = make_uint4((uint32_t)index, (uint32_t)(index >> 32), (uint32_t)stream, (uint32_t)(stream >> 32));
    uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
    return round10(ctr, key);
  }
  // (0,1) open interval, 24-bit resolution like torch's uniform_ on fp32
  static __device__ __forceinline__ float u01(uint32_t x) { return ((x >> 8) + 0.5f) * (1.0f / 16777216.0f); }
  static __device__ __forceinline__ double u01d(uint32_t a, uint32_t b) {
    const uint64_t x = (((uint64_t)a << 32) | b) >> 11;  // 53 bits
    return ((double)x + 0.5) * (1.0 / 9007199254740992.0);
  }
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// One-time PER-DEVICE initialisation (cudaFuncSetAttribute opt-ins, SM count): a process may drive several GPUs (learner
// and actor networks on different devices), and the shared-memory opt-in is per device/context.  Idempotent work only:
// two threads racing on the same device both perform it before either marks it done.
struct PerDeviceOnce {
  bool done[64] = {};
  int sms[64] = {};
  static int device() {
    int d = 0;
    cudaGetDevice(&d);
    return d & 63;
  }
};

// SM count of the current device: grid size of the persistent kernels and the split-K choices.
inline int riqn_sms() {
  static int sms[64] = {};
  const int d = PerDeviceOnce::device();
  if (sms[d] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, d) != cudaSuccess || n < 1) n = 132;   // H100 SXM
    sms[d] = n;
  }
  return sms[d];
}
