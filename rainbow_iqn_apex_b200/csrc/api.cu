// Library identification entry points of the C-ABI (include/riqn_b200.h).
#include "common.cuh"
#include "../../include/riqn_b200.h"

RIQN_API int riqn_version(void) { return RIQN_B200_ABI_VERSION; }

RIQN_API int riqn_device_ok(void) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return -(int)e;
  int major = 0;
  e = cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
  if (e != cudaSuccess) return -(int)e;
  return major == 9 ? 1 : 0;
}

#include <atomic>
namespace riqn {
static std::atomic<long long> g_launches{0};
void note_launches(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

__global__ void sum_slots_add_kernel(int slots, int n, const float* __restrict__ part, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float acc = 0.f;
  for (int k = 0; k < slots; ++k) acc += part[(long)k * n + i];
  out[i] += acc;
}

int sum_slots_add(int slots, int n, const float* part, float* out, cudaStream_t s) {
  sum_slots_add_kernel<<<riqn_cdiv(n, 256), 256, 0, s>>>(slots, n, part, out);
  return (int)cudaGetLastError();
}
}  // namespace riqn

RIQN_API long long riqn_launch_count(void) { return riqn::g_launches.load(std::memory_order_relaxed); }

RIQN_API int riqn_zero_f32(float* p, long n, void* stream) {
  return (int)cudaMemsetAsync(p, 0, sizeof(float) * (size_t)n, (cudaStream_t)stream);
}
