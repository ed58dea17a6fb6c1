// Periodic network resets (SR-SPR, BBF): redraw segments of a flat parameter arena from their initial distribution,
// shrink-and-perturb others towards a fresh draw, and restart the arena's Adam moments, in one launch.  The arithmetic
// is stated at riqn_arena_reset in include/riqn_b200.h.
#include <math.h>

#include "common.cuh"
#include "../../include/riqn_b200.h"

namespace riqn {

struct ResetTable {
  riqn_reset_segment seg[RIQN_RESET_MAX_SEGMENTS];
  int nseg;
};

__device__ __forceinline__ float reset_value(const riqn_reset_segment& g, float theta, uint32_t word) {
  const float fresh =
      g.kind == RIQN_RESET_UNIFORM ? __fmul_rn(g.value, __fsub_rn(__fmul_rn(2.f, Philox::u01(word)), 1.f)) : g.value;
  return g.alpha == 0.f ? fresh : __fadd_rn(__fmul_rn(g.alpha, theta), __fmul_rn(__fsub_rn(1.f, g.alpha), fresh));
}

// Thread t owns elements 4t .. 4t+3, the four words of Philox draw t, as in riqn_fill_uniform.  Segments are sorted and
// disjoint: a binary search finds the first segment ending past 4t, and the four elements walk forward from there.
// ``vec``: the three arrays are 16-byte aligned, so a quad inside [0, n) (and inside one segment) moves as one float4.
__global__ void arena_reset_kernel(long n, float* __restrict__ params, float* __restrict__ exp_avg,
                                   float* __restrict__ exp_avg_sq, const __grid_constant__ ResetTable table,
                                   uint64_t seed, uint64_t stream, int vec) {
  const long i4 = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const long i0 = i4 * 4;
  if (i0 >= n) return;
  const bool quad = vec && i0 + 4 <= n;
  if (exp_avg && quad) {
    reinterpret_cast<float4*>(exp_avg)[i4] = make_float4(0.f, 0.f, 0.f, 0.f);
    reinterpret_cast<float4*>(exp_avg_sq)[i4] = make_float4(0.f, 0.f, 0.f, 0.f);
  } else if (exp_avg) {
    for (int j = 0; j < 4; ++j)
      if (i0 + j < n) exp_avg[i0 + j] = 0.f, exp_avg_sq[i0 + j] = 0.f;
  }
  int lo = 0, hi = table.nseg;               // first segment with end > i0
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (table.seg[mid].end > i0) hi = mid;
    else lo = mid + 1;
  }
  if (lo == table.nseg || table.seg[lo].begin >= i0 + 4) return;
  const uint4 r = Philox::draw(seed, stream, (uint64_t)i4);
  const uint32_t w[4] = {r.x, r.y, r.z, r.w};
  if (quad && table.seg[lo].begin <= i0 && i0 + 4 <= table.seg[lo].end) {
    const riqn_reset_segment g = table.seg[lo];
    float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
    if (g.alpha != 0.f) t = reinterpret_cast<const float4*>(params)[i4];
    reinterpret_cast<float4*>(params)[i4] =
        make_float4(reset_value(g, t.x, w[0]), reset_value(g, t.y, w[1]), reset_value(g, t.z, w[2]),
                    reset_value(g, t.w, w[3]));
    return;
  }
  int s = lo;
  for (int j = 0; j < 4; ++j) {
    const long i = i0 + j;
    if (i >= n) break;
    while (s < table.nseg && table.seg[s].end <= i) ++s;
    if (s == table.nseg) break;
    const riqn_reset_segment g = table.seg[s];
    if (i < g.begin) continue;
    params[i] = reset_value(g, g.alpha == 0.f ? 0.f : params[i], w[j]);
  }
}

}  // namespace riqn

RIQN_API int riqn_arena_reset(long n, float* params, float* exp_avg, float* exp_avg_sq, int nseg,
                              const riqn_reset_segment* segs, unsigned long long seed, unsigned long long stream_id,
                              void* stream) {
  if (n < 1 || !params || (exp_avg == nullptr) != (exp_avg_sq == nullptr) || nseg < 1 ||
      nseg > RIQN_RESET_MAX_SEGMENTS || !segs)
    return (int)cudaErrorInvalidValue;
  riqn::ResetTable table;
  long prev_end = 0;
  for (int k = 0; k < nseg; ++k) {
    const riqn_reset_segment& g = segs[k];
    const bool kind_ok = (g.kind == RIQN_RESET_UNIFORM && isfinite(g.value) && g.value > 0.f) ||
                         (g.kind == RIQN_RESET_CONSTANT && isfinite(g.value));
    if (g.begin < prev_end || g.end <= g.begin || g.end > n || !kind_ok || !(g.alpha >= 0.f && g.alpha < 1.f))
      return (int)cudaErrorInvalidValue;
    prev_end = g.end;
    table.seg[k] = g;
  }
  table.nseg = nseg;
  const int vec = (((uintptr_t)params | (uintptr_t)exp_avg | (uintptr_t)exp_avg_sq) & 15) == 0;
  riqn::note_launches(1);
  riqn::arena_reset_kernel<<<riqn_cdiv((n + 3) / 4, 256), 256, 0, (cudaStream_t)stream>>>(
      n, params, exp_avg, exp_avg_sq, table, seed, stream_id, vec);
  return (int)cudaGetLastError();
}
