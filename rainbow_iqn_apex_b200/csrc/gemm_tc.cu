// wgmma / TMA GEMM for the NoisyLinear hidden layers of the IQN head (the >90% of the learner step's FLOPs:
// reference model.py:153-154 forward, and its dgrad / wgrad), sm_90a.
//
//   C[m,n] = sum_k A[m,k] * B[n,k]        A (M,K) and B (N,K) both K-major bf16 in HBM, fp32 accumulate in registers
//
// * operands arrive by TMA (cp.async.bulk.tensor.2d, 128-byte swizzle) into a multi-stage shared-memory ring, issued by
//   one thread of the producer warpgroup,
// * two consumer warpgroups each own 64 rows of the 128-row tile and issue wgmma.mma_async (m64nBNk16) on shared-memory
//   descriptors; the accumulator lives in their registers,
// * after a tile's last k-block the consumers pass the accumulator through a shared-memory slab, 64 columns at a time,
//   so that each warp holds 32 rows x 32 columns with one ROW per lane, and apply the fused epilogue from there while
//   the producer already fetches the next tile's operands (the 128x256 forward, the bf16 data gradient and the quantile
//   embedding instead stage their fragments for TMA stores and go on to the next tile while the stores drain: MODE
//   bit 3, see TcCfg),
// * persistent CTAs (one per SM) walk (m-tile, n-tile, k-split) work units round-robin.
//
// Precision: NSPLIT == 1 multiplies bf16(A) * bf16(B).  NSPLIT == 3 takes each operand as hi + lo bf16 pairs
// (a = a_hi + a_lo exactly to ~2^-17) and accumulates a_hi*b_hi + a_hi*b_lo + a_lo*b_hi into the same accumulator: an
// fp32-faithful product (rel. error ~1e-5 per term) at 3 MMAs per k-step, which keeps the IQN loss within 1e-6 of the
// fp32 reference instead of bf16's 1e-4.
#include <cuda.h>
#include <cudaTypedefs.h>
#include <algorithm>
#include <map>
#include <mutex>
#include <tuple>

#include "common.cuh"
#include "gemm.h"
#include "../../include/riqn_b200.h"

namespace riqn {

using bf16 = __nv_bfloat16;

constexpr int TBM = 128, TBK = 64, MMA_K = 16;   // tile N (BN) is a template parameter: 128, or 64 / 32 for narrow outputs
constexpr int kConsumerWGs = 2;                   // consumer warpgroup g owns tile rows [64 g, 64 g + 64)
constexpr int kEpiWarps = 4 * kConsumerWGs;
constexpr int kTcThreads = 128 * (1 + kConsumerWGs);   // warpgroup 0: TMA producer (one thread issues), then the consumers
// Accumulator slab of one consumer warpgroup: 64 rows x 64 columns fp32, rows padded to 72 words so that the fragment
// deposit (a half-warp = 4 rows x 8 columns) is bank-conflict free.  Once read back it holds the four 4 KB per-warp
// staging tiles of the store helpers below.
constexpr uint32_t kSlabStride = 72, kSlabBytes = 64 * kSlabStride * 4;
constexpr uint32_t kSmemLimit = 232448;           // 227 KB of opt-in shared memory per CTA

// NSPLIT 1: a_hi*b_hi.  NSPLIT 3: a_hi*b_hi + a_hi*b_lo + a_lo*b_hi.  NSPLIT 2: A is exact in bf16 (e.g. uint8 pixels),
// only B is split: a_hi*b_hi + a_hi*b_lo.
//
// TMAEPI (128x256 single-pass TC_BIAS_RELU / TC_STORE, and the 128x128 TC_EMBED): the accumulator leaves through TMA
// stores instead of the slab.  Each consumer warpgroup stages 32-column chunks of its 64 rows in kEpiBufs rotating
// buffers of kEpiChunkBytes: a 64 x 32 fp32 box (8 KB, 128-byte swizzle; TC_BIAS_RELU) and one 64 x 32 16-bit box per
// image (4 KB each, 64-byte swizzle; the o_hi image, or the embedding's o_hi and o_lo).  The ring keeps kEpiStages
// stages and the buffers take what is left, up to kEpiBufsMax:
//   128x256 (48 KB stages, 3 of them = 144 KB): 3 fp32 + bf16 buffers per warpgroup (72 KB) in the forward, the whole
//     128 x 256 bf16 tile (8 buffers, 64 KB) in the data gradient;
//   TC_EMBED (64 KB stages with split operands, 32 KB without): its tiles are ONE k-block long, so two stages already
//     keep the next tile's operands in flight under every product, and a buffer comes up for rewriting a few hundred
//     cycles after its stores were issued.  Six 8 KB buffers per warpgroup (96 KB; a tile and a half) let those stores
//     finish reading behind the next tile's product instead of in front of it; the ring gets 2 (split) / 4 stages.
template <int NSPLIT, int BN, int EPI, bool TMAEPI = false>
struct TcCfg {
  static constexpr int kAOps = NSPLIT == 3 ? 2 : 1, kBOps = NSPLIT == 1 ? 1 : 2;     // hi (+ lo) images per operand
  static constexpr int kOps = kAOps;                                                 // (A images; B tile starts after them)
  static constexpr uint32_t kABytes = TBM * TBK * 2, kBBytes = BN * TBK * 2;
  static constexpr uint32_t kStageBytes = kAOps * kABytes + kBOps * kBBytes;         // 32 / 48 / 64 KB at BN = 128
  static constexpr uint32_t kEpiF32Bytes = EPI == TC_BIAS_RELU ? 64 * 32 * 4 : 0;
  static constexpr uint32_t kEpiChunkBytes = kEpiF32Bytes + (EPI == TC_EMBED ? 2 : 1) * 64 * 32 * 2;
  static constexpr int kEpiStages = EPI == TC_EMBED ? 2 : 3;
  static constexpr int kEpiBufsMax = EPI == TC_EMBED ? 6 : BN / 32;
  static constexpr int kEpiBufsFit = (kSmemLimit - 1024 - 256 - kEpiStages * kStageBytes) / (kConsumerWGs * kEpiChunkBytes);
  static constexpr int kEpiBufs = kEpiBufsFit > kEpiBufsMax ? kEpiBufsMax : kEpiBufsFit;
  static constexpr uint32_t kEpiBytes = TMAEPI ? kConsumerWGs * kEpiBufs * kEpiChunkBytes : kConsumerWGs * kSlabBytes;
  static_assert(!TMAEPI || (kEpiBufs >= 2 && (EPI == TC_EMBED ? BN == 128
                                                              : BN == 256 && NSPLIT == 1 && (EPI == TC_BIAS_RELU || EPI == TC_STORE))),
                "TMA-store epilogue: 128x256 single-pass TC_BIAS_RELU / TC_STORE or 128x128 TC_EMBED, at least two staging buffers");
  static_assert(TMAEPI || EPI != TC_EMBED, "the embedding has no slab epilogue");
  static constexpr uint32_t kRingBytes = kSmemLimit - 1024 /*align*/ - kEpiBytes - 256 /*barriers*/;
  static constexpr int kStages = kRingBytes / kStageBytes > 6 ? 6 : kRingBytes / kStageBytes;
  static constexpr uint32_t kSmemBytes = kStages * kStageBytes + 1024 + kEpiBytes + 256;
  static_assert(kSmemBytes <= kSmemLimit && kStages >= 2, "exceeds the 227 KB per-CTA shared memory limit");
  static_assert(!TMAEPI || kStages >= kEpiStages, "the staging budget above assumes a ring of kEpiStages");
};

// ---------------------------------------------------------------------------------------------- PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(smem_u32(bar))
      : "memory");
}
// TMA store of a staged (rows x 32 elements) 16-bit tile; out-of-range rows / columns are clipped by the tensor map
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, uint32_t src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%1, %2}], [%3];" ::"l"(reinterpret_cast<uint64_t>(map)),
               "r"(c0), "r"(c1), "r"(src)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// at most N of this thread's most recent bulk store groups may still be reading shared memory
template <int N>
__device__ __forceinline__ void tma_store_wait_read_n() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// read-only 8-byte load that keeps its place among the other volatile statements (issued ahead of a wgmma wait)
__device__ __forceinline__ float2 ldg_nc_f2(const float* p) {
  float2 v;
  asm volatile("ld.global.nc.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "l"(p));
  return v;
}
// named barrier over the 128 threads of one warpgroup (id 0 is __syncthreads)
__device__ __forceinline__ void wg_bar(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// wgmma m64nNk16, fp32 accumulators d[N / 2] in the standard fragment layout (register 4j + 2h + e holds row
// 16 * warp + lane / 4 + 8 h, column 8 j + 2 (lane % 4) + e).  F16: fp16 operands, else bf16 (A and B always share the
// format).  TA / TB: the A / B tile is MN-major (transposed) instead of K-major.  acc == 0 overwrites d.
template <int N>
struct Wgmma;
template <>
struct Wgmma<32> {
  template <int F16, int TA, int TB>
  static __device__ __forceinline__ void mma(float (&d)[16], uint64_t da, uint64_t db, uint32_t acc) {
#define RIQN_WGMMA(TY) \
    asm volatile( \
        "{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n" \
        "wgmma.mma_async.sync.aligned.m64n32k16.f32." TY "." TY " " \
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %19, %20;\n}\n" \
        : \
        "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), \
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]) \
        : "l"(da), "l"(db), "r"(acc), "n"(TA), "n"(TB))
    if constexpr (F16) RIQN_WGMMA("f16"); else RIQN_WGMMA("bf16");
#undef RIQN_WGMMA
  }
};

template <>
struct Wgmma<64> {
  template <int F16, int TA, int TB>
  static __device__ __forceinline__ void mma(float (&d)[32], uint64_t da, uint64_t db, uint32_t acc) {
#define RIQN_WGMMA(TY) \
    asm volatile( \
        "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n" \
        "wgmma.mma_async.sync.aligned.m64n64k16.f32." TY "." TY " " \
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n}\n" \
        : \
        "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), \
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), \
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), \
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]) \
        : "l"(da), "l"(db), "r"(acc), "n"(TA), "n"(TB))
    if constexpr (F16) RIQN_WGMMA("f16"); else RIQN_WGMMA("bf16");
#undef RIQN_WGMMA
  }
};

template <>
struct Wgmma<128> {
  template <int F16, int TA, int TB>
  static __device__ __forceinline__ void mma(float (&d)[64], uint64_t da, uint64_t db, uint32_t acc) {
#define RIQN_WGMMA(TY) \
    asm volatile( \
        "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n" \
        "wgmma.mma_async.sync.aligned.m64n128k16.f32." TY "." TY " " \
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %67, %68;\n}\n" \
        : \
        "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), \
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), \
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), \
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), \
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), \
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), \
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), \
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]) \
        : "l"(da), "l"(db), "r"(acc), "n"(TA), "n"(TB))
    if constexpr (F16) RIQN_WGMMA("f16"); else RIQN_WGMMA("bf16");
#undef RIQN_WGMMA
  }
};

template <>
struct Wgmma<256> {
  template <int F16, int TA, int TB>
  static __device__ __forceinline__ void mma(float (&d)[128], uint64_t da, uint64_t db, uint32_t acc) {
#define RIQN_WGMMA(TY) \
    asm volatile( \
        "{\n.reg .pred p;\nsetp.ne.b32 p, %130, 0;\n" \
        "wgmma.mma_async.sync.aligned.m64n256k16.f32." TY "." TY " " \
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, %131, %132;\n}\n" \
        : \
        "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), \
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), \
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), \
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), \
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), \
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), \
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), \
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), \
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), \
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), \
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), \
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), \
        "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), \
        "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), \
        "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), \
        "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127]) \
        : "l"(da), "l"(db), "r"(acc), "n"(TA), "n"(TB))
    if constexpr (F16) RIQN_WGMMA("f16"); else RIQN_WGMMA("bf16");
#undef RIQN_WGMMA
  }
};

template <int N>
__device__ __forceinline__ void wgmma_tile(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t acc, bool f16, int mn) {
  const bool ta = (mn & 1) != 0, tb = (mn & 2) != 0;   // bit 0: A MN-major, bit 1: B MN-major
  if (f16) {
    if (ta) { if (tb) Wgmma<N>::template mma<1, 1, 1>(d, da, db, acc); else Wgmma<N>::template mma<1, 1, 0>(d, da, db, acc); }
    else    { if (tb) Wgmma<N>::template mma<1, 0, 1>(d, da, db, acc); else Wgmma<N>::template mma<1, 0, 0>(d, da, db, acc); }
  } else {
    if (ta) { if (tb) Wgmma<N>::template mma<0, 1, 1>(d, da, db, acc); else Wgmma<N>::template mma<0, 1, 0>(d, da, db, acc); }
    else    { if (tb) Wgmma<N>::template mma<0, 0, 1>(d, da, db, acc); else Wgmma<N>::template mma<0, 0, 0>(d, da, db, acc); }
  }
}

// Shared-memory matrix descriptor of wgmma: start >> 4 [0,14), leading byte offset >> 4 [16,30), stride byte offset
// >> 4 [32,46), swizzle [62,64) (1 = 128-byte swizzle).
// K-major, 128-byte-swizzled operand tile: rows of 64 16-bit values (128 B), 8-row swizzle atoms SBO = 1024 B apart
// (LBO unused).
__device__ __forceinline__ uint64_t gmma_desc_k128(uint32_t saddr) {
  return (uint64_t)((saddr & 0x3FFFF) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
// MN-major, 128-byte-swizzled operand tile: k-rows of 64 MN-elements (128 B), 8-row swizzle atoms SBO = 1024 B apart
// along K, further 64-element MN slabs LBO = 8192 B apart.
__device__ __forceinline__ uint64_t gmma_desc_mn128(uint32_t saddr) {
  return (uint64_t)((saddr & 0x3FFFF) >> 4) | ((uint64_t)(8192 >> 4) << 16) | ((uint64_t)(1024 >> 4) << 32) |
         ((uint64_t)1 << 62);
}
// two floats -> packed 16-bit pair (low half = a), fp16 or bf16
__device__ __forceinline__ uint32_t pack16x2(float a, float b, bool f16) {
  if (f16) {
    const __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&h);
  }
  const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&h);
}

// The epilogue holds the accumulator with one ROW per lane (read back from the slab): storing it directly makes every store instruction
// touch 32 different lines with 16-byte pieces (~2 TB/s).  These helpers transpose a 32x32 chunk through a padded
// per-warp shared-memory tile so that each store instruction writes one full row segment (128 B fp32 / 64 B bf16).
// Tile rows are 32 words (128 B) apart and the 16-byte piece j of row r lives at piece slot j ^ (r & 7), so that both the
// deposit (a quarter-warp = 8 rows, same j) and the drain (a quarter-warp = one row, 8 pieces) are bank-conflict free.
// Each lane deposits its row with 8 STS.128; then every instruction moves FOUR rows: lane l handles piece (l & 7) of
// row (l >> 3).
constexpr int kStRow = 32;
// explicit shared-space accesses: the staging pointer comes from an integer-aligned base, which the compiler would
// otherwise treat as a generic address (LD/ST instead of LDS/STS)
__device__ __forceinline__ void sts128(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ uint4 lds128(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr) : "memory");
  return v;
}
// st: 32-bit shared address of this warp's 32 x 32-word staging tile
__device__ __forceinline__ void stage_row(uint32_t st, const uint32_t (&w)[32], int lane) {
  __syncwarp();
  const uint32_t row = st + lane * (kStRow * 4);
#pragma unroll
  for (int j = 0; j < 8; ++j) sts128(row + ((j ^ (lane & 7)) << 4), w[4 * j], w[4 * j + 1], w[4 * j + 2], w[4 * j + 3]);
  __syncwarp();
}
__device__ __forceinline__ uint4 staged_piece(uint32_t st, int r, int piece) {
  return lds128(st + r * (kStRow * 4) + ((piece ^ (r & 7)) << 4));
}
__device__ __forceinline__ void warp_store_rows_f32(uint32_t st, const uint32_t (&w)[32], int lane, float* base, long ld,
                                                    int rows_valid) {
  stage_row(st, w, lane);
  const int sub = lane >> 3, piece = lane & 7;
#pragma unroll
  for (int r0 = 0; r0 < 32; r0 += 4) {
    const int r = r0 + sub;
    if (r < rows_valid) *reinterpret_cast<uint4*>(base + (long)r * ld + piece * 4) = staged_piece(st, r, piece);
  }
}
// w[0..15] = hi pairs (cols 2k, 2k+1), w[16..31] = lo pairs: pieces 0-3 go to the hi image, 4-7 to the lo image
__device__ __forceinline__ void warp_store_rows_bf16(uint32_t st, const uint32_t (&w)[32], int lane, bf16* hi_base,
                                                     bf16* lo_base, long ld, int rows_valid) {
  stage_row(st, w, lane);
  const int sub = lane >> 3, piece = lane & 7;
  bf16* dstb = piece < 4 ? hi_base : lo_base;
  if (dstb == nullptr) return;
#pragma unroll
  for (int r0 = 0; r0 < 32; r0 += 4) {
    const int r = r0 + sub;
    if (r < rows_valid) *reinterpret_cast<uint4*>(dstb + (long)r * ld + (piece & 3) * 8) = staged_piece(st, r, piece);
  }
}

// C += alpha * acc (and out2 += alpha * acc * eps for the NoisyLinear weight gradient) on full 128-byte row segments:
// 16-byte read-modify-writes (one CTA per tile: split-K products go through per-split partials instead).
template <bool NOISY>
__device__ __forceinline__ void warp_accum_rows_f32(uint32_t st, const uint32_t (&w)[32], int lane, float* c, float* out2,
                                                    const float* eps, long ld, int rows_valid, float alpha) {
  stage_row(st, w, lane);
  const int sub = lane >> 3, piece = lane & 7;
#pragma unroll
  for (int r0 = 0; r0 < 32; r0 += 4) {
    const int r = r0 + sub;
    if (r < rows_valid) {
      const uint4 au = staged_piece(st, r, piece);
      const float4 a = make_float4(__uint_as_float(au.x) * alpha, __uint_as_float(au.y) * alpha,
                                   __uint_as_float(au.z) * alpha, __uint_as_float(au.w) * alpha);
      const long off = (long)r * ld + piece * 4;
      float4 o = *reinterpret_cast<const float4*>(c + off);
      o.x += a.x; o.y += a.y; o.z += a.z; o.w += a.w;
      *reinterpret_cast<float4*>(c + off) = o;
      if (NOISY) {
        const float4 e = *reinterpret_cast<const float4*>(eps + off);
        float4 o2 = *reinterpret_cast<const float4*>(out2 + off);
        o2.x += a.x * e.x; o2.y += a.y * e.y; o2.z += a.z * e.z; o2.w += a.w * e.w;
        *reinterpret_cast<float4*>(out2 + off) = o2;
      }
    }
  }
}

// Transposed (N, M) bf16 image of a chunk whose 16 words hold the column pairs (2k, 2k+1) of this lane's row: lane pairs
// exchange words so that each lane stores TWO consecutive rows of ONE column (even lanes column 2k, odd lanes 2k+1) --
// 32-bit stores, 64 B contiguous per column.  M must be even.
__device__ __forceinline__ void store_transposed_pairs(bf16* tb, const uint32_t* w16, int n0, int m, int M, int lane,
                                                       bool row_ok) {
  const uint32_t sel = (lane & 1) ? 0x3276u : 0x5410u;
  uint32_t* tp = reinterpret_cast<uint32_t*>(tb + (long)(n0 + (lane & 1)) * M + (m & ~1));
  const long step = M;   // 2 columns = 2*M bf16 = M words
#pragma unroll
  for (int k = 0; k < 16; ++k) {
    const uint32_t mine = w16[k];
    const uint32_t other = __shfl_xor_sync(0xffffffffu, mine, 1);
    if (row_ok) tp[(long)k * step] = __byte_perm(mine, other, sel);
  }
}

// One k-block (four k16 steps) of a single-pass product.  mn: bit 0 A MN-major, bit 1 B MN-major.
template <int TBN>
__device__ __forceinline__ void mma_kblock(float (&d)[TBN / 2], uint32_t sa, uint32_t sb, bool first, bool f16, int mn) {
#pragma unroll
  for (int k = 0; k < TBK / MMA_K; ++k) {
    const uint32_t koff_mn = k * (MMA_K / 8) * 1024;   // MN-major: 16 reduction rows = two 8-row swizzle atoms
    const uint32_t koff_k = k * MMA_K * 2;             // K-major: bytes inside the 128 B swizzle row
    const uint64_t da = (mn & 1) ? gmma_desc_mn128(sa + koff_mn) : gmma_desc_k128(sa + koff_k);
    const uint64_t db = (mn & 2) ? gmma_desc_mn128(sb + koff_mn) : gmma_desc_k128(sb + koff_k);
    wgmma_tile<TBN>(d, da, db, (!first || k > 0) ? 1u : 0u, f16, mn);
  }
}

struct alignas(64) TcArgs {
  CUtensorMap mapO[2];   // MODE bit 3: C (fp32, box 32 x 64, 128-byte swizzle) / o_hi (bf16, box 32 x 64, 64-byte swizzle);
                         // TC_EMBED: o_hi / o_lo ((M, N) 16-bit row-major, box 32 x 64, 64-byte swizzle)
  int M, N, K;
  int m_tiles, n_tiles, k_splits, kb_per_split, kb_total;
  float* C;
  long ldc;
  const float* bias;     // TC_BIAS_RELU / _NCHW / TC_EMBED
  float* out2;           // TC_NOISY_WGRAD: grad_sigma
  const float* eps;      // TC_NOISY_WGRAD: weight_epsilon (same layout as C)
  float alpha;           // TC_ATOMIC: scale applied to the accumulator
  int vec_acc;           // TC_ATOMIC / TC_NOISY_WGRAD: C (out2, eps) rows are 16-byte aligned -> vectorised accumulate
  int ohw;               // TC_BIAS_RELU_NCHW: m = b*ohw + p -> C[(b*N + n)*ohw + p]
  int ci_h, ci_w, ci_cin, ci_stride;   // TC_CONV_DGRAD: the NCHW image din
  const float* feat;     // TC_EMBED: (samples, N) conv features, row m uses feat[m / batch] (batch = rows per sample)
  int batch;
  bf16 *o_hi, *o_lo;     // TC_EMBED: bf16 hi / lo images of the result, row-major (M, N)   (may be null)
  bf16 *o_hiT, *o_loT;   // TC_BIAS_RELU: transposed (N, M) bf16 image of the result          (may be null)
  int strip_t, strip_G, strip_kc, cv_oh, cv_ow, nx_s, nx_G;   // TC_CONV (see gemm.h)
  int mn_major, wg_t, wg_G, wg_kc;                             // MN-major operands / strip weight gradient (gemm.h)
  bf16 *nx_hi, *nx_lo;
  int fmt;               // bit 0: A image is fp16, bit 1: B image is fp16 (else bf16), bit 2: o_hi is written as fp16
  int grp_mt, a_wrap;    // TC_CONV, two weight sets (gemm.h): group 1's B maps live in mapO[0] / mapO[1]
  const float* bias2;
  long part_stride;      // TC_STORE of split-K partials: split ks writes C + ks * part_stride (0 otherwise)
};

// MODE: bits 0-1 = mn_major, bit 2 = fp16 operands (both 128x256 tiles only), bit 3 = TMA-store epilogue (128x256 tiles
// and TC_EMBED; 0 otherwise)
template <int NSPLIT, int EPI, int BN, int MODE = 0>
__global__ void __launch_bounds__(kTcThreads, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap mapA_hi, const __grid_constant__ CUtensorMap mapA_lo,
               const __grid_constant__ CUtensorMap mapB_hi, const __grid_constant__ CUtensorMap mapB_lo,
               const __grid_constant__ TcArgs p) {
  constexpr bool kTmaEpi = (MODE & 8) != 0;
  using Cfg = TcCfg<NSPLIT, BN, EPI, kTmaEpi>;
  constexpr int TBN = BN;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  // layout: operand ring | accumulator slabs or staging buffers (per consumer warpgroup, 1 KB aligned) | barriers
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::kStages * Cfg::kStageBytes + Cfg::kEpiBytes);
  uint64_t* full = bars;                       // [kStages]  TMA -> MMA
  uint64_t* empty = bars + Cfg::kStages;       // [kStages]  MMA -> TMA (one arrival per consumer warp)
  const uint32_t epi_base = (uint32_t)__cvta_generic_to_shared(smem + Cfg::kStages * Cfg::kStageBytes);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int total_units = p.m_tiles * p.n_tiles * p.k_splits;

  if (threadIdx.x == 0) {
    // descriptor fetch overlaps the barrier prologue instead of delaying the first TMA load
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&mapA_hi)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&mapB_hi)) : "memory");
    if (NSPLIT == 3) asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&mapA_lo)) : "memory");
    if (NSPLIT >= 2) asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&mapB_lo)) : "memory");
    for (int i = 0; i < Cfg::kStages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], kEpiWarps); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < 4) {
    // ------------------------------------------------------------------ TMA producer (one thread)
    // 128x256 tiles: the producer warpgroup hands its registers to the consumers' 128 accumulators per thread
    // (128 * 40 + 256 * 232 = the 64512 registers the launch gets at 168 per thread).  The embedding's consumers hold a
    // tile's feat / bias values (96 registers) beside their 64 accumulators.
    if constexpr (BN == 256 || EPI == TC_EMBED) asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
    if (warp == 0 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int u = blockIdx.x; u < total_units; u += gridDim.x) {
        // split-K units are k-split MAJOR: the CTAs in flight walk the SAME reduction range of all output tiles, so each
        // operand slab is fetched from HBM once and shared through L2 (tile-major order read 2.7x the algorithmic bytes)
        const int tiles = p.m_tiles * p.n_tiles;
        const int ks = u / tiles, t = u - ks * tiles;
        const int nt = t % p.n_tiles, mt = t / p.n_tiles;   // n fastest: the A tile is shared by the n-tiles in flight
        const int kb0 = ks * p.kb_per_split, kb1 = min(p.kb_total, kb0 + p.kb_per_split);
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1);
          uint8_t* s = smem + stage * Cfg::kStageBytes;
          mbar_expect_tx(&full[stage], Cfg::kStageBytes);
          if constexpr (EPI == TC_CONV_DGRAD) {
            // shift (dy, dx): dYg rows m0 - (dy*G + dx) (negative ones arrive as zeros), and that shift's (K, N) weight slab
            const int dy = kb / p.strip_t, dx = kb - dy * p.strip_t;
            tma_load_2d(s, &mapA_hi, 0, mt * TBM - (dy * p.strip_G + dx), &full[stage]);
#pragma unroll
            for (int i = 0; i < TBN / 64; ++i)
              tma_load_2d(s + Cfg::kABytes + i * 8192, &mapB_hi, kb * p.N + nt * TBN + 64 * i, 0, &full[stage]);
            if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
            continue;
          }
          if (NSPLIT == 1 && p.mn_major) {
            // MN-major operand ((K, MN) row-major): 64 x 64 boxes, inner coordinate = MN offset, outer = reduction row.
            // bit 0: A, bit 1: B; the other operand (if any) stays K-major.
            const int kk = kb * TBK;
            if (p.mn_major & 1) {
#pragma unroll
              for (int i = 0; i < TBM / 64; ++i) tma_load_2d(s + i * 8192, &mapA_hi, mt * TBM + 64 * i, kk, &full[stage]);
            } else {
              tma_load_2d(s, &mapA_hi, kk, mt * TBM, &full[stage]);
            }
            if (p.mn_major & 2) {
#pragma unroll
              for (int i = 0; i < (TBN >= 64 ? TBN / 64 : 1); ++i) {
                int b_in = nt * TBN + 64 * i, b_row = kk;
                if (p.wg_t) {                        // strip weight gradient: this 64-column slab has its own row shift
                  const int slab = b_in >> 6, sft = slab / p.wg_kc, dy = sft / p.wg_t;
                  b_in = (slab - sft * p.wg_kc) << 6;
                  b_row += dy * p.wg_G + (sft - dy * p.wg_t);
                }
                tma_load_2d(s + Cfg::kOps * Cfg::kABytes + i * 8192, &mapB_hi, b_in, b_row, &full[stage]);
              }
            } else {
              tma_load_2d(s + Cfg::kOps * Cfg::kABytes, &mapB_hi, kk, nt * TBN, &full[stage]);
            }
            if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
            continue;
          }
          int a_col = kb * TBK, a_row = mt * TBM;
          const CUtensorMap *mb_hi = &mapB_hi, *mb_lo = &mapB_lo;
          if (EPI == TC_CONV && p.grp_mt && mt >= p.grp_mt) {   // second weight set (and, for a shared A image, its rows again)
            mb_hi = &p.mapO[0];
            mb_lo = &p.mapO[1];
            if (p.a_wrap) a_row = (mt - p.grp_mt) * TBM;
          }
          if (EPI == TC_CONV) {     // strip convolution: shifted rows of the space-to-depth image
            const int sft = kb / p.strip_kc, dy = sft / p.strip_t;
            a_col = (kb - sft * p.strip_kc) * TBK;
            a_row += dy * p.strip_G + (sft - dy * p.strip_t);
          }
          tma_load_2d(s, &mapA_hi, a_col, a_row, &full[stage]);
          tma_load_2d(s + Cfg::kOps * Cfg::kABytes, mb_hi, kb * TBK, nt * TBN, &full[stage]);
          if (NSPLIT == 3) tma_load_2d(s + Cfg::kABytes, &mapA_lo, a_col, a_row, &full[stage]);
          if (NSPLIT >= 2)
            tma_load_2d(s + Cfg::kAOps * Cfg::kABytes + Cfg::kBBytes, mb_lo, kb * TBK, nt * TBN, &full[stage]);
          if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumer warpgroups (wgmma + epilogue)
  if constexpr (BN == 256 || EPI == TC_EMBED) asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
  const int g = (warp >> 2) - 1;               // this warpgroup's 64 tile rows start at 64 g
  const int wq = warp & 3;                      // warp in the warpgroup: fragment rows [16 wq, +16)
  const int band = wq & 1, colhalf = wq >> 1;   // epilogue: 32-row band of the slab, 32-column half of each 64-column chunk
  const int quarter = 2 * g + band;             // the tile rows [32 quarter, +32) this warp's lanes hold in the epilogue
  const uint32_t slab = epi_base + g * kSlabBytes;
  const uint32_t st = slab + wq * (32 * kStRow * 4);   // this warp's staging tile (overlays the slab once it is read)
  const bool f16 = (p.fmt & 3) != 0;
  float conv_bias[32];
  if (EPI == TC_CONV) {                         // one n-tile (N <= 64): this warp's 32 columns never change
#pragma unroll
    for (int j = 0; j < 32; ++j) conv_bias[j] = (32 * colhalf + j < p.N && 32 * colhalf < TBN) ? p.bias[32 * colhalf + j] : 0.f;
  }
  bool conv_grp1 = false;
  int stage = 0;
  uint32_t phase = 0;
  int epi_seq = 0;                              // TMA-store epilogue: chunks this warpgroup has staged so far
  for (int u = blockIdx.x; u < total_units; u += gridDim.x) {
    const int tiles = p.m_tiles * p.n_tiles;
    const int ks = u / tiles, t = u - ks * tiles;
    const int nt = t % p.n_tiles, mt = t / p.n_tiles;
    const int kb0 = ks * p.kb_per_split, kb1 = min(p.kb_total, kb0 + p.kb_per_split);
    if (EPI == TC_CONV && p.grp_mt && (mt >= p.grp_mt) != conv_grp1) {   // a CTA's tiles ascend: this happens at most once
      conv_grp1 = mt >= p.grp_mt;
      const float* bsrc = conv_grp1 ? p.bias2 : p.bias;
#pragma unroll
      for (int j = 0; j < 32; ++j) conv_bias[j] = (32 * colhalf + j < p.N && 32 * colhalf < TBN) ? bsrc[32 * colhalf + j] : 0.f;
    }
    // ---- mainloop: the wgmma groups of one k-block stay in flight while the next k-block's operands are awaited; a
    // ring slot is released once the groups that read it have retired
    float acc[TBN / 2];
    float dg_sum[TBN / 2];                      // TC_CONV_DGRAD: the sum over the shifts so far
    if constexpr (EPI == TC_CONV_DGRAD) {
#pragma unroll
      for (int i = 0; i < TBN / 2; ++i) dg_sum[i] = 0.f;
    }
    // TC_EMBED: bias and feat of this thread's fragment (column pairs 8 j + 2 (lane % 4) + {0, 1} of rows fr, fr + 8),
    // loaded here so that their L2 latency passes under the product.  The two rows may belong to different samples
    // (fewer than 64 rows per sample); rows >= M and columns >= N are only loaded from a valid place, never stored.
    float2 e_bias[TBN / 8], e_feat[2][TBN / 8];
    if constexpr (EPI == TC_EMBED) {
      const int m0 = mt * TBM + 64 * g + 16 * wq + (lane >> 2), m1 = m0 + 8;
      const float* f0 = p.feat + (long)((m0 < p.M ? m0 : 0) / p.batch) * p.N;
      const float* f1 = p.feat + (long)((m1 < p.M ? m1 : 0) / p.batch) * p.N;
#pragma unroll
      for (int j = 0; j < TBN / 8; ++j) {
        int n = nt * TBN + 8 * j + 2 * (lane & 3);
        if (n >= p.N) n = 0;
        e_bias[j] = ldg_nc_f2(p.bias + n);
        e_feat[0][j] = ldg_nc_f2(f0 + n);
        e_feat[1][j] = ldg_nc_f2(f1 + n);
      }
    }
    int prev = -1;
    for (int kb = kb0; kb < kb1; ++kb) {
      mbar_wait(&full[stage], phase);
      const uint32_t s0 = smem_u32(smem + stage * Cfg::kStageBytes);
      const uint32_t sa = s0 + g * 8192;        // this warpgroup's 64 rows (K-major) or 64-row MN slab (MN-major) of A
      const uint32_t sb = s0 + Cfg::kOps * Cfg::kABytes;
      wgmma_fence();
      if constexpr (EPI == TC_CONV_DGRAD) {
        mma_kblock<TBN>(acc, sa, sb, true, false, 2);   // every shift starts from a zeroed accumulator
      } else if constexpr (BN == 256) {
        // operand modes fixed at compile time: run-time choices between wgmma variants make ptxas serialise them.  For
        // the same reason the edge tile (N = 3136: 64 real columns in the last one) runs full-width on TMA's zero fill.
        mma_kblock<TBN>(acc, sa, sb, kb == kb0, (MODE & 4) != 0, MODE & 3);
      } else if (NSPLIT == 1 && p.mn_major) {
#pragma unroll
        for (int k = 0; k < TBK / MMA_K; ++k) {
          const uint32_t koff_mn = k * (MMA_K / 8) * 1024;   // MN-major: 16 reduction rows = two 8-row swizzle atoms
          const uint32_t koff_k = k * MMA_K * 2;             // K-major: bytes inside the 128 B swizzle row
          const uint64_t da = (p.mn_major & 1) ? gmma_desc_mn128(sa + koff_mn) : gmma_desc_k128(sa + koff_k);
          const uint64_t db = (p.mn_major & 2) ? gmma_desc_mn128(sb + koff_mn) : gmma_desc_k128(sb + koff_k);
          wgmma_tile<TBN>(acc, da, db, (kb > kb0 || k > 0) ? 1u : 0u, f16, p.mn_major);
        }
      } else {
#pragma unroll
        for (int k = 0; k < TBK / MMA_K; ++k) {
          const uint32_t koff = k * MMA_K * 2;   // bytes along K inside the 128 B swizzle row
          const uint64_t a_hi = gmma_desc_k128(sa + koff), b_hi = gmma_desc_k128(sb + koff);
          wgmma_tile<TBN>(acc, a_hi, b_hi, (kb > kb0 || k > 0) ? 1u : 0u, f16, 0);
          if (NSPLIT >= 2) wgmma_tile<TBN>(acc, a_hi, gmma_desc_k128(sb + Cfg::kBBytes + koff), 1u, false, 0);
          if (NSPLIT == 3) wgmma_tile<TBN>(acc, gmma_desc_k128(sa + Cfg::kABytes + koff), b_hi, 1u, false, 0);
        }
      }
      wgmma_commit();
      wgmma_wait<1>();                          // the previous k-block's groups have retired: its slot is free
      if (prev >= 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[prev]);
      }
      prev = stage;
      if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
      if constexpr (EPI == TC_CONV_DGRAD) {
        wgmma_wait<0>();
#pragma unroll
        for (int i = 0; i < TBN / 2; ++i) dg_sum[i] += acc[i];
      }
    }
    wgmma_wait<0>();
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[prev]);
    if constexpr (EPI == TC_CONV_DGRAD) {
#pragma unroll
      for (int i = 0; i < TBN / 2; ++i) acc[i] = dg_sum[i];
    }

    if constexpr (kTmaEpi) {
      // ---- TMA-store epilogue: the fragments go straight into the swizzled staging boxes (bias + ReLU, or the
      // embedding's x = feat * relu(acc + bias) (model.py:146-151) and its two 16-bit images, applied in registers),
      // one thread per warpgroup issues the bulk tensor stores, and the warpgroup goes on to the next tile
      // without waiting for them.  A staging buffer is rewritten only after the stores that read it have finished
      // READING shared memory; their global writes stay in flight.  TMA clips rows >= M and columns >= N.
      constexpr int kChunks = TBN / 32;
      constexpr bool kWhole = Cfg::kEpiBufs == kChunks;   // one buffer per chunk of the tile: one wait and two barriers per tile
      const int row0 = mt * TBM + 64 * g;
      const int nch = min(kChunks, (p.N - nt * TBN + 31) / 32);   // chunks holding real columns
      const bool elected = wq == 0 && lane == 0;
      const uint32_t stg = epi_base + g * (Cfg::kEpiBufs * Cfg::kEpiChunkBytes);
      const int fr = 16 * wq + (lane >> 2);     // fragment rows fr and fr + 8 of this warpgroup's 64
      if (row0 < p.M) {
#pragma unroll
        for (int h = 0; h < kChunks; ++h) {
          if (h >= nch) break;
          const int buf = kWhole ? h : epi_seq % Cfg::kEpiBufs;
          if (!kWhole || h == 0) {
            if (elected) tma_store_wait_read_n<kWhole ? 0 : Cfg::kEpiBufs - 1>();
            wg_bar(1 + g);
          }
          const uint32_t sf = stg + buf * Cfg::kEpiChunkBytes;   // fp32 box (64 rows x 128 B)
          const uint32_t sh = sf + Cfg::kEpiF32Bytes;            // bf16 box (64 rows x 64 B)
#pragma unroll
          for (int jj = 0; jj < 4; ++jj) {
            const int j = 4 * h + jj;               // accumulator column group: tile columns 8 j + 2 (lane % 4) + {0, 1}
            if constexpr (EPI == TC_EMBED) {
              const bool x_f16 = (p.fmt & 4) != 0;
#pragma unroll
              for (int hh = 0; hh < 2; ++hh) {
                const int r = fr + 8 * hh;
                const float x0 = e_feat[hh][j].x * fmaxf(acc[4 * j + 2 * hh] + e_bias[j].x, 0.f);
                const float x1 = e_feat[hh][j].y * fmaxf(acc[4 * j + 2 * hh + 1] + e_bias[j].y, 0.f);
                if (p.C != nullptr && row0 + r < p.M)   // fp32 x of the cross-check arithmetic modes
                  *reinterpret_cast<float2*>(p.C + (long)(row0 + r) * p.N + nt * TBN + 8 * j + 2 * (lane & 3)) = make_float2(x0, x1);
                // fp16(x) feeds the single-pass head forward and bf16(x) the backward products; otherwise bf16 hi + the
                // residual lo of the split-bf16 x3 head forward
                const uint32_t w0 = pack16x2(x0, x1, x_f16);
                const uint32_t w1 = x_f16 ? pack16x2(x0, x1, false)
                                          : pack16x2(x0 - __uint_as_float(w0 << 16), x1 - __uint_as_float(w0 & 0xffff0000u), false);
                const uint32_t so = sh + r * 64 + ((jj ^ ((r >> 1) & 3)) << 4) + 4 * (lane & 3);   // 64-byte swizzle, as below
                if (p.o_hi != nullptr) asm volatile("st.shared.b32 [%0], %1;" ::"r"(so), "r"(w0) : "memory");
                if (p.o_lo != nullptr) asm volatile("st.shared.b32 [%0], %1;" ::"r"(so + 64 * 32 * 2), "r"(w1) : "memory");
              }
              continue;
            }
            float b0 = 0.f, b1 = 0.f;
            if (EPI == TC_BIAS_RELU) {
              const int n = nt * TBN + 8 * j + 2 * (lane & 3);
              if (n < p.N) b0 = __ldg(p.bias + n);
              if (n + 1 < p.N) b1 = __ldg(p.bias + n + 1);
            }
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
              const int r = fr + 8 * hh;
              float x0 = acc[4 * j + 2 * hh], x1 = acc[4 * j + 2 * hh + 1];
              if (EPI == TC_BIAS_RELU) {
                x0 = fmaxf(x0 + b0, 0.f);
                x1 = fmaxf(x1 + b1, 0.f);
                // 128-byte swizzle: 16-byte piece q of row r sits at q ^ (r % 8)
                const uint32_t q = 2 * jj + ((lane & 3) >> 1);
                asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(sf + r * 128 + ((q ^ (r & 7)) << 4) + 8 * (lane & 1)),
                             "f"(x0), "f"(x1) : "memory");
              }
              if (EPI == TC_STORE || p.o_hi != nullptr) {
                // 64-byte swizzle: 16-byte piece q of row r sits at q ^ ((r / 2) % 4)
                const __nv_bfloat162 hv = __floats2bfloat162_rn(x0, x1);
                asm volatile("st.shared.b32 [%0], %1;" ::"r"(sh + r * 64 + ((jj ^ ((r >> 1) & 3)) << 4) + 4 * (lane & 3)),
                             "r"(*reinterpret_cast<const uint32_t*>(&hv)) : "memory");
              }
            }
          }
          fence_proxy_async();                      // generic-proxy writes -> visible to the TMA engine
          if (!kWhole || h == nch - 1) {
            wg_bar(1 + g);
            if (elected) {
#pragma unroll
              for (int i = kWhole ? 0 : h; i <= h; ++i) {
                const uint32_t si = kWhole ? stg + i * Cfg::kEpiChunkBytes : sf;
                const int c0 = nt * TBN + 32 * i;
                if (EPI == TC_EMBED) {
                  if (p.o_hi != nullptr) tma_store_2d(&p.mapO[0], si, c0, row0);
                  if (p.o_lo != nullptr) tma_store_2d(&p.mapO[1], si + 64 * 32 * 2, c0, row0);
                  continue;
                }
                if (EPI == TC_BIAS_RELU) tma_store_2d(&p.mapO[0], si, c0, row0);
                if (EPI == TC_STORE || p.o_hi != nullptr) tma_store_2d(&p.mapO[1], si + Cfg::kEpiF32Bytes, c0, row0);
              }
              tma_store_commit();
            }
          }
          ++epi_seq;
        }
      }
      continue;
    }

    // ---- epilogue, one 64-column chunk at a time: fragment -> slab -> (row per lane) v[32] -> fused epilogue
#pragma unroll
    for (int h = 0; h < (TBN + 63) / 64; ++h) {
      if (BN == 256 && nt * TBN + 64 * h >= p.N) break;         // edge tile: the remaining chunks hold no real column
      wg_bar(1 + g);
      {
        const uint32_t r0 = slab + ((16 * wq + (lane >> 2)) * kSlabStride + 2 * (lane & 3)) * 4;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int jj = 8 * h + j;
          if (jj * 8 < TBN) {
            asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(r0 + j * 32), "f"(acc[4 * jj]), "f"(acc[4 * jj + 1]) : "memory");
            asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(r0 + 8 * kSlabStride * 4 + j * 32), "f"(acc[4 * jj + 2]),
                         "f"(acc[4 * jj + 3]) : "memory");
          }
        }
      }
      wg_bar(1 + g);
      const int c = 64 * h + 32 * colhalf;
      uint32_t v[32];
      if (c < TBN) {
        const uint32_t rr = slab + ((32 * band + lane) * kSlabStride + 32 * colhalf) * 4;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const uint4 x = lds128(rr + 16 * j);
          v[4 * j] = x.x; v[4 * j + 1] = x.y; v[4 * j + 2] = x.z; v[4 * j + 3] = x.w;
        }
      }
      wg_bar(1 + g);                            // the slab is read: from here on it holds the per-warp staging tiles
      if (c >= TBN) continue;
      const int m = mt * TBM + quarter * 32 + lane;
      const int n0 = nt * TBN + c;
      if (m < p.M && n0 < p.N) {
        if (EPI == TC_STORE || EPI == TC_BIAS_RELU) {
          float* crow = p.C + ks * p.part_stride + (long)m * p.ldc + n0;
          if (n0 + 32 <= p.N && (EPI == TC_STORE || (p.M & 1) == 0)) {
            // handled below with the whole warp (coalesced row stores)
          } else if (n0 + 32 <= p.N) {
#pragma unroll
            for (int j = 0; j < 32; j += 4) {
              float4 o = make_float4(__uint_as_float(v[j]), __uint_as_float(v[j + 1]), __uint_as_float(v[j + 2]),
                                     __uint_as_float(v[j + 3]));
              if (EPI == TC_BIAS_RELU) {
                const float4 b = *reinterpret_cast<const float4*>(p.bias + n0 + j);
                o.x = fmaxf(o.x + b.x, 0.f); o.y = fmaxf(o.y + b.y, 0.f);
                o.z = fmaxf(o.z + b.z, 0.f); o.w = fmaxf(o.w + b.w, 0.f);
              }
              *reinterpret_cast<float4*>(crow + j) = o;
              if (EPI == TC_BIAS_RELU && p.o_hiT) {   // bf16 (N, M) image: lanes = consecutive m -> coalesced
                p.o_hiT[(long)(n0 + j) * p.M + m] = __float2bfloat16_rn(o.x);
                p.o_hiT[(long)(n0 + j + 1) * p.M + m] = __float2bfloat16_rn(o.y);
                p.o_hiT[(long)(n0 + j + 2) * p.M + m] = __float2bfloat16_rn(o.z);
                p.o_hiT[(long)(n0 + j + 3) * p.M + m] = __float2bfloat16_rn(o.w);
              }
            }
          } else {
#pragma unroll
            for (int j = 0; j < 32; ++j) {
              if (n0 + j < p.N) {
                float o = __uint_as_float(v[j]);
                if (EPI == TC_BIAS_RELU) o = fmaxf(o + p.bias[n0 + j], 0.f);
                crow[j] = o;
                if (EPI == TC_BIAS_RELU && p.o_hiT) p.o_hiT[(long)(n0 + j) * p.M + m] = __float2bfloat16_rn(o);
              }
            }
          }
        } else if (EPI == TC_BIAS_RELU_NCHW) {
          const int b = m / p.ohw, pp = m - b * p.ohw;
          float* cb = p.C + ((long)b * p.N + n0) * p.ohw + pp;   // lanes = consecutive pp: coalesced per n
#pragma unroll
          for (int j = 0; j < 32; ++j)
            if (n0 + j < p.N) cb[(long)j * p.ohw] = fmaxf(__uint_as_float(v[j]) + p.bias[n0 + j], 0.f);
        } else if (EPI == TC_CONV || EPI == TC_CONV_DGRAD) {
          // handled below with the whole warp
        } else if (!(p.vec_acc && n0 + 32 <= p.N)) {
          float* crow = p.C + (long)m * p.ldc + n0;
#pragma unroll
          for (int j = 0; j < 32; ++j) {
            if (n0 + j < p.N) {
              const float o = __uint_as_float(v[j]) * (EPI == TC_ATOMIC ? p.alpha : 1.f);
              crow[j] += o;              // the only writer of these rows (split-K: per-split partials)
              if (EPI == TC_NOISY_WGRAD) p.out2[(long)m * p.ldc + n0 + j] += o * p.eps[(long)m * p.ldc + n0 + j];
            }
          }
        }
      }
      if (EPI == TC_CONV && n0 < p.N) {
        // strip convolution: relu(acc + bias) -> (optional) fp32 NCHW output + the NEXT layer's space-to-depth images.
        // The bias of this warp's 32 columns sits in registers for the whole kernel (N <= 64 = one n-tile); the image
        // rows go through the staging transpose so that a quarter-warp writes one pixel's 64-byte channel run.
        const int gg = p.strip_G * p.strip_G;
        const int mm = m < p.M ? m : 0;
        const int b = mm / gg, rem = mm - b * gg;
        const int gy = rem / p.strip_G, gx = rem - gy * p.strip_G;
        const bool valid = m < p.M && gy < p.cv_oh && gx < p.cv_ow;
        float x[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) x[j] = n0 + j < p.N ? fmaxf(__uint_as_float(v[j]) + conv_bias[j], 0.f) : 0.f;
        if (p.C != nullptr && valid) {
          const int plane = p.cv_oh * p.cv_ow;
          float* cb = p.C + ((long)b * p.N + n0) * plane + gy * p.cv_ow + gx;     // lanes = consecutive gx
#pragma unroll
          for (int j = 0; j < 32; ++j)
            if (n0 + j < p.N) cb[(long)j * plane] = x[j];
        }
        if (p.nx_hi != nullptr && n0 + 32 <= p.N) {          // warp-uniform
          // this pixel's channels are contiguous in the next layer's space-to-depth row
          long o = -1;
          if (valid) {
            const int sn = p.nx_s, by = gy / sn, bx = gx / sn;
            const long r = ((long)b * p.nx_G + by) * p.nx_G + bx;
            o = r * ((long)sn * sn * p.N) + (long)((gy - by * sn) * sn + (gx - bx * sn)) * p.N + n0;
          }
          uint32_t hw[32];      // [0..15] hi pairs, [16..31] lo pairs
#pragma unroll
          for (int j = 0; j < 32; j += 2) {
            const uint32_t hwj = pack16x2(x[j], x[j + 1], false);
            hw[j / 2] = hwj;
            hw[16 + j / 2] = pack16x2(x[j] - __uint_as_float(hwj << 16), x[j + 1] - __uint_as_float(hwj & 0xffff0000u), false);
          }
          stage_row(st, hw, lane);
          const int sub = lane >> 3, piece = lane & 7;
          bf16* dstb = piece < 4 ? p.nx_hi : p.nx_lo;
          uint4 pc[8];                      // all pieces in flight before the first store (one shared-memory latency)
          long orow[8];
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            pc[i] = staged_piece(st, 4 * i + sub, piece);
            orow[i] = __shfl_sync(0xffffffffu, o, 4 * i + sub);
          }
#pragma unroll
          for (int i = 0; i < 8; ++i)
            if (orow[i] >= 0 && dstb != nullptr) *reinterpret_cast<uint4*>(dstb + orow[i] + (piece & 3) * 8) = pc[i];
        }
      }
      if (EPI == TC_CONV_DGRAD && n0 < p.N) {
        // din[b, c, gy*s + iy, gx*s + ix] = sum[(b, gy, gx), (iy, ix, c)]: lane j decodes column n0 + j once and the
        // offsets are broadcast by shuffle; lanes = consecutive gx, so a store instruction covers a few image row runs
        const int kcol = n0 + lane, s = p.ci_stride;
        int coff = -1;
        if (kcol < p.N) {
          const int blk = kcol / p.ci_cin, c = kcol - blk * p.ci_cin, iy = blk / s, ix = blk - iy * s;
          coff = (c * p.ci_h + iy) * p.ci_w + ix;
        }
        const bool row_ok = m < p.M;
        const int gg = p.strip_G * p.strip_G, mm = row_ok ? m : 0;
        const int b = mm / gg, rem = mm - b * gg, gy = rem / p.strip_G, gx = rem - gy * p.strip_G;
        float* base = p.C + ((long)b * p.ci_cin * p.ci_h + gy * s) * p.ci_w + gx * s;
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          const int off = __shfl_sync(0xffffffffu, coff, j);
          if (row_ok && off >= 0) base[off] = __uint_as_float(v[j]);
        }
      }
      if ((EPI == TC_STORE || (EPI == TC_BIAS_RELU && (p.M & 1) == 0) ||
           ((EPI == TC_ATOMIC || EPI == TC_NOISY_WGRAD) && p.vec_acc)) && n0 + 32 <= p.N) {
        const int m_base = mt * TBM + quarter * 32;
        const int rows_valid = min(32, p.M - m_base);            // warp-uniform
        if (rows_valid > 0) {
          if (EPI == TC_STORE) {
            if (p.o_hi != nullptr) {                           // bf16 result (M, N) instead of fp32: 64-byte row pieces
              uint32_t hw2[32];
#pragma unroll
              for (int j = 0; j < 16; ++j) {
                const __nv_bfloat162 h2 = __floats2bfloat162_rn(__uint_as_float(v[2 * j]), __uint_as_float(v[2 * j + 1]));
                hw2[j] = *reinterpret_cast<const uint32_t*>(&h2);
                hw2[16 + j] = 0u;
              }
              warp_store_rows_bf16(st, hw2, lane, p.o_hi + (long)m_base * p.N + n0, nullptr, p.N, rows_valid);
            } else {
              warp_store_rows_f32(st, v, lane, p.C + ks * p.part_stride + (long)m_base * p.ldc + n0, p.ldc, rows_valid);
            }
          } else if (EPI == TC_ATOMIC) {
            warp_accum_rows_f32<false>(st, v, lane, p.C + (long)m_base * p.ldc + n0, nullptr, nullptr, p.ldc, rows_valid,
                                       p.alpha);
          } else if (EPI == TC_NOISY_WGRAD) {
            const long o0 = (long)m_base * p.ldc + n0;
            warp_accum_rows_f32<true>(st, v, lane, p.C + o0, p.out2 + o0, p.eps + o0, p.ldc, rows_valid, 1.f);
          } else if (EPI == TC_BIAS_RELU) {
            const float* br = p.bias + n0;
            uint32_t hw[16];
#pragma unroll
            for (int j = 0; j < 32; j += 4) {
              const float4 bb = __ldg(reinterpret_cast<const float4*>(br + j));
              const float x0 = fmaxf(__uint_as_float(v[j]) + bb.x, 0.f), x1 = fmaxf(__uint_as_float(v[j + 1]) + bb.y, 0.f);
              const float x2 = fmaxf(__uint_as_float(v[j + 2]) + bb.z, 0.f), x3 = fmaxf(__uint_as_float(v[j + 3]) + bb.w, 0.f);
              const __nv_bfloat162 h01 = __floats2bfloat162_rn(x0, x1), h23 = __floats2bfloat162_rn(x2, x3);
              hw[j / 2] = *reinterpret_cast<const uint32_t*>(&h01);
              hw[j / 2 + 1] = *reinterpret_cast<const uint32_t*>(&h23);
              v[j] = __float_as_uint(x0); v[j + 1] = __float_as_uint(x1);
              v[j + 2] = __float_as_uint(x2); v[j + 3] = __float_as_uint(x3);
            }
            if (p.o_hiT) store_transposed_pairs(p.o_hiT, hw, n0, m, p.M, lane, m < p.M);
            warp_store_rows_f32(st, v, lane, p.C + ks * p.part_stride + (long)m_base * p.ldc + n0, p.ldc, rows_valid);
            if (p.o_hi) {                                     // bf16 row-major image (M, N): 64-byte row pieces
              uint32_t hw2[32];
#pragma unroll
              for (int j = 0; j < 16; ++j) { hw2[j] = hw[j]; hw2[16 + j] = 0u; }
              warp_store_rows_bf16(st, hw2, lane, p.o_hi + (long)m_base * p.N + n0, nullptr, p.N, rows_valid);
            }
          }
        }
      }
    }
  }
  if (kTmaEpi && lane == 0) tma_store_wait_all();   // bulk stores read this CTA's shared memory
}

// ---------------------------------------------------------------------------------------------- host side
static PFN_cuTensorMapEncodeTiled_v12000 get_encode() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
  });
  return fn;
}

// (rows, K) row-major bf16 matrix, box = box_rows x 64 elements, 128-byte swizzle.  Out-of-bounds -> zeros.
static int make_map(CUtensorMap* map, const bf16* base, long rows, long K, int box_rows) {
  auto enc = get_encode();
  if (!enc) return (int)cudaErrorNotSupported;
  cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)(K * sizeof(bf16))};
  cuuint32_t box[2] = {(cuuint32_t)TBK, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<bf16*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : (int)cudaErrorInvalidValue;
}

// (rows, cols) row-major 16-bit matrix written by TMA stores of 32 x box_rows boxes staged in the 64-byte-swizzle layout
static int make_store_map(CUtensorMap* map, const bf16* base, long rows, long cols, int box_rows = 32) {
  auto enc = get_encode();
  if (!enc) return (int)cudaErrorNotSupported;
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)(cols * sizeof(bf16))};
  cuuint32_t box[2] = {32, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<bf16*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : (int)cudaErrorInvalidValue;
}
// (rows, cols) fp32 matrix with row pitch ld, written by TMA stores of 32 x 64 boxes staged in the 128-byte-swizzle layout
static int make_store_map_f32(CUtensorMap* map, const float* base, long rows, long cols, long ld) {
  auto enc = get_encode();
  if (!enc) return (int)cudaErrorNotSupported;
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)(ld * sizeof(float))};
  cuuint32_t box[2] = {32, 64};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : (int)cudaErrorInvalidValue;
}

template <int NSPLIT, int EPI, int BN, int MODE = 0>
static int launch_tc(const CUtensorMap& a_hi, const CUtensorMap& a_lo, const CUtensorMap& b_hi, const CUtensorMap& b_lo,
                     const TcArgs& p, cudaStream_t s) {
  using Cfg = TcCfg<NSPLIT, BN, EPI, (MODE & 8) != 0>;
  static PerDeviceOnce attr_once;
  const int attr_dev = PerDeviceOnce::device();
  if (!attr_once.done[attr_dev]) {
    RIQN_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<NSPLIT, EPI, BN, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   (int)Cfg::kSmemBytes));
    attr_once.done[attr_dev] = true;
  }
  int sms = attr_once.sms[attr_dev];
  if (!sms) {
    RIQN_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, attr_dev));
    attr_once.sms[attr_dev] = sms;
  }
  const int units = p.m_tiles * p.n_tiles * p.k_splits;
  const int grid = units < sms ? units : sms;
  gemm_tc_kernel<NSPLIT, EPI, BN, MODE><<<grid, kTcThreads, Cfg::kSmemBytes, s>>>(a_hi, a_lo, b_hi, b_lo, p);
  return (int)cudaGetLastError();
}

// C[m, n] += alpha * sum_k part[k][m, n] (k ascending); out2[m, n] += (sum_k part[k][m, n]) * eps[m, n] when out2 is set
__global__ void split_k_reduce_kernel(int M, int N, int splits, long stride, long ldp, const float* __restrict__ part,
                                      float* __restrict__ C, long ldc, float alpha, float* __restrict__ out2,
                                      const float* __restrict__ eps) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long)M * N) return;
  const long m = i / N, n = i - m * N;
  float acc = 0.f;
  for (int k = 0; k < splits; ++k) acc += part[k * stride + m * ldp + n];
  C[m * ldc + n] += alpha * acc;
  if (out2 != nullptr) out2[m * ldc + n] += acc * eps[m * ldc + n];
}

// C (+)= A * B^T on the tensor cores.  A (M,K), B (N,K) bf16 row-major (K % 8 == 0); *_lo may be null (NSPLIT 1).
int gemm_bf16_tc(int M, int N, int K, const bf16* A_hi, const bf16* A_lo, const bf16* B_hi, const bf16* B_lo, float* C,
                 long ldc, int epi, const float* bias, float* out2, const float* eps, int split_k, cudaStream_t s,
                 const TcExtra* ex) {
  if (M <= 0 || N <= 0 || K <= 0) return 0;
  if ((K % 8) && !(ex != nullptr && ex->mn_major == 3)) return (int)cudaErrorInvalidValue;   // both MN-major: K counts rows
  const bool split3 = A_lo != nullptr && B_lo != nullptr;
  const bool split2 = A_lo == nullptr && B_lo != nullptr;
  // narrow outputs (conv channels, embedding width) get narrow tiles; only the epilogues that occur with them exist
  const bool narrow_ok = epi == TC_BIAS_RELU_NCHW || epi == TC_CONV || ((epi == TC_ATOMIC || epi == TC_STORE) && !split3 && !split2);
  const bool strip = epi == TC_CONV;
  if (strip && (ex == nullptr || ex->strip_t < 1 || ex->strip_kc < 1 || ex->strip_G < 1 || N > 64 ||
                K != ex->strip_t * ex->strip_t * ex->strip_kc * TBK || (ex->nx_hi && (N % 32))))
    return (int)cudaErrorInvalidValue;
  const long a_k = strip ? (long)ex->strip_kc * TBK : K;       // row length of the A image
  const bool dgrad = epi == TC_CONV_DGRAD;
  if (dgrad && (ex == nullptr || split3 || split2 || ex->mn_major || ex->strip_t < 1 || ex->strip_G < 1 || K > TBK ||
                N % 64 || split_k > 1 || ex->ci_cin < 1 || ex->ci_stride < 1 || N != ex->ci_stride * ex->ci_stride * ex->ci_cin ||
                ex->ci_h != ex->strip_G * ex->ci_stride || ex->ci_w != ex->ci_h))
    return (int)cudaErrorInvalidValue;
  const bool mn = ex != nullptr && ex->mn_major != 0;
  if (mn) {
    // A (K, M), B (K, N) row-major; only the plain single-bf16 product with full-width (or 64-wide) N tiles
    if (split3 || split2 || ((ex->mn_major & 1) && (M % 8)) || ((ex->mn_major & 2) && (N % 8)) ||
        (((ex->mn_major & 3) != 3) && (K % 8)))
      return (int)cudaErrorInvalidValue;
  }
  // 128x256 tiles for the head products (rule in gemm.h).  The split count is the one the 128-wide tiles get, so that
  // every output element keeps its reduction order; the NoisyLinear weight gradient goes wide only unsplit.
  const long kb_all = (K + TBK - 1) / TBK;
  bool wide = false;
  if (!split3 && !split2 && N > 128 && kb_all >= 16 && (mn ? (ex->mn_major != 1 && ex->wg_t == 0) : !strip) &&
      (epi == TC_STORE || epi == TC_NOISY_WGRAD ||
       (epi == TC_BIAS_RELU && !mn && (ex == nullptr || ex->o_hiT == nullptr)))) {
    const long sms = riqn_sms();
    const long t128 = (long)((M + TBM - 1) / TBM) * ((N + 127) / 128), t256 = (long)((M + TBM - 1) / TBM) * ((N + 255) / 256);
    const bool unsplit = std::min(std::max(split_k, 1), std::min<int>(tc_max_split(t128), (int)kb_all)) == 1;
    wide = (epi != TC_NOISY_WGRAD || unsplit) && (t256 >= sms || 2 * ((t256 + sms - 1) / sms) <= (t128 + sms - 1) / sms);
  }
  // 128-wide tiles: the m64n128 accumulator of each consumer warpgroup is 64 registers per thread
  const int bn = wide ? 256
                      : (dgrad || (ex != nullptr && ex->mn_major)) ? ((dgrad || narrow_ok) && N <= 64 ? 64 : 128)
                                                                   : (narrow_ok && N <= 32) ? 32 : (narrow_ok && N <= 64) ? 64 : 128;
  CUtensorMap ma_hi, ma_lo, mb_hi, mb_lo;
  int rc;
  if (dgrad) {
    // A = dYg (M, K), B = the strip-ordered weight (K, strip_t^2 * N) read in 64 x 64 MN-major boxes
    rc = make_map(&ma_hi, A_hi, M, K, TBM);
    if (rc) return rc;
    rc = make_map(&mb_hi, B_hi, K, (long)ex->strip_t * ex->strip_t * N, 64);
    if (rc) return rc;
  } else if (mn) {
    const long b_cols = ex->wg_t ? (long)ex->wg_kc * TBK : N;      // strip weight gradient: B is the block matrix
    rc = (ex->mn_major & 1) ? make_map(&ma_hi, A_hi, K, M, 64) : make_map(&ma_hi, A_hi, M, K, TBM);
    if (rc) return rc;
    rc = (ex->mn_major & 2) ? make_map(&mb_hi, B_hi, K, b_cols, 64) : make_map(&mb_hi, B_hi, N, K, bn);
    if (rc) return rc;
  } else {
    rc = make_map(&ma_hi, A_hi, (ex && ex->a_rows) ? ex->a_rows : M, a_k, TBM);
    if (rc) return rc;
    rc = make_map(&mb_hi, B_hi, N, K, bn);
    if (rc) return rc;
  }
  ma_lo = ma_hi;
  mb_lo = mb_hi;
  if (split3) {
    rc = make_map(&ma_lo, A_lo, (ex && ex->a_rows) ? ex->a_rows : M, a_k, TBM);
    if (rc) return rc;
  }
  if (split3 || split2) {
    rc = make_map(&mb_lo, B_lo, N, K, bn);
    if (rc) return rc;
  }
  TcArgs p;
  p.M = M; p.N = N; p.K = K;
  p.m_tiles = (M + TBM - 1) / TBM;
  p.n_tiles = (N + bn - 1) / bn;
  p.kb_total = dgrad ? ex->strip_t * ex->strip_t : (K + TBK - 1) / TBK;   // strip data gradient: one k-block per shift
  if (split_k < 1) split_k = 1;
  // at most one round of CTAs: more splits would only multiply the partial sums written to scratch (gemm.h)
  if (split_k > tc_max_split(p.m_tiles * p.n_tiles)) split_k = tc_max_split(p.m_tiles * p.n_tiles);
  if (split_k > p.kb_total) split_k = p.kb_total;
  p.kb_per_split = (p.kb_total + split_k - 1) / split_k;
  p.k_splits = (p.kb_total + p.kb_per_split - 1) / p.kb_per_split;
  if (p.k_splits > 1 && epi != TC_ATOMIC && epi != TC_NOISY_WGRAD) return (int)cudaErrorInvalidValue;
  p.C = C; p.ldc = ldc; p.bias = bias; p.out2 = out2; p.eps = eps; p.part_stride = 0;
  p.alpha = ex ? ex->alpha : 1.f;
  p.vec_acc = (ldc % 4 == 0) && (reinterpret_cast<uintptr_t>(C) & 15) == 0 && (reinterpret_cast<uintptr_t>(out2) & 15) == 0 &&
              (reinterpret_cast<uintptr_t>(eps) & 15) == 0;
  p.ohw = ex ? ex->ohw : 1; p.feat = ex ? ex->feat : nullptr; p.batch = ex ? ex->batch : 1;
  p.ci_h = ex ? ex->ci_h : 0; p.ci_w = ex ? ex->ci_w : 0; p.ci_cin = ex ? ex->ci_cin : 0; p.ci_stride = ex ? ex->ci_stride : 0;
  p.strip_t = ex ? ex->strip_t : 0; p.strip_G = ex ? ex->strip_G : 0; p.strip_kc = ex ? ex->strip_kc : 0;
  p.cv_oh = ex ? ex->cv_oh : 0; p.cv_ow = ex ? ex->cv_ow : 0; p.nx_s = ex ? ex->nx_s : 0; p.nx_G = ex ? ex->nx_G : 0;
  p.nx_hi = ex ? ex->nx_hi : nullptr; p.nx_lo = ex ? ex->nx_lo : nullptr;
  p.mn_major = mn ? ex->mn_major : 0; p.wg_t = ex ? ex->wg_t : 0; p.wg_G = ex ? ex->wg_G : 0; p.wg_kc = ex ? ex->wg_kc : 0;
  p.o_hi = ex ? ex->o_hi : nullptr; p.o_lo = ex ? ex->o_lo : nullptr;
  p.o_hiT = ex ? ex->o_hiT : nullptr; p.o_loT = ex ? ex->o_loT : nullptr;
  p.fmt = ex ? ex->fmt : 0;
  p.grp_mt = ex ? ex->grp_mt : 0; p.a_wrap = ex ? ex->a_wrap : 0; p.bias2 = ex ? ex->bias2 : nullptr;
  if (p.grp_mt) {
    if (epi != TC_CONV || !ex->b2_hi || !ex->bias2 || p.m_tiles != 2 * p.grp_mt || (split3 || split2) != (ex->b2_lo != nullptr))
      return (int)cudaErrorInvalidValue;
    if ((rc = make_map(&p.mapO[0], ex->b2_hi, N, K, bn))) return rc;
    p.mapO[1] = p.mapO[0];
    if (ex->b2_lo && (rc = make_map(&p.mapO[1], ex->b2_lo, N, K, bn))) return rc;
  }
  if ((p.fmt & 3) && (split3 || split2)) return (int)cudaErrorInvalidValue;      // fp16 images are single-pass operands
  if ((p.fmt & 3) == 1 || (p.fmt & 3) == 2) return (int)cudaErrorInvalidValue;   // wgmma takes one 16-bit format for A and B
  if ((p.fmt & 4) && epi != TC_EMBED) return (int)cudaErrorInvalidValue;
  if (epi == TC_EMBED && ((N % 32) || (M % 2) || p.o_hiT || p.o_loT)) return (int)cudaErrorInvalidValue;
  if (epi == TC_EMBED) {            // the 16-bit images leave through TMA stores
    if (p.o_hi && (rc = make_store_map(&p.mapO[0], p.o_hi, M, N, 64))) return rc;
    if (p.o_lo && (rc = make_store_map(&p.mapO[1], p.o_lo, M, N, 64))) return rc;
  }
  // 128x256 forward (fp32 C, optional bf16 image) and bf16 data gradient (MN-major weight operand): the accumulator
  // leaves through TMA stores.  Their bases and row pitches must be 16-byte aligned; the slab epilogue's vector stores
  // needed the same, so an unaligned output is refused here instead of faulting in the kernel.
  const bool tma_epi = bn == 256 && (epi == TC_BIAS_RELU || (epi == TC_STORE && p.o_hi != nullptr && (p.mn_major & 2)));
  if (tma_epi) {
    const auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
    if ((epi == TC_BIAS_RELU && (!al16(C) || ldc % 4)) || (p.o_hi && (!al16(p.o_hi) || N % 8)))
      return (int)cudaErrorInvalidValue;
    if (epi == TC_BIAS_RELU && (rc = make_store_map_f32(&p.mapO[0], C, M, N, ldc))) return rc;
    if (p.o_hi && (rc = make_store_map(&p.mapO[1], p.o_hi, M, N, 64))) return rc;
  }
  const auto go = [&](int epi) -> int {
#define RIQN_TC_GO(NS, EP) return launch_tc<NS, EP, 128>(ma_hi, ma_lo, mb_hi, mb_lo, p, s)
#define RIQN_TC_NARROW(NS, EP)                                                                  \
    if (bn == 32) return launch_tc<NS, EP, 32>(ma_hi, ma_lo, mb_hi, mb_lo, p, s);                  \
    if (bn == 64) return launch_tc<NS, EP, 64>(ma_hi, ma_lo, mb_hi, mb_lo, p, s)
    if (split3) {
      switch (epi) {
        case TC_STORE: RIQN_TC_GO(3, TC_STORE);
        case TC_BIAS_RELU: RIQN_TC_GO(3, TC_BIAS_RELU);
        case TC_ATOMIC: RIQN_TC_GO(3, TC_ATOMIC);
        case TC_NOISY_WGRAD: RIQN_TC_GO(3, TC_NOISY_WGRAD);
        case TC_BIAS_RELU_NCHW: RIQN_TC_NARROW(3, TC_BIAS_RELU_NCHW); RIQN_TC_GO(3, TC_BIAS_RELU_NCHW);
        case TC_CONV: RIQN_TC_NARROW(3, TC_CONV); break;
        case TC_EMBED: return launch_tc<3, TC_EMBED, 128, 8>(ma_hi, ma_lo, mb_hi, mb_lo, p, s);
      }
    } else if (split2) {
      switch (epi) {
        case TC_BIAS_RELU_NCHW: RIQN_TC_NARROW(2, TC_BIAS_RELU_NCHW); RIQN_TC_GO(2, TC_BIAS_RELU_NCHW);
        case TC_CONV: RIQN_TC_NARROW(2, TC_CONV); break;
        case TC_STORE: RIQN_TC_GO(2, TC_STORE);
        default: return (int)cudaErrorInvalidValue;
      }
    } else if (bn == 256) {
      const int mode = p.mn_major | ((p.fmt & 3) ? 4 : 0) | (tma_epi ? 8 : 0);
#define RIQN_TC_WIDE(EP, MD) if (epi == EP && mode == MD) return launch_tc<1, EP, 256, MD>(ma_hi, ma_lo, mb_hi, mb_lo, p, s)
      RIQN_TC_WIDE(TC_BIAS_RELU, 8); RIQN_TC_WIDE(TC_BIAS_RELU, 12);
      RIQN_TC_WIDE(TC_STORE, 10); RIQN_TC_WIDE(TC_STORE, 11); RIQN_TC_WIDE(TC_STORE, 14); RIQN_TC_WIDE(TC_STORE, 15);
      RIQN_TC_WIDE(TC_STORE, 0); RIQN_TC_WIDE(TC_STORE, 2); RIQN_TC_WIDE(TC_STORE, 3);
      RIQN_TC_WIDE(TC_STORE, 4); RIQN_TC_WIDE(TC_STORE, 6); RIQN_TC_WIDE(TC_STORE, 7);
      RIQN_TC_WIDE(TC_NOISY_WGRAD, 0); RIQN_TC_WIDE(TC_NOISY_WGRAD, 2); RIQN_TC_WIDE(TC_NOISY_WGRAD, 3);
      RIQN_TC_WIDE(TC_NOISY_WGRAD, 4); RIQN_TC_WIDE(TC_NOISY_WGRAD, 6); RIQN_TC_WIDE(TC_NOISY_WGRAD, 7);
#undef RIQN_TC_WIDE
    } else {
      switch (epi) {
        case TC_STORE: RIQN_TC_NARROW(1, TC_STORE); RIQN_TC_GO(1, TC_STORE);
        case TC_CONV_DGRAD:
          if (bn == 64) return launch_tc<1, TC_CONV_DGRAD, 64>(ma_hi, ma_lo, mb_hi, mb_lo, p, s);
          RIQN_TC_GO(1, TC_CONV_DGRAD);
        case TC_BIAS_RELU: RIQN_TC_GO(1, TC_BIAS_RELU);
        case TC_ATOMIC: RIQN_TC_NARROW(1, TC_ATOMIC); RIQN_TC_GO(1, TC_ATOMIC);
        case TC_NOISY_WGRAD: RIQN_TC_GO(1, TC_NOISY_WGRAD);
        case TC_BIAS_RELU_NCHW: RIQN_TC_NARROW(1, TC_BIAS_RELU_NCHW); RIQN_TC_GO(1, TC_BIAS_RELU_NCHW);
        case TC_CONV: RIQN_TC_NARROW(1, TC_CONV); break;
        case TC_EMBED: return launch_tc<1, TC_EMBED, 128, 8>(ma_hi, ma_lo, mb_hi, mb_lo, p, s);
      }
    }
#undef RIQN_TC_NARROW
#undef RIQN_TC_GO
    return (int)cudaErrorInvalidValue;
  };
  if (p.k_splits == 1) return go(epi);
  // split-K: every split stores its partial product in its own slab of scratch (plain stores), then one pass adds the
  // slabs in split order into C (and out2), so the sum does not depend on which CTA finishes first
  const long ldp = (N + 3) & ~3L;           // 16-byte aligned slab rows for the vectorised stores
  StreamScratch part;
  RIQN_CUDA(part.alloc((size_t)p.k_splits * M * ldp, s));
  const float alpha = epi == TC_ATOMIC ? p.alpha : 1.f;
  p.C = part.p;
  p.ldc = ldp;
  p.part_stride = (long)M * ldp;
  p.o_hi = nullptr;
  if ((rc = go(TC_STORE))) return rc;
  const long n = (long)M * N;
  split_k_reduce_kernel<<<riqn_cdiv(n, 256), 256, 0, s>>>(M, N, p.k_splits, p.part_stride, ldp, part.p, C, ldc, alpha,
                                                          epi == TC_NOISY_WGRAD ? out2 : nullptr, eps);
  return (int)cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------- operand producers
// fp32 (rows, cols) -> bf16 hi (+ lo = bf16(x - hi)), optionally also transposed copies (cols, rows).
__global__ void split_bf16_kernel(long rows, int cols, const float* __restrict__ src, bf16* __restrict__ hi,
                                  bf16* __restrict__ lo, bf16* __restrict__ hiT, bf16* __restrict__ loT, int fp16) {
  __shared__ float tile[32][33];
  const long r0 = (long)blockIdx.y * 32;
  const int c0 = blockIdx.x * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;   // 32 x 8
  for (int i = ty; i < 32; i += 8) {
    const long r = r0 + i;
    const int c = c0 + tx;
    float x = 0.f;
    if (r < rows && c < cols) {
      x = src[r * cols + c];
      if (fp16) {                       // hi = fp16(x); lo (optional) = bf16(x), NOT a residual
        reinterpret_cast<__half*>(hi)[r * cols + c] = __float2half_rn(x);
        if (lo) lo[r * cols + c] = __float2bfloat16_rn(x);
        continue;
      }
      const bf16 h = __float2bfloat16_rn(x);
      if (hi) hi[r * cols + c] = h;
      if (lo) lo[r * cols + c] = __float2bfloat16_rn(x - __bfloat162float(h));
    }
    tile[i][tx] = x;
  }
  if (!hiT) return;
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {
    const int c = c0 + i;
    const long r = r0 + tx;
    if (r < rows && c < cols) {
      const float x = tile[tx][i];
      const bf16 h = __float2bfloat16_rn(x);
      hiT[(long)c * rows + r] = h;
      if (loT) loT[(long)c * rows + r] = __float2bfloat16_rn(x - __bfloat162float(h));
    }
  }
}

int split_bf16(long rows, int cols, const float* src, bf16* hi, bf16* lo, bf16* hiT, bf16* loT, cudaStream_t s, int fp16) {
  if (fp16 && (hi == nullptr || hiT != nullptr || loT != nullptr)) return (int)cudaErrorInvalidValue;
  dim3 grid((cols + 31) / 32, (unsigned)((rows + 31) / 32));
  split_bf16_kernel<<<grid, 256, 0, s>>>(rows, cols, src, hi, lo, hiT, loT, fp16);
  return (int)cudaGetLastError();
}

}  // namespace riqn

using namespace riqn;

__global__ void split_bf16_scaled_kernel(long n, const float* __restrict__ src, float scale, riqn::bf16* __restrict__ hi,
                                         riqn::bf16* __restrict__ lo) {
  const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float x = __fdiv_rn(src[i], scale);      // weight / 255, like the reference divides the pixel
  const riqn::bf16 h = __float2bfloat16_rn(x);
  hi[i] = h;
  if (lo) lo[i] = __float2bfloat16_rn(x - __bfloat162float(h));
}

RIQN_API int riqn_split_bf16_scaled(long rows, int cols, const float* src, float scale, void* hi, void* lo, void* stream) {
  riqn::note_launches(1);
  const long n = rows * cols;
  split_bf16_scaled_kernel<<<riqn_cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(n, src, scale, (riqn::bf16*)hi, (riqn::bf16*)lo);
  return (int)cudaGetLastError();
}

struct SplitJobs {
  riqn_split_job j[12];
  int blk_end[12];
  int n;
};

__global__ void split_bf16_multi_kernel(SplitJobs t) {
  int ji = 0;
  while (ji < t.n - 1 && (int)blockIdx.x >= t.blk_end[ji]) ++ji;
  const riqn_split_job& J = t.j[ji];
  const int idx = (blockIdx.x - (ji ? t.blk_end[ji - 1] : 0)) * blockDim.x + threadIdx.x;
  if (idx >= J.rows * J.cols) return;
  const int r = idx / J.cols, c = idx - r * J.cols;
  float x = J.src[(long)r * J.cols + (J.perm ? J.perm[c] : c)];
  if (J.div != 1.0f) x = __fdiv_rn(x, J.div);
  const riqn::bf16 h = __float2bfloat16_rn(x);
  reinterpret_cast<riqn::bf16*>(J.hi)[idx] = h;
  if (J.lo) reinterpret_cast<riqn::bf16*>(J.lo)[idx] = __float2bfloat16_rn(x - __bfloat162float(h));
  if (J.hi_t) reinterpret_cast<riqn::bf16*>(J.hi_t)[(long)c * J.rows + r] = h;
}

RIQN_API int riqn_split_bf16_multi(int n_jobs, const riqn_split_job* jobs, void* stream) {
  riqn::note_launches(1);
  if (n_jobs < 1 || n_jobs > 12 || jobs == nullptr) return (int)cudaErrorInvalidValue;
  SplitJobs t;
  t.n = n_jobs;
  int blocks = 0;
  for (int i = 0; i < n_jobs; ++i) {
    if (jobs[i].src == nullptr || jobs[i].hi == nullptr || jobs[i].rows < 1 || jobs[i].cols < 1) return (int)cudaErrorInvalidValue;
    t.j[i] = jobs[i];
    blocks += (int)riqn_cdiv((long)jobs[i].rows * jobs[i].cols, 256);
    t.blk_end[i] = blocks;
  }
  split_bf16_multi_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(t);
  return (int)cudaGetLastError();
}

RIQN_API int riqn_split_bf16(long rows, int cols, const float* src, void* hi, void* lo, void* hi_t, void* lo_t, int fp16,
                             void* stream) {
  riqn::note_launches(1);
  if (lo_t != nullptr && hi_t == nullptr) return (int)cudaErrorInvalidValue;   // the kernel writes lo_t beside hi_t only
  return split_bf16(rows, cols, src, (bf16*)hi, (bf16*)lo, (bf16*)hi_t, (bf16*)lo_t, (cudaStream_t)stream, fp16);
}

// Argument checks of the two C-ABI GEMM entry points (include/riqn_b200.h), made before anything is launched.  Every
// 32-column chunk that lies wholly inside N leaves as vectors: epilogues 0 / 1 store C as 16-byte row pieces (float4
// per row at odd M), epilogue 1 reads bias as float4, c_bf16 goes out in 16-byte pieces and c_t_bf16, at even M, in
// 32-bit pairs.  So from N = 32 on those bases must be aligned and C's pitch a multiple of 4 floats (narrower outputs
// take the scalar stores); epilogues 2 / 3 choose between vector and scalar accumulation at run time.  split_k > 1 is
// refused before gemm_bf16_tc clamps it, so that the answer does not depend on the SM count.
static bool tc_args_ok(int M, int N, float* c, long ldc, int epilogue, bool c_written, const float* bias, float* out2,
                       const float* eps, int split_k, const void* c_t_bf16, const void* c_bf16) {
  const auto al = [](const void* q, uintptr_t a) { return (reinterpret_cast<uintptr_t>(q) & (a - 1)) == 0; };
  const bool vec = N >= 32;
  if (epilogue < TC_STORE || epilogue > TC_NOISY_WGRAD) return false;
  if (split_k > 1 && epilogue != TC_ATOMIC && epilogue != TC_NOISY_WGRAD) return false;
  if (c_written && (c == nullptr || ldc < N)) return false;
  if (c_written && vec && epilogue <= TC_BIAS_RELU && (!al(c, 16) || ldc % 4)) return false;
  if (epilogue == TC_BIAS_RELU && (bias == nullptr || (vec && !al(bias, 16)))) return false;
  if (epilogue == TC_NOISY_WGRAD && (out2 == nullptr || eps == nullptr)) return false;
  if (c_bf16 && !al(c_bf16, 16)) return false;
  if (c_t_bf16 && (epilogue != TC_BIAS_RELU || (vec && M % 2 == 0 && !al(c_t_bf16, 4)))) return false;
  return true;
}

RIQN_API int riqn_gemm_bf16_tc(int M, int N, int K, const void* a_hi, const void* a_lo, const void* b_hi, const void* b_lo,
                               float* c, long ldc, int epilogue, const float* bias, float* out2, const float* eps,
                               int split_k, void* c_t_bf16, void* c_bf16, int fmt, void* stream) {
  riqn::note_launches(1);
  TcExtra ex;
  ex.o_hiT = (bf16*)c_t_bf16;
  ex.o_hi = (bf16*)c_bf16;
  ex.fmt = fmt & 3;
  if (c_bf16 && (epilogue != TC_BIAS_RELU || (M & 1) || (N % 32))) return (int)cudaErrorInvalidValue;
  if (!tc_args_ok(M, N, c, ldc, epilogue, true, bias, out2, eps, split_k, c_t_bf16, c_bf16)) return (int)cudaErrorInvalidValue;
  if (a_lo != nullptr && b_lo == nullptr) return (int)cudaErrorInvalidValue;        // x3 needs both lo images
  if (a_lo == nullptr && b_lo != nullptr && epilogue != TC_STORE) return (int)cudaErrorInvalidValue;   // split-2: store only
  return gemm_bf16_tc(M, N, K, (const bf16*)a_hi, (const bf16*)a_lo, (const bf16*)b_hi, (const bf16*)b_lo, c, ldc, epilogue,
                      bias, out2, eps, split_k, (cudaStream_t)stream, &ex);
}

RIQN_API int riqn_gemm_bf16_tc_mn(int M, int N, int K, const void* a, const void* b_kn, int a_is_km, float* c, long ldc,
                                  int epilogue, float* out2, const float* eps, float alpha, int split_k, void* c_bf16,
                                  int fmt, void* stream) {
  riqn::note_launches(1);
  if (epilogue != TC_STORE && epilogue != TC_ATOMIC && epilogue != TC_NOISY_WGRAD) return (int)cudaErrorInvalidValue;
  if (c_bf16 && (epilogue != TC_STORE || (N % 32))) return (int)cudaErrorInvalidValue;
  if (alpha != 1.f && epilogue != TC_ATOMIC) return (int)cudaErrorInvalidValue;     // only epilogue 2 scales
  if (!tc_args_ok(M, N, c, ldc, epilogue, c_bf16 == nullptr, nullptr, out2, eps, split_k, nullptr, c_bf16))
    return (int)cudaErrorInvalidValue;
  TcExtra ex;
  ex.o_hi = (bf16*)c_bf16;
  ex.mn_major = a_is_km ? 3 : 2;
  ex.alpha = alpha;
  ex.fmt = fmt & 3;
  return gemm_bf16_tc(M, N, K, (const bf16*)a, nullptr, (const bf16*)b_kn, nullptr, c, ldc, epilogue, nullptr, out2, eps,
                      split_k, (cudaStream_t)stream, &ex);
}
