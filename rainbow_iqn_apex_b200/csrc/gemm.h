// Internal GEMM interface shared by the op implementations (not part of the C-ABI).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include "common.cuh"

namespace riqn {

// C[m,n] (+)= epi( sum_k A[m*sAm + k*sAk] * B[n*sBn + k*sBk] )
enum Epi {
  EPI_STORE = 0,           // C = alpha*acc
  EPI_BIAS_RELU = 1,       // C = relu(acc + bias[n])
  EPI_BIAS_RELU_NCHW = 2,  // m = b*ohw + p ; C[(b*N + n)*ohw + p] = relu(acc + bias[n])
  EPI_EMBED = 3,           // C = feat[(m / batch)*N + n] * relu(acc + bias[n]), batch = rows per sample (model.py:146-151)
  EPI_NOISY_WGRAD = 5,     // C += acc ; out2 += acc * eps[m,n]  (dL/dmu, dL/dsigma of NoisyLinear; split 1 only)
  EPI_BIAS = 6,            // C = acc + bias[n]
  EPI_SLAB = 7,            // C[z * slab + m*ldc + n] = acc of split z (split-K partials, summed by the caller in split order)
};

struct EpiArgs {
  const float* bias = nullptr;
  const float* feat = nullptr;
  int batch = 1;
  int ohw = 1;
  float* out2 = nullptr;
  const float* eps = nullptr;
  float alpha = 1.0f;
  long slab = 0;
};

// fp32 CUDA-core GEMM with arbitrary operand strides.  Returns a cudaError_t as int.  split_k > 1 (EPI_SLAB only) cuts K
// into gemm_f32_splits(K, split_k) chunks of gemm_f32_kchunk(K, split_k), one grid z-slice each.
int gemm_f32_kchunk(int K, int split_k);
int gemm_f32_splits(int K, int split_k);
int gemm_f32(int M, int N, int K, const float* A, long sAm, long sAk, const float* B, long sBn, long sBk,
             float* C, long ldc, int epi, const EpiArgs& e, int split_k, cudaStream_t stream);
// C (M, N row-major) += A B^T, split-K: each split an fmaf chain over its k ascending, the splits added in split order
int gemm_f32_add(int M, int N, int K, const float* A, long sAm, long sAk, const float* B, long sBn, long sBk, float* C,
                 int split_k, cudaStream_t stream);

// ---- wgmma / TMA path (gemm_tc.cu) ---------------------------------------------------------------------------
enum TcEpi { TC_STORE = 0, TC_BIAS_RELU = 1, TC_ATOMIC = 2, TC_NOISY_WGRAD = 3, TC_BIAS_RELU_NCHW = 4, TC_EMBED = 5,
             TC_CONV = 7, TC_CONV_DGRAD = 8 };

struct TcExtra {
  int ohw = 1;
  float alpha = 1.0f;
  const float* feat = nullptr;
  int batch = 1;
  __nv_bfloat16 *o_hi = nullptr, *o_lo = nullptr, *o_hiT = nullptr, *o_loT = nullptr;
  int ci_h = 0, ci_w = 0, ci_cin = 0, ci_stride = 0;     // TC_CONV_DGRAD: the image din (see below)
  // Strip convolution (TC_CONV): A is the space-to-depth image (B*G*G rows of strip_kc*64 values); k-block kb reads rows
  // m0 + dy*G + dx (shift = kb / strip_kc = dy*strip_t + dx), columns (kb % strip_kc)*64.  Row m = (b, gy, gx) on the
  // G x G grid is a real output iff gy < cv_oh and gx < cv_ow; C is the NCHW fp32 output (relu(acc + bias)); nx_hi / nx_lo
  // (may be null) receive the bf16 images in the NEXT layer's space-to-depth layout (block edge nx_s, grid nx_G).
  int strip_t = 0, strip_G = 0, strip_kc = 0, cv_oh = 0, cv_ow = 0, nx_s = 0, nx_G = 0;
  __nv_bfloat16 *nx_hi = nullptr, *nx_lo = nullptr;
  // Data gradient of a strip convolution (TC_CONV_DGRAD), the same block grid read the other way: row m = (b, gy, gx) is
  // one input block, column n = (iy, ix, c) one of its N = stride^2 * Cin values.  A = dYg (M, K = Cout <= 64) and
  // k-block (dy, dx) (kb = dy*strip_t + dx, strip_t^2 of them) reads its rows m0 - (dy*strip_G + dx): the outputs that
  // block (gy, gx) fed through that shift.  Rows off the real outputs are zeros in dYg, and rows before the start come
  // from TMA's zero fill at negative coordinates, so no term crosses a row or a sample.  B = the strip-ordered weight
  // (K, strip_t^2 * N), k-block kb reading its columns [kb*N, (kb+1)*N) as an MN-major operand.  Each shift's product is
  // formed in a fresh accumulator and added to the fp32 sum in kb order (the order of kh, then kw, ascending);
  // C = din, NCHW (ci_cin, ci_h, ci_w, ci_stride; ci_h == strip_G * ci_stride), written once.
  // MN-major operands (mn_major bit 0: A is (K, M) row-major, bit 1: B is (K, N) row-major): the reduction index is the
  // ROW, as in a weight gradient dW = dY^T X taken straight from the row-major activations, or a data gradient
  // dX = dY W read from the untransposed weight (mn_major = 2).  NSPLIT 1 only.
  // wg_t > 0 additionally applies the strip-convolution shifts to B: column n = (shift, within-block) reads the rows
  // k + dy*wg_G + dx of a block matrix with wg_kc*64 columns (shift = n / (wg_kc*64) = dy*wg_t + dx).
  int mn_major = 0, wg_t = 0, wg_G = 0, wg_kc = 0;
  // 16-bit operand formats: 0 = both operand images bf16, 3 = both fp16 (single-pass products only; mixing the two is an
  // illegal instruction), bit 2 = TC_EMBED writes o_hi as fp16(x) and o_lo (optional) as bf16(x) instead of hi / residual
  int fmt = 0;
  // TC_CONV with TWO weight sets over one stacked batch (the online and the target network's trunks over the same frames
  // in one launch): m-tiles [0, grp_mt) use B_hi / B_lo / bias, m-tiles [grp_mt, 2*grp_mt) use b2_hi / b2_lo / bias2.
  // a_wrap != 0: both groups read the SAME A rows (a_rows = rows of the A image; conv1: the pixel block matrix is shared).
  int grp_mt = 0, a_wrap = 0;
  long a_rows = 0;
  const __nv_bfloat16 *b2_hi = nullptr, *b2_lo = nullptr;
  const float* bias2 = nullptr;
};

// C (+)= A B^T, A (M,K) / B (N,K) row-major bf16 (K % 8 == 0); *_lo non-null selects the split-bf16 x3 product.
// (TC_CONV: M = B*G*G grid rows, K = strip_t^2 * strip_kc * 64.  TC_CONV_DGRAD: K = Cout, the reduction of one shift.)
int gemm_bf16_tc(int M, int N, int K, const __nv_bfloat16* A_hi, const __nv_bfloat16* A_lo, const __nv_bfloat16* B_hi,
                 const __nv_bfloat16* B_lo, float* C, long ldc, int epi, const float* bias, float* out2, const float* eps,
                 int split_k, cudaStream_t s, const TcExtra* ex);
//
// Tile choice.  Single-pass (fp16 or bf16) products take 128x256 tiles (one producer and two m64n256 consumer
// warpgroups) when
//   * the epilogue is TC_BIAS_RELU without a transposed image, TC_STORE, or TC_NOISY_WGRAD that the split rule below
//     leaves unsplit (the wide tiles never change a product's split count, so every output element keeps its reduction
//     order and the result is bitwise the one of 128-wide tiles),
//   * the operands are K-major, or mn_major 2 / 3 without strip shifts,
//   * N > 128 and K >= 1024 (16 k-blocks: with fewer the epilogue dominates and 128-wide tiles spread it over more SMs),
//   * and the wide tiles fill the SMs (at least one per SM), or take at most half as many rounds of CTAs as the 128-wide
//     ones (the 1024 x 3136 weight gradient: 104 wide tiles in one round against 200 narrow ones in two).
// These are the NoisyLinear head's forward, data gradient and weight gradient.  Everything else runs 128x{128,64,32}
// tiles: split-bf16 x3, the convolutions, the embedding, narrow outputs, split products and small products that
// would leave SMs idle.
//
// Split-K over a persistent grid of one CTA per SM: every split writes its partial product to scratch and one pass adds
// them in split order, so splits beyond one round of CTAs only add partial sums.  tc_max_split is the most splits that
// still fit in one round for `tiles` output tiles; tc_pick_split takes that many, but no more than the `kb` reduction
// blocks of 64 (e.g. 25 tiles on 132 SMs -> 5 splits, 125 units).
inline int tc_max_split(long tiles) {
  if (tiles < 1) tiles = 1;
  const long s = riqn_sms() / tiles;
  return s < 1 ? 1 : (int)s;
}
inline int tc_pick_split(int tiles, long kb) {
  const int s = tc_max_split(tiles);
  return kb < s ? (int)(kb < 1 ? 1 : kb) : s;
}

int split_bf16(long rows, int cols, const float* src, __nv_bfloat16* hi, __nv_bfloat16* lo, __nv_bfloat16* hiT,
               __nv_bfloat16* loT, cudaStream_t s, int fp16 = 0);

}  // namespace riqn
