/* riqn_b200.h -- C-ABI of the H100-native (sm_90a) Rainbow-IQN Ape-X learner hot path.
 *
 * The reference (valeoai/rainbow-iqn-apex) is pure Python/PyTorch and has no FFI or operator registry:
 * its boundary for this path is the Python class surface Agent / Learner / DQN / NoisyLinear /
 * ReplayRedisMemory (SURVEY.md section 8b).  This header is the boundary a native replacement exports
 * underneath that surface; rainbow_iqn_apex_b200/*.py binds it with ctypes (see INTEGRATION.md) and
 * re-creates the reference classes on top.
 *
 * Conventions
 *   - every function returns 0 on success or a cudaError_t value; all buffers are caller-owned DEVICE pointers
 *     unless stated; work is enqueued on `stream` (a cudaStream_t passed as void*) and is stream-ordered,
 *     re-entrant per stream.  The only memory a call takes itself is temporary scratch for partial sums (and the
 *     strip-ordered weight copy of riqn_conv_bwd_strip), allocated
 *     from the device's stream-ordered pool on `stream` and released on `stream` before the call returns
 *     (cudaMallocAsync / cudaFreeAsync): no host synchronisation, no state shared between calls or streams, and
 *     inside a CUDA graph capture it becomes part of the graph;
 *   - results are bitwise reproducible: no sum across thread blocks uses float atomics;
 *   - fp32 tensors row-major.  tau, q and dtheta use the reference's quantile-major rows r = q * batch + b
 *     (rainbowiqn/model.py:149, compute_loss_iqn.py:238-310); the head-internal matrices (cos, x, h, dh, dz and
 *     their bf16 images) use sample-major rows r' = b * num_quantiles + q, which makes the Hadamard operand
 *     feat[b,:] a warp-broadcast and the reduction over a sample's quantiles contiguous;
 *   - `long long*` index buffers are int64 like the reference's torch.int64 / numpy int64.
 *
 * Each entry point cites the reference code it replaces (paths relative to the reference repository).
 */
#ifndef RIQN_B200_H
#define RIQN_B200_H

#ifdef __cplusplus
extern "C" {
#endif

#define RIQN_B200_ABI_VERSION 1

/* Library / build identification.  Returns RIQN_B200_ABI_VERSION. */
int riqn_version(void);
/* Number of CUDA kernels this library has launched in this process (bench.py's gpu_launches). */
long long riqn_launch_count(void);
/* 1 if the running device is compute capability 9.x (sm_90a cubins only), else 0; <0 on CUDA error. */
int riqn_device_ok(void);

/* Per-step scalars that change from one learner step to the next, kept in DEVICE memory so that a whole step can be
 * captured once in a CUDA graph and replayed: entry points taking `dyn` read these instead of their by-value arguments
 * when dyn != NULL (the host rewrites the 32-byte struct with one async copy before each replay). */
typedef struct riqn_dyn_state {
  unsigned long long rng_offset;   /* added to every Philox stream id (advance by >= 64 per step)          */
  float adam_neg_step_size;        /* -(lr / (1 - beta1^t))                                                 */
  float adam_sqrt_bc2;             /* sqrt(1 - beta2^t)                                                     */
  double is_capacity;              /* current replay fill, ReplayRedisMemory.sample_byte capacity (:467)    */
  double is_beta;                  /* priority_weight beta (annealed by the caller, launch_learner.py:167)  */
} riqn_dyn_state;

/* Update horizon of one learner step under n-step and discount annealing (BBF), kept in DEVICE memory beside
 * riqn_dyn_state so that a captured step follows the schedule on replay.  One host writer (dynstate.HorizonState)
 * fills it with one async copy per step and guarantees 1 <= n_step <= the entry point's n_max; the entry points keep
 * n_step in 1..n_max all the same. */
#define RIQN_MAX_HORIZON 16
typedef struct riqn_horizon_state {
  int n_step;                              /* this step's n                                                    */
  float gamma_n;                           /* fl32(gamma ** n_step), the power taken in double on the host     */
  double gamma_pow[RIQN_MAX_HORIZON];      /* gamma ** k in double for k < n_step (ReplayMemory._gamma_pow)    */
} riqn_horizon_state;

/* ------------------------------------------------------------------------------------------------
 * Conv trunk                                     replaces nn.Conv2d x3 + ReLU, rainbowiqn/model.py:65-67,115-118
 * ---------------------------------------------------------------------------------------------- */
typedef struct riqn_conv_geom {
  int B, Cin, H, W;          /* input  (B, Cin, H, W), NCHW                                     */
  int Cout, KH, KW;          /* weight (Cout, Cin, KH, KW)                                       */
  int stride, pad;
  int OH, OW;                /* output (B, Cout, OH, OW), NCHW (flattens C-major, model.py:118)  */
  long in_bstride;           /* elements between consecutive samples of the input (>= Cin*H*W):
                                lets conv1 read states / next_states as strided views of the
                                (B, history+n, 84, 84) replay window                             */
} riqn_conv_geom;

/* The trunk takes one of three paths:
 *   - strip convolution (riqn_s2d_u8, riqn_conv_fwd_strip, riqn_conv_bwd_strip): uint8 frames with 16-byte aligned
 *     samples and history 4, in every tensor-core precision mode;
 *   - explicit im2col on the tensor cores (riqn_conv_fwd_tc, riqn_conv_bwd_tc): every other input (fp32 frames, uint8
 *     frames that are unaligned or of another history);
 *   - fp32 on the CUDA cores (riqn_conv_fwd, riqn_conv_bwd), the cross-check path.  riqn_conv_bwd on the operands of
 *     riqn_im2col_f32 is also the backward of the other two when the backward is not bf16 or an im2col row count
 *     (B*OH*OW) is not a multiple of 8. */

/* out = relu(conv(in) + bias).  `in` is uint8 frames (x/255 applied on the fly, reproducing
 * redis_memory.py:527-536) when in_is_u8 != 0, else fp32.  `col` (B*OH*OW, Cin*KH*KW) is workspace
 * that riqn_conv_bwd re-uses. */
int riqn_conv_fwd(const riqn_conv_geom* g, const void* in, int in_is_u8, const float* w, const float* bias,
                  float* col, float* out, void* stream);
/* Backward of the above: dout is dL/d(out) (post-ReLU), `out` the forward output (ReLU mask).
 * dw/dbias are ACCUMULATED into (zero them first, like zero_grad -- learner.py:22); din (may be NULL
 * for the first layer) is overwritten with dL/d(in).  dY (B*OH*OW, Cout) and dcol (like col) are
 * workspaces.  dw += the split-K product dY^T col: each split an fp32 fmaf chain over its rows ascending, the splits
 * added in split order, the sum added once; din[b, c, ih, iw] = the fp32 sum over (kh, kw) ascending of dcol. */
int riqn_conv_bwd(const riqn_conv_geom* g, const float* dout, const float* out, const float* col, const float* w,
                  float* dY, float* dcol, float* dw, float* dbias, float* din, void* stream);

/* fp32 im2col alone: col (B*OH*OW, Cin*KH*KW), the workspace riqn_conv_bwd expects. */
int riqn_im2col_f32(const riqn_conv_geom* g, const void* in, int in_is_u8, float* col, void* stream);

/* Tensor-core variants (wgmma GEMM on bf16 im2col operands written straight from the uint8 / fp32 input).
 * w_hi / w_lo: bf16 images of the (Cout, Cin*KH*KW) weight (riqn_split_bf16); col_lo == NULL selects the
 * single-bf16 product, otherwise split-bf16 x3 (fp32-faithful).  col_hi/col_lo (M, K) bf16 workspaces; colT_hi
 * (K, M), if non-NULL, is also written for riqn_conv_bwd_tc (needs B*OH*OW % 8 == 0). */
int riqn_conv_fwd_tc(const riqn_conv_geom* g, const void* in, int in_is_u8, const void* w_hi, const void* w_lo,
                     const float* bias, void* col_hi, void* col_lo, void* colT_hi, float* out, void* stream);
/* Strip convolution: the forward of nn.Conv2d + ReLU (model.py:65-67,115-118) with NO im2col matrix.  With kernel edge
 * k = t*stride the padded input is cut into stride x stride blocks (block matrix: B*G*G rows of stride^2*Cin values,
 * G = OH + t - 1) and the outputs are laid on the same G x G grid, so that every k-block of the implicit im2col matrix
 * is a 2-D tile of the block matrix at a row offset (TMA).  Requires stride^2*Cin % 64 == 0, Cout <= 64.
 *   riqn_s2d_u8: uint8 frame stack -> block matrix a_px (B*G*G, stride^2*Cin) bf16 of raw pixel values, within-block
 *                order (c, iy, ix); the 1/255 of redis_memory.py:527-536 is folded into the weights.
 *   riqn_conv_fwd_strip: a_hi / a_lo (lo may be NULL) block matrices; w_hi / w_lo (Cout, K) bf16 weights with K
 *                ordered (dy, dx, within-block); out (B, Cout, OH, OW) fp32 = relu(conv + bias), or NULL when only the
 *                next layer's images are wanted (no-grad passes); next_hi / next_lo (may be
 *                NULL) receive the result as the NEXT layer's block matrix (block edge next_stride, grid next_grid,
 *                within-block order (iy, ix, c)). */
int riqn_s2d_u8(const riqn_conv_geom* g, const unsigned char* in, void* a_px, void* stream);
/* Random-shift augmentation (DrQ): edge-replicating shifts of two batches of (C, H, W) images into one contiguous
 * (nimg, C, H, W) buffer in the inputs' element type (is_u8: uint8, else fp32).  Image i < B reads in0 + i*in0_bstride,
 * image B + i reads in1 + i*in1_bstride (strides in elements); in1 may be NULL (nimg = B, else 2B).  With (dy, dx) =
 * (shifts[2i], shifts[2i+1]) of image i,
 *   out[i, c, y, x] = in_i[c, clamp(y + dy, 0, H-1), clamp(x + dx, 0, W-1)]
 * i.e. ReplicationPad2d(p) followed by a crop at (dy + p, dx + p) for |dy|, |dx| <= p; larger shifts clamp too.
 * Returns cudaErrorInvalidValue (and writes nothing) for B, C, H or W < 1, a NULL in0 / shifts / out, is_u8 not 0 or 1,
 * a batch stride < C*H*W, an in0 / in1 / out address or a batch stride in bytes that is not a multiple of 16, or an
 * (H, W) plane whose size in bytes is not a multiple of 16 or exceeds 48 KB. */
int riqn_random_shift(int B, int C, int H, int W, const void* in0, long in0_bstride, const void* in1, long in1_bstride,
                      int is_u8, const int* shifts, void* out, void* stream);
int riqn_conv_fwd_strip(const riqn_conv_geom* g, const void* a_hi, const void* a_lo, const void* w_hi, const void* w_lo,
                        const float* bias, float* out, void* next_hi, void* next_lo, int next_stride, int next_grid,
                        const void* w2_hi, const void* w2_lo, const float* bias2, int share_a, void* stream);
/* w2_hi != NULL: TWO networks in one launch (the online and the target trunk over the same next_states): g->B counts both
 * halves of a stacked batch, samples [0, B/2) use w_hi / w_lo / bias, samples [B/2, B) use w2_hi / w2_lo / bias2; outputs and
 * next-layer images are the stacked (B, ...) tensors.  share_a != 0: the A image holds B/2 samples read by both halves (first
 * layer: the pixel block matrix).  Needs (B/2)*G*G % 128 == 0. */
/* Backward of a strip convolution on the tensor cores, again without im2col matrices: a_hi is the block matrix the
 * forward read (riqn_s2d_u8 / the previous layer's next_hi); w_hi (Cout, K) bf16 weight in the ORIGINAL k order (the
 * data gradient reads a strip-ordered copy the call makes in its scratch); perm (K ints): strip k order -> original k;
 * dYg (B*G*G, Cout) bf16 and dwp_scratch (Cout*K floats) workspaces; dw / dbias accumulated; din (may be NULL; pad == 0
 * and H == W == G*stride only) overwritten, every element once, as the transposed strip convolution of dYg.
 * wgrad_scale = 1/255 when a_hi holds raw pixel values. */
int riqn_conv_bwd_strip(const riqn_conv_geom* g, const float* dout, const float* out, const void* a_hi, const void* w_hi,
                        const int* perm, void* dYg, float* dwp_scratch, float* dw, float* dbias, float* din,
                        float wgrad_scale, void* stream);

/* Backward of riqn_conv_fwd_tc on the tensor cores (bf16 operands, fp32 accumulate): colT_hi as that forward wrote it;
 * wT_hi (K, Cout) bf16; dY_hi (M, Cout) and dYT_hi (Cout, M) bf16 workspaces; dcol fp32 (M, K) workspace; dw/dbias
 * accumulated, dw += wgrad_scale * (dY^T col) (the trunk passes 1); din may be NULL; with din, dcol = dY W (non-NULL)
 * and din[b, c, ih, iw] = the fp32 sum over (kh, kw) ascending of dcol. */
int riqn_conv_bwd_tc(const riqn_conv_geom* g, const float* dout, const float* out, const void* colT_hi, const void* wT_hi,
                     void* dY_hi, void* dYT_hi, float* dcol, float* dw, float* dbias, float* din, float wgrad_scale,
                     void* stream);
/* split of (src * scale): bf16 hi / lo images of a scaled matrix (e.g. weight/255). */
int riqn_split_bf16_scaled(long rows, int cols, const float* src, float scale, void* hi, void* lo, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Randomness                       replaces torch normal_/uniform_ draws, model.py:32-37 and :131-134
 * ---------------------------------------------------------------------------------------------- */
/* out[i] ~ U(0,1): the quantile fractions tau.  Philox4x32-10 keyed by (seed, stream_id). */
int riqn_fill_uniform(long n, unsigned long long seed, unsigned long long stream_id, float* out,
                      const riqn_dyn_state* dyn, void* stream);

/* Distortion risk measures beta of riqn_fill_tau_distorted (IQN paper, Dabney et al. 2018, section 3.1). */
#define RIQN_RISK_NEUTRAL 0   /* beta(t) = t                                                          */
#define RIQN_RISK_CVAR 1      /* beta(t) = eta t,                                      0 < eta <= 1   */
#define RIQN_RISK_WANG 2      /* beta(t) = Phi(Phi^-1(t) + eta),                       eta finite     */
#define RIQN_RISK_CPW 3       /* beta(t) = t^eta / (t^eta + (1-t)^eta)^(1/eta),        eta > 0        */
#define RIQN_RISK_POW 4       /* beta(t) = t^(1/(1+|eta|)) for eta >= 0, 1-(1-t)^(1/(1+|eta|)) for eta < 0, eta finite */
#define RIQN_RISK_NORM 5      /* mean of eta uniforms,                                 eta in {1..32} */
/* out[i] = beta(u_i): the distorted quantile fractions of risk-sensitive action selection.  u is exactly what
 * riqn_fill_uniform(n, seed, stream_id) writes (same Philox counters, same dyn->rng_offset), so out[i] applies beta to
 * the plain draw's element i.  Norm: out[i] = (u'[i*eta] + ... + u'[i*eta + eta-1]) / eta, summed in that order, where
 * u' is what riqn_fill_uniform(n * eta, seed, stream_id) writes.  beta is evaluated in double and rounded once to float.
 * Returns cudaErrorInvalidValue (and writes nothing) for an unknown measure or an eta outside its domain. */
int riqn_fill_tau_distorted(long n, unsigned long long seed, unsigned long long stream_id, int measure, float eta,
                            float* out, const riqn_dyn_state* dyn, void* stream);
/* out[i] = sign(x) sqrt|x|, x ~ N(0,1): NoisyLinear._scale_noise (model.py:32-37). */
int riqn_noisy_sample(long n, unsigned long long seed, unsigned long long stream_id, float* out,
                      const riqn_dyn_state* dyn, void* stream);
/* n random shifts (dy, dx) in [-pad, pad]^2 for random-shift augmentation (DrQ), out (n, 2) int32.  Component j of pair i
 * reads the Philox word x that riqn_fill_uniform(2n, seed, stream_id) turns into its value at position 2i + j (same
 * counters, same dyn->rng_offset); with m = x >> 8, the 24 bits behind that uniform u = (m + 0.5) / 2^24,
 *   out[2i + j] = ((m (2 pad + 1)) >> 24) - pad        (integer arithmetic: exact, and within [-pad, pad] for every m)
 * Returns cudaErrorInvalidValue (and writes nothing) for n < 0, pad outside [0, 2^30) or a NULL out with n > 0. */
int riqn_fill_shifts(long n, int pad, unsigned long long seed, unsigned long long stream_id, int* out,
                     const riqn_dyn_state* dyn, void* stream);

/* ------------------------------------------------------------------------------------------------
 * NoisyLinear                                             replaces rainbowiqn/model.py:9-53
 * ---------------------------------------------------------------------------------------------- */
/* reset_noise + effective weights in one pass.  If eps_in/eps_out are non-NULL, weight_epsilon :=
 * eps_out (x) eps_in and bias_epsilon := eps_out are (re)written (model.py:39-43); otherwise the
 * stored epsilons are used.  w_eff = mu + sigma*eps, b_eff likewise (training != 0, model.py:46-51)
 * or the mu's alone (eval, model.py:52-53). */
int riqn_noisy_compose(int out_features, int in_features, const float* weight_mu, const float* weight_sigma,
                       float* weight_epsilon, const float* eps_in, const float* eps_out, const float* bias_mu,
                       const float* bias_sigma, float* bias_epsilon, float* w_eff, float* b_eff, int training,
                       void* stream);

/* One NoisyLinear layer of a network-wide noise reset (riqn_noisy_reset_net). */
typedef struct riqn_noisy_layer {
  int out_features, in_features;                 /* in_features % 4 == 0 */
  const float* weight_mu;
  const float* weight_sigma;
  float* weight_epsilon;                         /* (out, in): eps_out (x) eps_in is written here */
  const float* bias_mu;
  const float* bias_sigma;
  float* bias_epsilon;                           /* (out) */
  float* eps_in;                                 /* (in)  factor vector f(eps_in): drawn here when sample != 0 */
  float* eps_out;                                /* (out) factor vector f(eps_out) */
  float* w_eff;                                  /* (out, in) mu + sigma * eps   (mu when training == 0) */
  float* b_eff;                                  /* (out) */
  unsigned long long stream_in, stream_out;      /* Philox stream ids of the two draws */
  void* w_hi;                                    /* (out, in) bf16 image of w_eff for the tensor-core products, or NULL */
  void* w_lo;                                    /* (out, in) bf16(w_eff - hi), or NULL */
  int w_fp16;                                    /* != 0: w_hi = fp16(w_eff), w_lo (or NULL) = bf16(w_eff) -- fp16 head forward */
} riqn_noisy_layer;

/* DQN.reset_noise() for all NoisyLinear layers of one network in two launches (model.py:159-162 -> :39-43 -> :32-37):
 * draw every factor vector (sample != 0; same values as riqn_noisy_sample on the same seed / stream ids), then
 * compose every layer like riqn_noisy_compose.  layers is a HOST array of n_layers <= 8 descriptors. */
int riqn_noisy_reset_net(int n_layers, const riqn_noisy_layer* layers, unsigned long long seed, int sample, int training,
                         const riqn_dyn_state* dyn, void* stream);
/* h = relu(x w_eff^T + b_eff)   (the hidden layers fcnoisy_h_v | fcnoisy_h_a concatenated along out_features,
 * model.py:153-154 with the F.relu folded in). */
int riqn_noisy_linear_fwd(long rows, int in_features, int out_features, const float* x, const float* w_eff,
                          const float* b_eff, float* h, void* stream);
/* dx = dh w_eff   (dh already masked by the ReLU). */
int riqn_noisy_linear_dgrad(long rows, int in_features, int out_features, const float* dh, const float* w_eff,
                            float* dx, void* stream);
/* grad_weight_mu += dh^T x ; grad_weight_sigma += (dh^T x) * weight_epsilon ; bias grads likewise.
 * db_scratch: out_features floats. */
int riqn_noisy_linear_wgrad(long rows, int in_features, int out_features, const float* dh, const float* x,
                            const float* weight_epsilon, const float* bias_epsilon, float* db_scratch,
                            float* grad_weight_mu, float* grad_weight_sigma, float* grad_bias_mu,
                            float* grad_bias_sigma, void* stream);

/* Bias half of the above alone (used when the weight half runs on the tensor cores).  dh == NULL: db_scratch already holds
 * the column sums of dh (riqn_dueling_bwd_bf16). */
int riqn_noisy_bias_grad(long rows, int out_features, const float* dh, const float* bias_epsilon, float* db_scratch,
                         float* grad_bias_mu, float* grad_bias_sigma, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Quantile embedding                                      replaces rainbowiqn/model.py:136-151
 * ---------------------------------------------------------------------------------------------- */
/* cosv[r',i] = cos(fl(fl(i+1)*fl(pi)) * tau[q*batch+b]);  x[r',:] = feat[b,:] * relu(cosv[r',:] iqn_w^T + iqn_b),
 * r' = b*num_quantiles + q (sample-major output rows, quantile-major tau).
 * tau (rows), feat (batch, feat_dim), iqn_w (feat_dim, embed_dim); cosv (rows, embed_dim) and
 * x (rows, feat_dim) are outputs, rows = batch * num_quantiles. */
int riqn_quantile_embed_fwd(int batch, int num_quantiles, int embed_dim, int feat_dim, const float* tau,
                            const float* feat, const float* iqn_w, const float* iqn_b, float* cosv, float* x,
                            void* stream);
/* Given dL/dx in dx_inout (overwritten with dL/d(pre-activation of iqn_fc)): dfeat (batch, feat_dim) is
 * overwritten; grad_iqn_w / grad_iqn_b are accumulated into. */
int riqn_quantile_embed_bwd(int batch, int num_quantiles, int embed_dim, int feat_dim, const float* x,
                            const float* feat, const float* cosv, float* dx_inout, float* dfeat, float* grad_iqn_w,
                            float* grad_iqn_b, void* stream);

/* Tensor-core variants.  Forward: the wgmma GEMM's epilogue applies relu / bias / the Hadamard with feat and writes
 * the bf16 operand images of x directly: x_hi, x_lo (rows, feat_dim) for the NoisyLinear product, x_hi_t / x_lo_t
 * (feat_dim, rows) for its weight gradient in the cross-check arithmetic modes (each may be NULL; the transposed images
 * are split from x32 by a second launch and therefore need x32 != NULL); x32 (may be NULL) is the fp32 matrix.  cos_hi / cos_lo
 * (rows, embed_dim) and cos_t_hi (embed_dim, rows; may be NULL) are outputs too.  cos_lo == NULL selects the
 * single-bf16 product.  iqn_w_hi / iqn_w_lo: bf16 images of iqn_fc.weight (riqn_split_bf16).  rows % 2, feat_dim % 32
 * and embed_dim % 8 must be 0, cos_hi, cos_lo, iqn_w_hi, iqn_w_lo, x32, x_hi, x_lo 16-byte aligned, and feat and iqn_b
 * 8-byte aligned; a call rejected for its shapes or alignment (cudaErrorInvalidValue) writes nothing. */
int riqn_quantile_embed_fwd_tc(int batch, int num_quantiles, int embed_dim, int feat_dim, const float* tau,
                               const float* feat, const void* iqn_w_hi, const void* iqn_w_lo, const float* iqn_b,
                               void* cos_hi, void* cos_lo, void* cos_t_hi, float* x32, void* x_hi, void* x_lo, void* x_hi_t,
                               void* x_lo_t, int x_fp16, void* stream);
/* x_fp16 != 0: x_hi = fp16(x), the operand of the single-pass fp16 head product (same tensor-core rate as bf16, 11-bit
 * significand), and x_lo (or NULL) = bf16(x), the operand of the bf16 backward; x_hi_t / x_lo_t must be NULL. */
/* Backward on bf16 operands (rows % 8 == 0): dx (rows, feat_dim) from the head dgrad, fp32 or (dx_is_bf16 != 0) bf16;
 * x_lo may be NULL (x = x_hi); cos_hi (rows, embed_dim) bf16 row-major (the forward's image); dpre (rows, feat_dim) bf16
 * workspace; dfeat overwritten; grad_iqn_w / grad_iqn_b accumulated. */
int riqn_quantile_embed_bwd_tc(int batch, int num_quantiles, int embed_dim, int feat_dim, const void* x_hi, const void* x_lo,
                               const float* feat, const void* cos_hi, const void* dx, int dx_is_bf16, void* dpre,
                               float* dfeat, float* grad_iqn_w, float* grad_iqn_b, void* stream);

/* ------------------------------------------------------------------------------------------------
 * z-layers + dueling aggregation                          replaces rainbowiqn/model.py:153-156
 * ---------------------------------------------------------------------------------------------- */
/* h (rows, 2*hidden) = [value-stream hidden | advantage-stream hidden]; wz (1+A, hidden) = effective
 * weights of fcnoisy_z_v (row 0) and fcnoisy_z_a; bz (1+A).  q (rows, A) = v + a - mean_a a, row r of h (sample-major,
 * r = b*(rows/batch) + k) going to row k*batch + b of q (quantile-major).  Returns cudaErrorInvalidValue, writing
 * nothing, unless hidden == 512, 1 <= action_space <= 31, batch >= 1, rows % batch == 0, and h and wz are 16-byte
 * aligned. */
int riqn_dueling_fwd(long rows, int batch, int hidden, int action_space, const float* h, const float* wz,
                     const float* bz, float* q, void* stream);
/* Backward for the gathered action: dq[r, actions[b]] = dtheta[r] * gscale[b].  Writes dh (rows, 2*hidden),
 * already masked by h > 0, and dz (rows, 32) = [dv, da_0.., 0..] for riqn_z_wgrad; dz_bf16 (may be NULL) is its bf16
 * image (rows, 32) for riqn_z_wgrad_tc. */
int riqn_dueling_bwd(long rows, int batch, int hidden, int action_space, const float* h, const float* wz,
                     const float* dtheta, const float* gscale, float gscale_mul, const long long* actions, float* dh,
                     float* dz, void* dz_bf16, void* stream);
/* (gscale_mul multiplies gscale[b]: the learner passes the IS weights and 1/B, learner.py:23's .mean(), without an extra
 * elementwise launch) */
/* Same backward for bf16 tensor-core consumers (rows % 8 == 0): instead of the fp32 dh it writes dh_hi (rows, 2*hidden)
 * as bf16 (and its transpose dh_hi_t (2*hidden, rows) if non-NULL), dh_colsum (2*hidden) = the fp32 column sums of dh
 * (zeroed here; pass it to riqn_noisy_bias_grad with dh == NULL) and dz_bf16 (rows, 32), if non-NULL, the bf16 image of
 * dz for riqn_z_wgrad_tc.  Only the sign of h matters here (ReLU mask): h_bf16 (rows, 2*hidden), if non-NULL, is read
 * instead of h. */
int riqn_dueling_bwd_bf16(long rows, int batch, int hidden, int action_space, const float* h, const void* h_bf16,
                          const float* wz,
                          const float* dtheta, const float* gscale, float gscale_mul, const long long* actions, void* dh_hi,
                          void* dh_hi_t,
                          float* dh_colsum, float* dz, void* dz_bf16, void* stream);
/* The same two backwards for a dense upstream gradient grad_q = dL/dq (rows, A), fp32, quantile-major rows q*batch+b as
 * riqn_dueling_fwd writes q:  dv = sum_a grad_q[a] ; da_k = grad_q[k] - dv/A ; dh_v = dv * w_zv ; dh_a = sum_k da_k w_za[k],
 * both masked by h > 0.  Outputs and their layouts are those of riqn_dueling_bwd / riqn_dueling_bwd_bf16. */
int riqn_dueling_bwd_dense(long rows, int batch, int hidden, int action_space, const float* h, const float* wz,
                           const float* grad_q, float* dh, float* dz, void* dz_bf16, void* stream);
int riqn_dueling_bwd_dense_bf16(long rows, int batch, int hidden, int action_space, const float* h, const void* h_bf16,
                                const float* wz, const float* grad_q, void* dh_hi, void* dh_hi_t, float* dh_colsum,
                                float* dz, void* dz_bf16, void* stream);
/* Parameter gradients of the two z-layers (accumulated): dwz_scratch 32*2*hidden floats, dbz_scratch 32.
 * 1 <= action_space <= 31, else cudaErrorInvalidValue and nothing is written. */
/* Same with the reduction dz^T h on the tensor cores, straight from the row-major bf16 images dz_bf16 (rows, 32) and
 * h_bf16 (rows, 2*hidden) (rows % 8 == 0). */
int riqn_z_wgrad_tc(long rows, int hidden, int action_space, const void* dz_bf16, const void* h_bf16, const float* dz,
                    float* dwz_scratch, float* dbz_scratch, const float* eps_w_zv, const float* eps_b_zv,
                    const float* eps_w_za, const float* eps_b_za, float* g_mu_zv, float* g_sig_zv, float* g_bmu_zv,
                    float* g_bsig_zv, float* g_mu_za, float* g_sig_za, float* g_bmu_za, float* g_bsig_za, void* stream);
int riqn_z_wgrad(long rows, int hidden, int action_space, const float* dz, const float* h, float* dwz_scratch,
                 float* dbz_scratch, const float* eps_w_zv, const float* eps_b_zv, const float* eps_w_za,
                 const float* eps_b_za, float* g_mu_zv, float* g_sig_zv, float* g_bmu_zv, float* g_bsig_zv,
                 float* g_mu_za, float* g_sig_za, float* g_bmu_za, float* g_bsig_za, void* stream);

/* ------------------------------------------------------------------------------------------------
 * IQN loss                                     replaces rainbowiqn/compute_loss_iqn.py:216-358
 * ---------------------------------------------------------------------------------------------- */
/* a_star[b] = argmax_a mean_k q[k*batch+b, a]            (compute_loss_iqn.py:238-245)
 * The mean is the fp32 sum over k ascending divided once by num_quantiles; the first maximal index wins.  Returns
 * cudaErrorInvalidValue, writing nothing, unless batch >= 1, num_quantiles >= 1 and 1 <= action_space <= 32. */
int riqn_argmax_mean(int batch, int num_quantiles, int action_space, const float* q, long long* a_star, void* stream);
/* Fused n-step target + pairwise quantile-Huber loss and its gradient (compute_loss_iqn.py:262-357):
 *   target[b,j] = returns[b] + gamma_n*nonterminals[b]*q_target[j*batch+b, a_star[b]]
 *   theta[b,i]  = q_online[i*batch+b, actions[b]]
 *   loss[b]     = mean_j sum_i |tau[i*batch+b] - 1{d<0}| huber_kappa(d)/kappa ,  d = target_j - theta_i
 *   dtheta[i*batch+b] = d loss[b] / d theta[b,i]
 * theta_out (batch, n_tau) / target_out (batch, n_tau_prime) are optional debug outputs (may be NULL).
 * Returns cudaErrorInvalidValue, writing nothing, unless batch, n_tau, n_tau_prime >= 1, 1 <= action_space <= 32, kappa
 * is finite and > 0, and (n_tau_prime + 32) * 4 <= 48 KB (the staged targets).  riqn_iqn_loss_fwd_bwd_h and
 * riqn_miqn_loss_fwd_bwd take the same limits, the latter less its kernel's static shared memory (1 KB on sm_90a). */
int riqn_iqn_loss_fwd_bwd(int batch, int n_tau, int n_tau_prime, int action_space, const float* q_online,
                          const float* q_target, const float* tau, const long long* actions, const long long* a_star,
                          const float* returns, const float* nonterminals, float gamma_n, float kappa, float* loss,
                          float* dtheta, float* theta_out, float* target_out, void* stream);
/* Munchausen-IQN (Vieillard, Pietquin & Geist 2020): the same loss and gradient against a soft, entropy-regularised target
 * with a clipped log-policy bonus, in place of the double-DQN one.  q_target is ONE target-network pass over the stacked
 * frames [next_states; states] with n_tau_prime * 2 * batch rows: row j*2*batch + b is s_{t+n}, row j*2*batch + batch + b
 * is s_t of transition b.  With te = entropy_tau:
 *   qbar'(a) = mean_j q_target[j*2*batch+b, a] ,  qbar(a) = mean_j q_target[j*2*batch+batch+b, a]     (j ascending)
 *   l'(a)    = qbar'(a) - max qbar' - te * ln sum_a exp((qbar'(a) - max qbar') / te)   (a ascending; l from qbar likewise)
 *   pi'(a)   = exp((qbar'(a) - max qbar') / te) / sum_a exp((qbar'(a) - max qbar') / te)
 *   bonus[b] = alpha * min(max(l(actions[b]), l0), 0)
 *   target[b,j] = returns[b] + bonus[b] + gamma_n*nonterminals[b] * sum_a pi'(a) (q_target[j*2*batch+b, a] - l'(a))
 *   theta, loss, dtheta as in riqn_iqn_loss_fwd_bwd.
 * The bonus also enters on terminal transitions.  The log-policy is never formed as log(pi): an underflowing pi gives a
 * finite, very negative l, which the clip takes to l0.  bonus_out (batch), like theta_out / target_out, may be NULL.
 * Returns cudaErrorInvalidValue (and writes nothing) outside the limits of riqn_iqn_loss_fwd_bwd, for entropy_tau <= 0,
 * l0 > 0, alpha < 0, or any of the three non-finite. */
int riqn_miqn_loss_fwd_bwd(int batch, int n_tau, int n_tau_prime, int action_space, const float* q_online,
                           const float* q_target, const float* tau, const long long* actions, const float* returns,
                           const float* nonterminals, float gamma_n, float kappa, float alpha, float entropy_tau, float l0,
                           float* loss, float* dtheta, float* theta_out, float* target_out, float* bonus_out, void* stream);
/* CQL (Kumar, Zhou, Tucker & Levine 2020): riqn_iqn_loss_fwd_bwd's loss plus alpha times the log-sum-exp gap of the
 * online pass.  Per transition b, with N = n_tau and a_t = actions[b]:
 *   Q_a      = fl(S_a / N),  S_a = fp32 sum over i ascending of q_online[i*batch+b, a]   (riqn_argmax_mean's mean)
 *   lse      = m + log(sum_a exp(Q_a - m)),  m = max_a Q_a                 (double, a ascending, no atomics)
 *   pi[b,a]  = fl(exp(Q_a - lse))              (batch, A)   the softmax of the means
 *   gap[b]   = fl(lse - Q_{a_t}) >= 0
 *   td_loss[b], dtheta, theta_out, target_out  bit for bit those of riqn_iqn_loss_fwd_bwd on the same inputs
 *   loss[b]  = fl(td_loss[b] + fl(alpha * gap[b]))
 * dtheta is the gradient of td_loss alone: the gap's, (alpha / N)(pi[b,a] - 1{a = a_t}) on every row i*batch + b, is
 * dense over actions and riqn_cql_dense_grad folds it in.  gap, theta_out and target_out may be NULL.  Returns
 * cudaErrorInvalidValue, writing nothing, outside the limits of riqn_iqn_loss_fwd_bwd, unless alpha is finite and > 0,
 * or when loss, td_loss, pi or dtheta is NULL. */
int riqn_cql_loss_fwd_bwd(int batch, int n_tau, int n_tau_prime, int action_space, const float* q_online,
                          const float* q_target, const float* tau, const long long* actions, const long long* a_star,
                          const float* returns, const float* nonterminals, float gamma_n, float kappa, float alpha,
                          float* loss, float* td_loss, float* pi, float* dtheta, float* gap, float* theta_out,
                          float* target_out, void* stream);
/* riqn_cql_loss_fwd_bwd against riqn_iqn_loss_fwd_bwd_h's transformed target; the gap is taken on the h-space outputs.
 * Its limits, and eps finite and >= 0. */
int riqn_cql_loss_fwd_bwd_h(int batch, int n_tau, int n_tau_prime, int action_space, const float* q_online,
                            const float* q_target, const float* tau, const long long* actions, const long long* a_star,
                            const float* returns, const float* nonterminals, float gamma_n, float kappa, float alpha,
                            float eps, float* loss, float* td_loss, float* pi, float* dtheta, float* gap,
                            float* theta_out, float* target_out, void* stream);
/* The dense upstream gradient grad_q (n*batch, A), quantile-major, of sum_b gscale[b]*gscale_mul*loss[b] at the CQL loss,
 * from its dtheta (n*batch) and pi (batch, A), every operation rounded on its own:
 *   w_b = fl(gscale[b] * gscale_mul),  c = fl(alpha / n),  g = fl(c * pi[b,a])
 *   grad_q[i*batch+b, a] = fl(w_b * g)                                  for a != actions[b]
 *                        = fl(w_b * fl(dtheta[i*batch+b] + fl(g - c)))   for a == actions[b]
 * for riqn_dueling_bwd_dense / riqn_qr_head_bwd_dense.  Returns cudaErrorInvalidValue, writing nothing, unless batch, n >= 1,
 * 1 <= action_space <= 32, alpha is finite and > 0 and no pointer is NULL. */
int riqn_cql_dense_grad(int batch, int n, int action_space, const float* dtheta, const float* pi, const long long* actions,
                        const float* gscale, float gscale_mul, float alpha, float* grad_q, void* stream);
/* DQfD (Hester et al. 2018): riqn_iqn_loss_fwd_bwd's loss plus lambda times the large-margin imitation loss on the rows
 * flagged as demonstrations.  Per transition b, with N = n_tau, a_E = actions[b] and l = margin:
 *   Q_a      = fl(S_a / N),  S_a = fp32 sum over i ascending of q_online[i*batch+b, a]   (riqn_argmax_mean's mean)
 *   v_a      = Q_a for a = a_E,  fl(Q_a + l) otherwise
 *   a_hat[b] = the first a (ascending) with v_a = M,  M = max_a v_a
 *   margin_out[b] = J = fl(M - Q_{a_E}) >= 0
 *   td_loss[b], dtheta, theta_out, target_out  bit for bit those of riqn_iqn_loss_fwd_bwd on the same inputs
 *   loss[b]  = fl(td_loss[b] + fl(lambda * J)) if demo[b] != 0, else td_loss[b]
 * demo: (batch,) flags, or NULL for no demonstration.  dtheta is the gradient of td_loss alone: J's, (1/N)(1{a = a_hat}
 * - 1{a = a_E}) on every row i*batch + b of a flagged transition, is folded in by riqn_dqfd_dense_grad.  margin_out,
 * theta_out and target_out may be NULL.  Returns cudaErrorInvalidValue, writing nothing, outside the limits of
 * riqn_iqn_loss_fwd_bwd, unless margin and lambda are finite and > 0, or when loss, td_loss, a_hat or dtheta is NULL. */
int riqn_dqfd_loss_fwd_bwd(int batch, int n_tau, int n_tau_prime, int action_space, const float* q_online,
                           const float* q_target, const float* tau, const long long* actions, const long long* a_star,
                           const float* returns, const float* nonterminals, const unsigned char* demo, float gamma_n,
                           float kappa, float margin, float lambda, float* loss, float* td_loss, float* dtheta,
                           float* margin_out, long long* a_hat, float* theta_out, float* target_out, void* stream);
/* riqn_dqfd_loss_fwd_bwd against riqn_iqn_loss_fwd_bwd_h's transformed target; the margin is taken on the h-space outputs,
 * in h-space units.  Its limits, and eps finite and >= 0. */
int riqn_dqfd_loss_fwd_bwd_h(int batch, int n_tau, int n_tau_prime, int action_space, const float* q_online,
                             const float* q_target, const float* tau, const long long* actions, const long long* a_star,
                             const float* returns, const float* nonterminals, const unsigned char* demo, float gamma_n,
                             float kappa, float margin, float lambda, float eps, float* loss, float* td_loss,
                             float* dtheta, float* margin_out, long long* a_hat, float* theta_out, float* target_out,
                             void* stream);
/* The dense upstream gradient grad_q (n*batch, A), quantile-major, of sum_b gscale[b]*gscale_mul*loss[b] at the DQfD loss,
 * from its dtheta (n*batch) and a_hat (batch), every operation rounded on its own; zero in every column not named:
 *   w_b = fl(gscale[b] * gscale_mul),  c = fl(lambda / n)
 *   demo NULL, demo[b] == 0 or a_hat[b] == actions[b]:  grad_q[i*batch+b, actions[b]] = fl(w_b * dtheta[i*batch+b])
 *   otherwise:  grad_q[i*batch+b, a_hat[b]] = fl(w_b * c),  grad_q[i*batch+b, actions[b]] = fl(w_b * fl(dtheta - c))
 * for riqn_dueling_bwd_dense / riqn_qr_head_bwd_dense.  Returns cudaErrorInvalidValue, writing nothing, unless batch, n >= 1,
 * 1 <= action_space <= 32, lambda is finite and > 0 and no pointer but demo is NULL. */
int riqn_dqfd_dense_grad(int batch, int n, int action_space, const float* dtheta, const long long* a_hat,
                         const long long* actions, const unsigned char* demo, const float* gscale, float gscale_mul,
                         float lambda, float* grad_q, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Value-function rescaling (Pohlen et al. 2018, the transformed Bellman operator; no counterpart in the reference)
 *   h(x) = sign(x) (sqrt(|x| + 1) - 1) + eps x, evaluated in double in the cancellation-free forms
 *   h(x):     a = |x|;  m = a / (sqrt(a + 1) + 1);  h = copysign(m, x) + eps x
 *   h^-1(y):  a = |y|;  u = (a + 1) + eps;  s = sqrt(1 + (4 eps) u);  d = ((4u) a) / (((2u - 1) + s) (s + 1));
 *             h^-1 = copysign(d (d + 2), y)
 * with every operation rounded on its own (no FMA), eps the float argument widened to double, and each stored value
 * rounded once to float.  Every entry point below returns cudaErrorInvalidValue, writing nothing, for eps < 0 or
 * non-finite, and for the limits it names.
 * ---------------------------------------------------------------------------------------------- */
/* out[i] = fl(h(x[i])) (inverse == 0) or fl(h^-1(x[i])) (inverse == 1), i < n.  out must not be NULL. */
int riqn_value_rescale(long n, const float* x, float eps, int inverse, float* out, void* stream);
/* riqn_iqn_loss_fwd_bwd against the transformed target, with g = fl(gamma_n * nonterminals[b]) as there:
 *   target[b,j] = fl(h(returns[b] + g * h^-1(q_target[j*batch+b, a_star[b]])))     (sum and product in double)
 * theta, loss and dtheta as in riqn_iqn_loss_fwd_bwd, and its limits. */
int riqn_iqn_loss_fwd_bwd_h(int batch, int n_tau, int n_tau_prime, int action_space, const float* q_online,
                            const float* q_target, const float* tau, const long long* actions, const long long* a_star,
                            const float* returns, const float* nonterminals, float gamma_n, float kappa, float eps,
                            float* loss, float* dtheta, float* theta_out, float* target_out, void* stream);
/* The expected return on the original scale of h-space quantiles q (n*batch, A), quantile-major, and its argmax:
 *   values[b,a] = fl(sum_k w[k*batch+b] * h^-1(q[k*batch+b, a]))   (FQF: w = dtau)
 *   values[b,a] = fl((sum_k h^-1(q[k*batch+b, a])) / n)             (w == NULL: IQN's mean over K fractions)
 * summed in double over k ascending; a_star[b] = argmax_a values[b,a] on the rounded values, the first maximal index
 * winning.  values (batch, A) and a_star (batch) may each be NULL, not both.  batch, n >= 1, 1 <= action_space <= 32. */
int riqn_argmax_expected_h(int batch, int n, int action_space, const float* q, const float* w, float eps, float* values,
                           long long* a_star, void* stream);

/* ------------------------------------------------------------------------------------------------
 * FQF: fraction proposal network (Yang et al., NeurIPS 2019; no counterpart in the reference)
 * The proposal's logits (batch, n) = feat W_f^T + b_f come from riqn_linear_fwd_ld (split-1 fp32 store, deterministic).
 * Every entry point below takes 2 <= n <= 256 (and 1 <= action_space <= 32, batch >= 1) and returns
 * cudaErrorInvalidValue, writing nothing, for anything else.
 * ---------------------------------------------------------------------------------------------- */
/* P = softmax(logits[b, :]), max-shifted, e_k = exp(l_k - max l) in double.  The cumulative sums c_i = sum_{k<i} e_k are
 * formed in double with k ascending (one sequential sum per sample) and rounded once:
 *   tau[b, 0] = 0, tau[b, i] = fl(c_i / c_n) (i = 1..n-1), tau[b, n] = 1 exactly      (batch, n+1), non-decreasing
 *   tau_hat[i*batch + b] = (tau[b,i] + tau[b,i+1]) / 2, dtau[i*batch + b] = tau[b,i+1] - tau[b,i]   (quantile-major, fp32)
 *   entropy[b] (may be NULL) = -sum_k P_k log P_k, formed as log c_n - sum_k (e_k / c_n)(l_k - max l) in double.
 * A P_k that underflows float gives dtau == 0, never NaN. */
int riqn_fqf_fractions(int batch, int n, const float* logits, float* tau, float* tau_hat, float* dtau, float* entropy,
                       void* stream);
/* Backward of the fraction loss with the quantile values detached.  q_hat (n*batch, A) is the pass at tau_hat, q_bnd
 * ((n-1)*batch, A; more rows are allowed and ignored) the pass at the inner boundaries tau_1..tau_{n-1}, both
 * quantile-major; with F(.) the value of action a = actions[b] and w = gscale[b] * gscale_mul (gscale may be NULL: 1):
 *   g_i       = 2 F(tau_i) - F(tau_hat_i) - F(tau_hat_{i-1})             i = 1..n-1 (dW1/dtau_i, FQF Proposition 1)
 *   loss[b]   = sum_i g_i tau_i - entropy_coef * H(P)                    (loss_out, unweighted; may be NULL)
 *   G_k       = sum_{i>k} g_i                                            (dL/dP_k, k descending)
 *   dlogits[b, k] = w * (P_k (G_k - sum_m P_m G_m) + entropy_coef * P_k (log P_k + H))
 * All sums in double in the stated order, P recomputed from logits exactly as riqn_fqf_fractions does.  entropy_coef must
 * be finite and >= 0, gscale_mul finite. */
int riqn_fqf_fraction_bwd(int batch, int n, int action_space, const float* logits, const float* tau, const float* q_hat,
                          const float* q_bnd, const long long* actions, const float* gscale, float gscale_mul,
                          float entropy_coef, float* dlogits, float* loss_out, void* stream);
/* grad_w (n, feat_dim) += dlogits^T feat, grad_b (n) += sum_b dlogits[b, :]: each element is one fp32 fmaf chain over b
 * ascending, then added once.  No atomics.  The fraction layer's form of riqn_linear_wgrad (same kernel), with its
 * 2 <= n <= 256. */
int riqn_fqf_fraction_wgrad(int batch, int n, int feat_dim, const float* dlogits, const float* feat, float* grad_w,
                            float* grad_b, void* stream);
/* Generic linear-layer weight gradient: grad_w (n, feat_dim) += dy^T x, grad_b (n) += sum_b dy[b, :], dy (batch, n) and
 * x (batch, feat_dim) row-major, rounded exactly as riqn_fqf_fraction_wgrad.  Any n >= 1 (CURL's projection: 512 and 128);
 * batch >= 1, feat_dim >= 1 and non-NULL pointers, else cudaErrorInvalidValue with nothing written. */
int riqn_linear_wgrad(int batch, int n, int feat_dim, const float* dy, const float* x, float* grad_w, float* grad_b,
                      void* stream);
/* a_star[b] = argmax_a sum_k w[k*batch+b] * q[k*batch+b, a]: fp32 fmaf chain over k ascending, the first maximal index
 * winning (as riqn_argmax_mean).  FQF's Q(s, a) = sum_i dtau_i F(s, tau_hat_i, a). */
int riqn_argmax_weighted(int batch, int n, int action_space, const float* q, const float* w, long long* a_star,
                         void* stream);

/* ------------------------------------------------------------------------------------------------
 * Rainbow-only (C51) head and loss           replaces rainbowiqn/model.py:120-129, rainbowiqn/agent.py:77-141
 * ---------------------------------------------------------------------------------------------- */
/* zv (batch, atoms), za (batch, A*atoms) -> q = v + a - mean_a a; p / logp (batch, A, atoms) = (log_)softmax over
 * atoms (either may be NULL); a_star (may be NULL) = argmax_a sum_j support[j] p[b,a,j], the first maximal index
 * winning (agent.py:92-99).  atoms <= 64, else cudaErrorInvalidValue before anything is written. */
int riqn_c51_head_fwd(int batch, int action_space, int atoms, const float* zv, const float* za, const float* support,
                      float* p, float* logp, long long* a_star, void* stream);
/* Bellman projection of p_target[b, a_star[b], :] onto the support (agent.py:104-133, incl. the l == u fix),
 * loss[b] = -sum_j m_j logp_online[b, actions[b], j] (agent.py:141) and dq (batch, atoms) = dloss/dq[b, actions[b], :].
 * The projection index b_j = (clamp(tz_j, v_min, v_max) - v_min) / delta_z is clamped to atoms - 1 as well: fp32
 * rounding can take it just above (v_min = -1, v_max = 1, 62 atoms), where the reference's index_add_ writes the next
 * sample's atom 0.  With the clamp sum_j m_j = sum_j p_target[b, a_star[b], j].  m_out (batch, atoms) optional. */
int riqn_c51_loss_fwd_bwd(int batch, int action_space, int atoms, const float* logp_online, const float* p_target,
                          const long long* actions, const long long* a_star, const float* returns,
                          const float* nonterminals, const float* support, float gamma_n, float v_min, float v_max,
                          float delta_z, float* loss, float* dq, float* m_out, void* stream);
/* riqn_c51_loss_fwd_bwd with the transformed Bellman target (value rescaling, see riqn_value_rescale): each atom moves to
 *   tz_j = fl(h(returns[b] + g * h^-1(support[j])))     g = fl(nonterminals[b] * gamma_n), sum and product in double
 * before the clamp to [v_min, v_max]; the index, the l == u fix, the projection, loss and dq follow as there.  support is
 * the h-space support.  atoms <= 64; eps as for riqn_value_rescale. */
int riqn_c51_loss_fwd_bwd_h(int batch, int action_space, int atoms, const float* logp_online, const float* p_target,
                            const long long* actions, const long long* a_star, const float* returns,
                            const float* nonterminals, const float* support, float gamma_n, float v_min, float v_max,
                            float delta_z, float eps, float* loss, float* dq, float* m_out, void* stream);
/* dzv (batch, atoms), dza (batch, A*atoms) from dq scaled by gscale[b] (dueling backward). */
int riqn_c51_head_bwd(int batch, int action_space, int atoms, const float* dq, const float* gscale, float gscale_mul,
                      const long long* actions, float* dzv, float* dza, void* stream);
/* The same for a dense upstream gradient grad_out = dL/dout (batch, A, atoms) of the head's output out = p (is_log == 0)
 * or log p (is_log != 0) as riqn_c51_head_fwd wrote it:  log: dq = grad_out - p * sum_atoms grad_out ;
 * softmax: dq = p * (grad_out - sum_atoms p grad_out) ; then dzv[b,j] = sum_a dq[b,a,j], dza[b,a,j] = dq[b,a,j] - dzv[b,j]/A.
 * atoms <= 64. */
int riqn_c51_head_bwd_dense(int batch, int action_space, int atoms, const float* out, const float* grad_out, int is_log,
                            float* dzv, float* dza, void* stream);

/* ------------------------------------------------------------------------------------------------
 * QR-DQN head (Dabney, Rowland, Bellemare & Munos, AAAI 2018; no counterpart in the reference)
 * The C51-shaped z-layers zv (batch, n), za (batch, A*n) give n quantile values per action at the fixed fractions
 * tau_hat_i = (2i+1)/(2n); q is written quantile-major (n*batch, A), row i*batch + b, as the IQN head writes it, so the
 * quantile-Huber loss, riqn_argmax_mean and riqn_argmax_expected_h read it unchanged.  Every entry point below returns
 * cudaErrorInvalidValue, writing nothing, unless 2 <= n <= 256, 1 <= action_space <= 32 and batch >= 1.  No atomics:
 * each output element is computed by one thread in the stated order.
 * ---------------------------------------------------------------------------------------------- */
/* The dueling sum per quantile, with every operation rounded to fp32 on its own:
 *   s_i = sum_a za[b, a*n + i]                         (fp32 adds, a ascending, starting from 0)
 *   q[(i*batch + b)*A + a] = fl(fl(zv[b,i] + za[b, a*n + i]) - fl(s_i / A)) */
int riqn_qr_head_fwd(int batch, int action_space, int n, const float* zv, const float* za, float* q, void* stream);
/* Backward of the loss kernel's one-hot gradient dL/dq[i*batch+b, a] = 1{a == actions[b]} dtheta[i*batch+b] w_b,
 * w_b = fl(gscale[b] * gscale_mul) (gscale may be NULL: w_b = gscale_mul), with dtheta (n*batch) quantile-major as
 * riqn_iqn_loss_fwd_bwd writes it.  Rounded as riqn_c51_head_bwd on dq[b, i] = dtheta[i*batch+b] (bit for bit):
 *   g = fl(dtheta[i*batch+b] * w_b) ;  dzv[b,i] = g ;  dza[b, a*n+i] = fl(g * fl(1{a == actions[b]} - fl(1 / A))) */
int riqn_qr_head_bwd(int batch, int action_space, int n, const float* dtheta, const float* gscale, float gscale_mul,
                     const long long* actions, float* dzv, float* dza, void* stream);
/* Backward of a dense G = dL/dq (n*batch, A), quantile-major:
 *   dzv[b,i] = sum_a G[i*batch+b, a]   (fp32 adds, a ascending, starting from 0)
 *   dza[b, a*n+i] = fl(G[i*batch+b, a] - fl(dzv[b,i] / A)) */
int riqn_qr_head_bwd_dense(int batch, int action_space, int n, const float* grad_q, float* dzv, float* dza, void* stream);

/* ------------------------------------------------------------------------------------------------
 * MMDQN loss (Nguyen-Tang, Gupta & Venkatesh, AAAI 2021; no counterpart in the reference) on the QR-DQN head's
 * particles, with g = fl(gamma_n * nonterminals[b]) and a* = a_star[b] as in riqn_iqn_loss_fwd_bwd:
 *   theta_i = q_online[i*batch + b, actions[b]] ,  T_j = fl(returns[b] + fl(g * q_target[j*batch + b, a*]))
 *   k(x, y) = sum_h exp(-(x - y)^2 / h)      over the n_bandwidths bandwidths h
 *   loss[b] = max(0, (1/n^2) sum_i sum_j [k(theta_i, theta_j) + k(T_i, T_j) - 2 k(theta_i, T_j)])
 *   dtheta[i*batch + b] = (2/n^2) sum_j [k1(theta_i, theta_j) - k1(theta_i, T_j)],
 *                         k1(x, y) = -sum_h (2 (x - y) / h) exp(-(x - y)^2 / h)   (gradient of the unclamped sum)
 * dtheta is quantile-major (n*batch), as riqn_qr_head_bwd takes it; theta_out (batch, n) and target_out (batch, n) are
 * optional (NULL: not written).  `bandwidths` is a HOST array of n_bandwidths floats, read during the call: the kernel
 * receives the constants c_h = fl(-log2(e) / h) and w_h = fl(2 / h) by value (a captured graph holds them) and evaluates
 * exp(-(x - y)^2 / h) as exp2f(fl(fl(d * d) * c_h)), d = fl(x - y).  The sums are grouped per (i, j) bracket, j ascending,
 * so T_j = theta_j for every j gives loss 0 and dtheta 0 exactly.  One CTA per transition, no atomics.  Returns
 * cudaErrorInvalidValue, writing nothing, unless batch >= 1, 1 <= n <= 256, 1 <= action_space <= 32,
 * 1 <= n_bandwidths <= 16 and every bandwidth is finite and > 0 with finite c_h and w_h. */
int riqn_mmd_loss_fwd_bwd(int batch, int n, int action_space, const float* q_online, const float* q_target,
                          const long long* actions, const long long* a_star, const float* returns,
                          const float* nonterminals, float gamma_n, int n_bandwidths, const float* bandwidths,
                          float* loss, float* dtheta, float* theta_out, float* target_out, void* stream);
/* riqn_mmd_loss_fwd_bwd against the transformed target, as riqn_iqn_loss_fwd_bwd_h forms it:
 *   T_j = fl(h(returns[b] + g * h^-1(q_target[j*batch + b, a*])))     (sum and product in double)
 * eps must be finite and >= 0. */
int riqn_mmd_loss_fwd_bwd_h(int batch, int n, int action_space, const float* q_online, const float* q_target,
                            const long long* actions, const long long* a_star, const float* returns,
                            const float* nonterminals, float gamma_n, int n_bandwidths, const float* bandwidths,
                            float eps, float* loss, float* dtheta, float* theta_out, float* target_out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * HL-Gauss loss (Farebrother et al., ICML 2024; Imani & White, ICML 2018; no counterpart in the reference) on the C51
 * head: cross-entropy against the Gaussian histogram of the scalar double-DQN target.  Operands as riqn_c51_loss_fwd_bwd
 * (logp_online and p_target (batch, A, atoms), a* = a_star[b]); every double operation is rounded on its own:
 *   g  = fl(nonterminals[b] * gamma_n) ;  Q' = sum_j fl64(p_target[b, a*, j] * support[j])   (double, j ascending, from 0)
 *   y  = clamp(returns[b] + g * Q', v_min, v_max)            (double) ;  target_out[b] = fl32(y)
 *   D  = (v_max - v_min) / (atoms - 1) ;  e_i = v_min + (i - 0.5) * D ;  u_i = (e_i - y) / s ,  s = (sigma_ratio * D) * sqrt(2)
 *   c_i = 0.5 * erfc(|u_i|)   (i = 0..atoms) ;  mass_j = c_j - c_j+1 if u_j >= 0, c_j+1 - c_j if u_j+1 <= 0, else
 *   (0.5 - c_j) + (0.5 - c_j+1) ;  m_j = fl32(mass_j / ((0.5 - c_0) + (0.5 - c_atoms)))
 *   loss[b] = -sum_j fl(m_j * logp_online[b, actions[b], j])   (fp32, lanes 0..31 and 32..63 by the warp_sum butterfly,
 *             then (0 + warp 0) + warp 1) ;  mt = sum_j m_j in the same order
 *   dq[b, j] = -fl(m_j - fl(p_j * mt)) ,  p_j = fl32(exp(double logp_online[b, actions[b], j]))
 * dq (batch, atoms) is the gradient riqn_c51_head_bwd takes; m_out (batch, atoms) and target_out (batch) are optional
 * (NULL: not written).  One CTA of 64 threads per transition, no atomics.  Returns cudaErrorInvalidValue, writing
 * nothing, unless batch >= 1, action_space >= 1, 2 <= atoms <= 64, v_min and v_max are finite with v_min < v_max, and
 * sigma_ratio (sigma in bin widths) is finite with 0 < sigma_ratio <= 1000. */
int riqn_hl_gauss_loss_fwd_bwd(int batch, int action_space, int atoms, const float* logp_online, const float* p_target,
                               const long long* actions, const long long* a_star, const float* returns,
                               const float* nonterminals, const float* support, float gamma_n, float v_min, float v_max,
                               float sigma_ratio, float* loss, float* dq, float* m_out, float* target_out, void* stream);
/* riqn_hl_gauss_loss_fwd_bwd with the transformed target (value rescaling): support is the h-space support, and
 *   Q' = sum_j fl64(p_target[b, a*, j] * h^-1(support[j])) ,  y = clamp(h(returns[b] + g * Q'), v_min, v_max)
 * (the expectation on the linear scale, the quantity a* is chosen on).  eps as for riqn_value_rescale. */
int riqn_hl_gauss_loss_fwd_bwd_h(int batch, int action_space, int atoms, const float* logp_online,
                                 const float* p_target, const long long* actions, const long long* a_star,
                                 const float* returns, const float* nonterminals, const float* support, float gamma_n,
                                 float v_min, float v_max, float sigma_ratio, float eps, float* loss, float* dq,
                                 float* m_out, float* target_out, void* stream);
/* n floats <- 0 (the gradient arena's zero_grad, learner.py:22): cudaMemsetAsync on the caller's stream. */
int riqn_zero_f32(float* p, long n, void* stream);
/* grad[i] = 0 where act[i] <= 0. */
int riqn_relu_mask(long n, const float* act, float* grad, void* stream);
/* Strided fp32 linear-layer helpers for the small z-layers: y = x w^T + bias (optional ReLU); dx = dy w;
 * grad_mu += dy^T x, grad_sigma += (dy^T x) * weight_epsilon (split-K partials added in split order, no atomics:
 * bitwise reproducible). */
int riqn_linear_fwd_ld(long rows, int in_features, int out_features, const float* x, long ldx, const float* w,
                       const float* bias, float* y, long ldy, int relu, void* stream);
int riqn_linear_dgrad_ld(long rows, int in_features, int out_features, const float* dy, long lddy, const float* w,
                         float* dx, long lddx, void* stream);
int riqn_noisy_wgrad_ld(long rows, int in_features, int out_features, const float* dy, long lddy, const float* x, long ldx,
                        const float* weight_epsilon, float* grad_mu, float* grad_sigma, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Optimiser                              replaces torch.optim.Adam.step, agent.py:43 / learner.py:24
 * ---------------------------------------------------------------------------------------------- */
/* One Adam step over a flat arena of n fp32 parameters; `step` is the 1-based step count; grads are
 * multiplied by grad_scale first (1/world_size after a gradient all-reduce). */
int riqn_adam_step(long n, float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int step, float lr,
                   float beta1, float beta2, float eps, float grad_scale, const riqn_dyn_state* dyn, void* stream);
/* One AdamW step (torch.optim.AdamW, non-amsgrad): first params[i] = fl(params[i] * d) with d = fl32(1 - lr *
 * weight_decay) computed in double, then riqn_adam_step's update on the decayed params in the same pass (its bias
 * corrections read from dyn when dyn != NULL; d is always taken by value).  weight_decay = 0 gives riqn_adam_step's
 * bits.  n >= 1, step >= 1, non-NULL params / grads / exp_avg / exp_avg_sq, a finite weight_decay >= 0 and d in
 * (0, 1], else cudaErrorInvalidValue with nothing written. */
int riqn_adamw_step(long n, float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int step, float lr,
                    float beta1, float beta2, float eps, float weight_decay, float grad_scale, const riqn_dyn_state* dyn,
                    void* stream);

/* ------------------------------------------------------------------------------------------------
 * Prioritized replay: sum-tree          replaces RedisSegmentTree / ReplayRedisMemory, redis_memory.py
 * tree: 2*capacity-1 float64 nodes in HBM, leaf of data index d at d + capacity - 1.
 * ---------------------------------------------------------------------------------------------- */
/* Stratified sample values, one per segment of total/n, shuffled (redis_memory.py:276-287): value s is
 * a + (b - a) * u with a = s*seg, b = (s+1)*seg, seg = tree[0] / n, u = (((x << 32 | y) >> 11) + 0.5) * 2^-53 of the words
 * x, y of Philox draw s at stream_id (+ dyn->rng_offset when dyn != NULL); it goes to output slot rank(key_s), keys =
 * word x of the draws at stream_id ^ 0x5bd1e995, ties broken by s.  Returns cudaErrorInvalidValue, writing nothing,
 * unless 1 <= n <= 12000, or for a NULL tree or values. */
int riqn_sumtree_stratified(int n, unsigned long long seed, unsigned long long stream_id, const double* tree,
                            double* values, const riqn_dyn_state* dyn, void* stream);
/* Descent (_retrieve_multiple_values :205-229) + transform_to_valid_tree_indexes (:242-264) + priority
 * read (:315-321).  index_actor: per-actor write heads (int64).  Bit-exact with the reference.  Returns
 * cudaErrorInvalidValue, writing nothing, for capacity or actor_capacity < 1, a capacity that is not a multiple of
 * actor_capacity, history or n_step < 0, or a NULL pointer; n <= 0 does nothing. */
int riqn_sumtree_sample(int n, long capacity, int actor_capacity, const double* tree, const double* values,
                        const long long* index_actor, int history, int n_step, long long* tree_idx,
                        long long* data_idx, double* priorities, void* stream);
/* riqn_sumtree_sample with the valid-index shift at n_step = hz->n_step, read on the device (kept in 1..n_max): bit for
 * bit riqn_sumtree_sample at that n_step.  Returns cudaErrorInvalidValue, writing nothing, for the arguments
 * riqn_sumtree_sample refuses, n_max outside 1..RIQN_MAX_HORIZON or a NULL hz; n <= 0 does nothing. */
int riqn_sumtree_sample_horizon(int n, long capacity, int actor_capacity, const double* tree, const double* values,
                                const long long* index_actor, int history, int n_max, const riqn_horizon_state* hz,
                                long long* tree_idx, long long* data_idx, double* priorities, void* stream);
/* Importance-sampling weights (sample_byte :465-475); n_nonpositive (device int, may be NULL) counts the
 * priorities <= 0 that were replaced by 1/capacity (:446-456).  With dyn != NULL, dyn->is_capacity and dyn->is_beta
 * replace current_capacity and priority_weight.  Returns cudaErrorInvalidValue, writing nothing, for n < 1, a NULL
 * tree, priorities, w64 or w32, or (dyn == NULL) a current_capacity or priority_weight that is not finite and >= 0.
 * current_capacity 0 gives the reference's NaN weights ((0 * p)^-beta / max). */
int riqn_sumtree_is_weights(int n, const double* tree, const double* priorities, double current_capacity,
                            double priority_weight, double* w64, float* w32, int* n_nonpositive,
                            const riqn_dyn_state* dyn, void* stream);
/* update_priorities / update_multiple_value / _propagate_multiple_values (:557-573,139-151,94-105).
 * apply_pow != 0: new = np.power(loss, float32(priority_exponent)) first.  new_priorities (n floats) and
 * diff_scratch (n doubles) are outputs/workspace; *max_priority (device double) is raised if needed.
 * n <= 4096.  The tree arithmetic is bit-exact with the reference (including duplicated indices) given the
 * float32 priorities; the power itself is the correctly rounded float32 value, which numpy/libm powf only
 * approximates (<= 1 ulp apart, platform dependent).  Returns cudaErrorInvalidValue, writing nothing, for n > 4096,
 * capacity < 1 or a NULL pointer; n <= 0 does nothing. */
int riqn_sumtree_update(int n, long capacity, double* tree, const long long* tree_idx, const float* loss,
                        float priority_exponent, int apply_pow, float* new_priorities, double* diff_scratch,
                        double* max_priority, void* stream);
/* riqn_sumtree_update with DQfD's demonstration priority bonus eps_d (Hester et al. 2018): after the power, every entry
 * with tree_idx >= demo_leaf (the leaves of the demonstration segments) takes new = fl(new + bonus).  The diff, the
 * propagation (duplicates included) and max_priority are riqn_sumtree_update's on those priorities.  Returns
 * cudaErrorInvalidValue, writing nothing, unless bonus is finite and >= 0 and demo_leaf >= 0, and for the arguments
 * riqn_sumtree_update refuses. */
int riqn_sumtree_update_demo(int n, long capacity, double* tree, const long long* tree_idx, const float* loss,
                             float priority_exponent, int apply_pow, float* new_priorities, double* diff_scratch,
                             double* max_priority, long long demo_leaf, float bonus, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Prioritized replay: frame store            replaces the Redis hashes "transitions<i>" (:184-193)
 * ---------------------------------------------------------------------------------------------- */
/* Frame half of append_actor_buffer (:159-199): n consecutive transitions of one actor into its ring, slot
 * (start + i) % actor_capacity + id_actor * actor_capacity.  Returns cudaErrorInvalidValue, writing nothing, for
 * actor_capacity < 1, id_actor < 0, start outside [0, actor_capacity), n > actor_capacity (a slot written twice in one
 * launch) or a NULL pointer; n <= 0 does nothing. */
int riqn_replay_append(int n, int actor_capacity, int id_actor, int start, const unsigned char* frames,
                       const int* timestep, const int* action, const float* reward, const unsigned char* nonterminal,
                       unsigned char* s_frames, int* s_timestep, int* s_action, float* s_reward,
                       unsigned char* s_nonterminal, void* stream);
/* Transition assembly (:347-369, :479-541): window (batch, history+n_step, 84, 84) uint8 with blank frames
 * across episode boundaries; states = window[:, :history], next_states = window[:, n_step:].
 * gamma_pow: n_step doubles, discount**k.  Returns cudaErrorInvalidValue, writing nothing, for actor_capacity, history
 * or n_step < 1, history + n_step > 16, or a NULL pointer; batch <= 0 does nothing. */
int riqn_frame_gather(int batch, int actor_capacity, int history, int n_step, const long long* data_idx,
                      const unsigned char* s_frames, const int* s_timestep, const int* s_action, const float* s_reward,
                      const unsigned char* s_nonterminal, const double* gamma_pow, unsigned char* window,
                      long long* actions, float* returns, float* nonterminals, void* stream);
/* Transition assembly at this step's n = hz->n_step, read on the device (kept in 1..n_max): frames (batch, 2*history,
 * 84, 84) uint8 holds the states in frames[:, :history] and the next states in frames[:, history:], at offsets that do
 * not depend on n.  The slots, blank frames, float64 return sum_{k<n} hz->gamma_pow[k] r_{t+k}, actions and 0/1
 * nonterminals are riqn_frame_gather's at n_step = n (with gamma_pow = hz->gamma_pow), bit for bit, and the next states
 * its window[:, n:n+history]; discounts[b] = fl32(hz->gamma_n * nonterminals[b]), the per-transition bootstrap factor a
 * loss kernel takes in place of the nonterminals with gamma_n = 1.  Returns cudaErrorInvalidValue, writing nothing, for
 * actor_capacity, history or n_max < 1, history + n_max > 16, or a NULL pointer; batch <= 0 does nothing. */
int riqn_frame_gather_horizon(int batch, int actor_capacity, int history, int n_max, const long long* data_idx,
                              const unsigned char* s_frames, const int* s_timestep, const int* s_action,
                              const float* s_reward, const unsigned char* s_nonterminal, const riqn_horizon_state* hz,
                              unsigned char* frames, long long* actions, float* returns, float* nonterminals,
                              float* discounts, void* stream);
/* SPR's K-step sequence (Schwarzer et al., ICLR 2021): window (batch, history+K, 84, 84) uint8 with the slots and blank
 * frames of riqn_frame_gather at n_step = K (so window[:, :history] is its states, bit for bit), actions (batch, K) int64
 * a_t .. a_{t+K-1} as stored (actions[:, 0] is riqn_frame_gather's), and valid (batch, K) uint8: valid[b, k-1] = 1 iff
 * the last frame of s_{t+k} (window index history-1+k) is not blank and, with p the sampled position in its segment and
 * h = index_actor[segment] (read on the device), the distance (h - p) mod actor_capacity is not in 1..k (the walk
 * p+1 .. p+k never reaches the write head, past which lie an older episode or unwritten slots).  Returns
 * cudaErrorInvalidValue, writing nothing, for batch, actor_capacity, history or K < 1, history + K > 16, or a NULL
 * pointer. */
int riqn_sequence_gather(int batch, int actor_capacity, int history, int K, const long long* data_idx,
                         const long long* index_actor, const unsigned char* s_frames, const int* s_timestep,
                         const int* s_action, const unsigned char* s_nonterminal, unsigned char* window,
                         long long* actions, unsigned char* valid, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Tensor-core building blocks of the NoisyLinear products (wgmma + TMA; csrc/gemm_tc.cu).
 * ---------------------------------------------------------------------------------------------- */
/* fp32 (rows, cols) -> bf16 hi and lo = bf16(x - hi) (either may be NULL); hi_t / lo_t (may be NULL) receive the
 * transposed (cols, rows) copies the weight-gradient product consumes. */
int riqn_split_bf16(long rows, int cols, const float* src, void* hi, void* lo, void* hi_t, void* lo_t, int fp16, void* stream);
/* fp16 != 0: hi = fp16(x) and lo (or NULL) = bf16(x) instead (hi_t / lo_t must be NULL).  Returns cudaErrorInvalidValue,
 * writing nothing, for fp16 with hi NULL or hi_t / lo_t set, and for lo_t without hi_t. */
/* Several small splits in ONE launch (the per-step refresh of the noise-free weight images): for each job
 * out[r, c] = src[r, perm ? perm[c] : c] / div (div == 1: unscaled), written as hi / lo = bf16(x - hi) (lo, hi_t may be
 * NULL; hi_t is the transposed (cols, rows) hi image).  Same values as riqn_split_bf16 / riqn_split_bf16_scaled on a
 * column-permuted source.  jobs: HOST array of n_jobs <= 12. */
typedef struct riqn_split_job {
  const float* src;     /* (rows, cols) fp32 */
  const int* perm;      /* cols ints or NULL */
  int rows, cols;
  float div;
  void* hi;
  void* lo;
  void* hi_t;
} riqn_split_job;
int riqn_split_bf16_multi(int n_jobs, const riqn_split_job* jobs, void* stream);
/* C (+)= A B^T with A (M,K), B (N,K) row-major bf16, K % 8 == 0, fp32 accumulation in registers.  a_lo and b_lo
 * non-NULL select the split-bf16 x3 (fp32-faithful) product a_hi b_hi + a_hi b_lo + a_lo b_hi; b_lo alone selects the
 * split-2 product a_hi (b_hi + b_lo) (epilogue 0 only).  epilogue: 0 store, 1 relu(acc+bias[n]), 2 add into C,
 * 3 add into C and acc*eps[m,n] into out2 (NoisyLinear dmu / dsigma).  split_k > 1 needs 2 or 3: the splits' partial
 * products are added in split order, so the result does not depend on scheduling.
 * c_t_bf16 / c_bf16 (may be NULL; epilogue 1 only): bf16 transposed (N, M) / row-major (M, N) images of the result.
 * Returns cudaErrorInvalidValue, writing nothing, when: the epilogue is outside 0..3; split_k > 1 with epilogue 0 or 1
 * (whatever the SM count); a_lo without b_lo; split-2 with epilogue != 0; C is NULL or ldc < N; epilogue 1 with a NULL
 * bias or epilogue 3 with a NULL out2 or eps; c_bf16 not 16-byte aligned, with an epilogue other than 1, odd M or
 * N % 32 != 0; c_t_bf16 with an epilogue other than 1.  From N = 32 on, whole 32-column chunks leave as vectors, so
 * then also when: on epilogues 0 and 1, C is not 16-byte aligned or ldc % 4 != 0; the bias of epilogue 1 is not 16-byte
 * aligned; at even M, c_t_bf16 is not 4-byte aligned. */
int riqn_gemm_bf16_tc(int M, int N, int K, const void* a_hi, const void* a_lo, const void* b_hi, const void* b_lo,
                      float* c, long ldc, int epilogue, const float* bias, float* out2, const float* eps, int split_k,
                      void* c_t_bf16, void* c_bf16, int fmt, void* stream);
/* fmt (both GEMM entry points): 0 = both operand images hold bf16, 3 = both hold fp16 (single-pass: a_lo == b_lo == NULL).
 * 1 / 2 (mixed) are rejected: wgmma takes a single 16-bit format for A and B. */
/* Products whose B operand is (K, N) row-major bf16 (MN-major wgmma operand, N % 8 == 0) -- no transposed copies:
 *   a_is_km != 0: C (+)= A^T B with A (K, M) row-major (M % 8 == 0): the reduction runs over the ROWS of both, i.e. a
 *                 weight gradient dW = dY^T X straight from the row-major activations;
 *   a_is_km == 0: C (+)= A B with A (M, K) row-major (K % 8 == 0): a data gradient dX = dY W from the untransposed W.
 * epilogue 0 / 2 / 3 as above (2 adds alpha * acc into C; 0 and 3 need alpha == 1); single-bf16 product.  c_bf16 (may be
 * NULL; epilogue 0, N % 32 == 0, 16-byte aligned): write the result as bf16 (M, N) there INSTEAD of fp32 into c (c may
 * then be NULL).  Refused as riqn_gemm_bf16_tc, and besides when a_is_km != 0 and M % 8 != 0, when N % 8 != 0, when
 * a_is_km == 0 and K % 8 != 0 (a_is_km != 0: any K), for epilogue 1, and for alpha != 1 unless the epilogue is 2. */
int riqn_gemm_bf16_tc_mn(int M, int N, int K, const void* a, const void* b_kn, int a_is_km, float* c, long ldc, int epilogue,
                         float* out2, const float* eps, float alpha, int split_k, void* c_bf16, int fmt, void* stream);

/* ------------------------------------------------------------------------------------------------
 * CURL (Srinivas, Laskin & Abbeel, ICML 2020; no counterpart in the reference): contrastive auxiliary loss on the trunk
 * ---------------------------------------------------------------------------------------------- */
/* Bilinear InfoNCE of anchors z_a (batch, dim) against keys z_k (batch, dim) with W (dim, dim), all row-major fp32, and its
 * gradient with respect to z_a and W; the positive of anchor i is key i.  With s = fl(coef / batch):
 *   v_i = W^T z_a,i          v_i[q] = sum_p z_a[i,p] W[p,q]                   (fmaf chain, p ascending)
 *   l_ij = v_i . z_k,j                                                         (fmaf chain, q ascending)
 *   m_i = max_j l_ij ;  S_i = sum_j expf(l_ij - m_i)       (lane chains over j = lane + 32k, then the warp_sum butterfly)
 *   loss_rows[i] = fl(fl(m_i + logf(S_i)) - l_ii)                              (unscaled; the loss is s * sum_i)
 *   dl_ij = fl(s * fl(fl(expf(l_ij - m_i) * fl(1 / S_i)) - [i == j]))
 *   g_i[q] = sum_j dl_ij z_k[j,q]   (fmaf, j ascending) ;  dz_a[i,p] = sum_q W[p,q] g_i[q]   (fmaf, q ascending)
 *   dw[p,q] += sum_i z_a[i,p] g_i[q]                                           (fmaf chain over i ascending, added once)
 * logits_out (batch, batch) may be NULL.  Two launches (the row kernel, then the dW reduction), scratch from the stream's
 * pool, no atomics.  dim must be 128 and 2 <= batch <= 4096, coef finite, the other pointers non-NULL; otherwise
 * cudaErrorInvalidValue and nothing is written. */
int riqn_curl_infonce_fwd_bwd(int batch, int dim, const float* z_a, const float* z_k, const float* w, float coef,
                              float* loss_rows, float* dz_a, float* dw, float* logits_out, void* stream);
/* Row LayerNorm without affine parameters, eps = 1e-5, width 128 or 512 (one warp per row, lane l holding the elements
 * l + 32k; the sums are lane chains over k then the warp_sum butterfly), of the rows x, or of fl(x + bias[col]) when
 * bias (width) is non-NULL (the bias of a product whose epilogue has none):
 *   mean = fl(sum x / width) ;  d = fl(x - mean) ;  rstd = fl(1 / sqrtf(fl(sum d*d / width) + 1e-5)) ;  x_hat = fl(d * rstd)
 *   y = x_hat, or max(x_hat, 0) when relu != 0.
 * The backward takes the forward's INPUT x and recomputes x_hat bit for bit; with g = dy (relu: 0 where x_hat <= 0):
 *   dx = fl(rstd * fl(fl(g - mean(g)) - fl(x_hat * mean(g * x_hat)))).
 * rows >= 1 and non-NULL pointers, else cudaErrorInvalidValue with nothing written. */
int riqn_layernorm_fwd(long rows, int width, const float* x, const float* bias, int relu, float* y, void* stream);
int riqn_layernorm_bwd(long rows, int width, const float* x, const float* bias, const float* dy, int relu, float* dx,
                       void* stream);
/* out[c] += sum_r x[r, c] (rows, cols) row-major, in a fixed order (per-block partials added in block order; two
 * launches, no atomics): the bias gradient of a product on the tensor cores.  rows, cols >= 1 and non-NULL pointers,
 * else cudaErrorInvalidValue with nothing written. */
int riqn_colsum_add(long rows, int cols, const float* x, float* out, void* stream);
/* Momentum update xi[i] = fl(xi[i] + fl(tau * fl(theta[i] - xi[i]))), every operation rounded on its own (no fma).
 * n >= 1, finite 0 < tau <= 1, non-NULL pointers, else cudaErrorInvalidValue with nothing written. */
int riqn_ema_f32(long n, const float* theta, float* xi, float tau, void* stream);
/* out[i] = fl(a[i] + b[i]) (out may alias a or b).  n >= 1 and non-NULL pointers, else cudaErrorInvalidValue. */
int riqn_add_f32(long n, const float* a, const float* b, float* out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * SPR (Schwarzer et al., ICLR 2021; no counterpart in the reference): the transition model on the (B, 64, 7, 7) latent
 * runs on riqn_conv_fwd_strip / riqn_conv_bwd_strip with conv3's geometry (3x3, stride 1, pad 0, H = W = 9) over the
 * zero-bordered latent.
 * ---------------------------------------------------------------------------------------------- */
/* The A operand of that strip convolution: hi / lo (batch*81, channels) bf16 (lo = bf16(x - hi)), row (b, gy, gx) of
 * the 9x9 grid, column c: latent[b, c, gy-1, gx-1] for c < 64 inside the border; with channels = 128, also the one-hot
 * action planes, 1 at c = 64 + actions[b * action_stride] for 64 <= c < 64 + num_actions inside the border; 0 elsewhere
 * (an action outside 0..num_actions-1 sets no plane).  channels = 64 takes actions == NULL; channels = 128 a non-NULL
 * actions, 1 <= num_actions <= 64 and action_stride >= 1.  Otherwise cudaErrorInvalidValue with nothing written. */
int riqn_spr_pack(int batch, int channels, const float* latent, const long long* actions, int action_stride,
                  int num_actions, void* hi, void* lo, void* stream);
/* Adjoint of riqn_spr_pack's latent part: out (batch, 64, 7, 7) = fl(acc + din[:, :64, 1:8, 1:8]) element by element, or
 * the crop alone when acc is NULL; din (batch, channels, 9, 9) fp32 is riqn_conv_bwd_strip's data gradient.  out may
 * alias acc.  channels 64 or 128, non-NULL din / out, else cudaErrorInvalidValue. */
int riqn_spr_unpack_grad(int batch, int channels, const float* din, const float* acc, float* out, void* stream);
/* bf16 images of a 3x3 convolution weight w (cout, cin, 3, 3) fp32 zero-padded to cpad input channels: hi / lo
 * (cout, 9*cpad) in strip order, column (dy*3 + dx)*cpad + c (riqn_conv_fwd_strip's w_hi / w_lo), and hi_orig
 * (cout, cpad*9) in the original order c*9 + dy*3 + dx (riqn_conv_bwd_strip's w_hi).  1 <= cout <= 64,
 * 1 <= cin <= cpad, cpad % 64 == 0 and non-NULL pointers, else cudaErrorInvalidValue. */
int riqn_spr_weight_images(int cout, int cin, int cpad, const float* w, void* hi, void* lo, void* hi_orig, void* stream);
/* gw[o, c, s] = fl(gw[o, c, s] + gpad[o, c, s]) for c < cin: a padded weight gradient (cout, cpad, 9) into the
 * unpadded one (cout, cin, 9).  cout, cin >= 1, cin <= cpad, non-NULL pointers, else cudaErrorInvalidValue. */
int riqn_spr_weight_grad_add(int cout, int cin, int cpad, const float* gpad, float* gw, void* stream);
/* Masked negative cosine of predictions p = pred[k*rows + b] against targets t = target[k*rows + b] ((K, rows, dim)
 * fp32), its loss per sample and its gradient with respect to the predictions.  With s = fl(coef / rows), v =
 * valid[b*K + k] ((rows, K) uint8) and lanes l holding elements l + 32j (j = 0..3):
 *   P = sum p*p, T = sum t*t, Q = sum p*t       (lane chains of fl(fl(a*b) + acc) over j, then the warp_sum butterfly)
 *   |p| = sqrtf(P) ; np = max(|p|, 1e-12) ; nt = max(sqrtf(T), 1e-12) ; cos = fl(Q / fl(np * nt))
 *   loss_rows[b] = sum_k (v ? -cos : 0)          (k ascending; the loss is s * sum_b loss_rows[b])
 *   dpred = fl((v ? -s : 0) * fl(g / np)),  g = fl(fl(t / nt) - fl(cos * fl(p / np))) when |p| > 1e-12, else fl(t / nt)
 * i.e. the gradient of -s v cos(F.normalize(p), F.normalize(t)) with eps 1e-12 on both norms.  One CTA per sample, no
 * atomics.  dim must be 128, 1 <= K <= 12, 1 <= rows <= 4096, coef finite, the pointers non-NULL; otherwise
 * cudaErrorInvalidValue and nothing is written. */
int riqn_spr_cosine_fwd_bwd(int rows, int K, int dim, const float* pred, const float* target, const unsigned char* valid,
                            float coef, float* loss_rows, float* dpred, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Periodic network resets (SR-SPR, D'Oro et al. 2023; BBF, Schwarzer et al. 2023; no counterpart in the reference)
 * ---------------------------------------------------------------------------------------------- */
#define RIQN_RESET_MAX_SEGMENTS 64
#define RIQN_RESET_UNIFORM 0    /* fresh draw U(-value, value) */
#define RIQN_RESET_CONSTANT 1   /* fresh draw = value          */
typedef struct riqn_reset_segment {
  long long begin, end;   /* the arena elements [begin, end)                                       */
  int kind;               /* RIQN_RESET_UNIFORM or RIQN_RESET_CONSTANT                              */
  float value;            /* the uniform bound b, or the constant                                  */
  float alpha;            /* the share of the old value that is kept, 0 <= alpha < 1               */
} riqn_reset_segment;
/* Reset the segments `segs` (a HOST array of nseg, passed by value to one launch) of the fp32 arena params[0:n], and
 * restart its Adam moments: exp_avg[0:n] = exp_avg_sq[0:n] = 0 when both are non-NULL (both NULL: no moments).
 * Element i of a segment becomes
 *   u_i    = the (0,1) uniform riqn_fill_uniform(n, seed, stream_id, dyn = NULL) writes at position i (Philox4x32-10 word
 *            i % 4 of draw i / 4, x -> fl(fl((x >> 8) + 0.5) / 2^24));
 *   theta0 = fl(value * (2 u_i - 1)) for a uniform segment (2 u_i - 1 is exact in fp32), value for a constant one;
 *   theta' = fl(fl(alpha * theta) + fl(fl(1 - alpha) * theta0)), each operation rounded on its own (no fma);
 *            alpha = 0 writes theta0 itself (the same value for every finite theta; a non-finite theta is replaced too).
 * The draw depends on (seed, stream_id, i) only, not on the launch geometry.  Elements in no segment (alignment padding,
 * parameters a reset keeps) keep their bits.  Refused with cudaErrorInvalidValue, nothing written, when n < 1, params is
 * NULL, exactly one moment pointer is NULL, segs is NULL, nseg is not in 1..64, the segments are not sorted, disjoint
 * and non-empty inside [0, n) (0 <= begin < end <= n, begin >= the previous end), a kind is unknown, a uniform bound is
 * not finite and > 0, a constant is not finite, or an alpha is not in [0, 1). */
int riqn_arena_reset(long n, float* params, float* exp_avg, float* exp_avg_sq, int nseg, const riqn_reset_segment* segs,
                     unsigned long long seed, unsigned long long stream_id, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Test hook: plain strided fp32 product C[m,n] = sum_k A[m*sAm + k*sAk] * B[n*sBn + k*sBk].
 * ---------------------------------------------------------------------------------------------- */
int riqn_gemm_f32(int M, int N, int K, const float* A, long sAm, long sAk, const float* B, long sBn, long sBk,
                  float* C, long ldc, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* RIQN_B200_H */
