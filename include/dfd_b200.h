/* dfd_b200.h — C ABI of libdfd_b200.so: the sm_90a (H100) device kernels behind the data-parallel train / validate
 * step of TARTRL/Deepfake_Detection (dfd/runners/train.py:610-649, :713-746).
 *
 * The reference has NO native/FFI layer (SURVEY.md section 2.1): every entry point below replaces a stock
 * PyTorch op (ATen / cuDNN / cuBLAS dispatch) that the reference's nn.Module tree issues on the hot path; the
 * citation on each function is the reference call site it stands in for.  INTEGRATION.md shows the binding a
 * maintainer adds on the reference side (ctypes, because the reference is pure Python).
 *
 * Conventions
 *   - plain C types only; every pointer is a DEVICE pointer owned by the caller (no ownership transfer);
 *   - activations are NHWC, 16-bit: dt = DFD_DT_BF16 (0) or DFD_DT_FP16 (1); parameters, gradients, BN
 *     statistics, SE vectors, logits and the loss are fp32; channel counts are multiples of 8;
 *   - `stream` is a cudaStream_t; kernels are enqueued on it and nothing synchronises the host;
 *   - return value: 0 on success, negative DFD_ERR_* otherwise (dfd_last_error() gives the message); the
 *     Python host raises RuntimeError, the reference's only error convention;
 *   - per-channel statistics buffers hold DFD_STAT_SLOTS (= dfd_stat_slots() = 8) interleaved fp64 copies,
 *     i.e. [8][C] doubles, accumulated with atomics and zeroed by the caller once per step.
 */
#ifndef DFD_B200_H
#define DFD_B200_H

#ifdef __cplusplus
extern "C" {
#endif

#define DFD_OK 0
#define DFD_ERR_ARG (-1)
#define DFD_ERR_CUDA (-2)
#define DFD_ERR_UNSUPPORTED (-3)

#define DFD_DT_BF16 0
#define DFD_DT_FP16 1

#define DFD_ACT_NONE 0
#define DFD_ACT_SWISH 1
#define DFD_ACT_RELU 2

/* global pool types (layers/adaptive_avgmax_pool.py:35-48); pooled width P = F for all but CATAVGMAX (P = 2F) */
#define DFD_POOL_AVG 0
#define DFD_POOL_MAX 1
#define DFD_POOL_AVGMAX 2
#define DFD_POOL_CATAVGMAX 3

/* ---- runtime ---------------------------------------------------------------------------------------- */
const char* dfd_last_error(void);
int dfd_abi_version(void);
int dfd_stat_slots(void);
/* optimizer.zero_grad() (train.py:631) and per-step scratch clearing */
int dfd_memset_async(void* p, int value, long long bytes, void* stream);

/* ---- pointwise (1x1) convolution: nn.Conv2d via create_conv2d, efficientnet_blocks.py:165,277,299,
 *      efficientnet.py:292, resnet.py:192,199 -------------------------------------------------------- */
/* C[M,N] = A[M,K] * B[N,K]^T on wgmma (TMA in/out, accumulators in registers). Forward: A = input [N*H*W, Cin],
 * B = weight [Cout, Cin]. Input gradient: A = dY [N*H*W, Cout], B = weight^T [Cin, Cout].
 * dsum/dsq (optional): per-column sum / sum of squares of the stored C for the following BatchNorm. */
int dfd_gemm_tn(const void* A, const void* B, void* C, long long M, int N, int K, int dt, double* dsum, double* dsq,
                const void* fin, void* stream);
/* `fin` (optional; here and on dfd_gemm_tn_rowpack / dfd_dwconv_fwd): device pointer to a BnFinDesc (csrc/bn_finalize.cuh) -
 * the LAST CTA of the launch then finalises the BatchNorm behind the convolution (what dfd_bn_finalize does in its own
 * one-block launch): scale / shift / mean / rstd and the running statistics. The backward producers (dfd_act_bwd,
 * dfd_bn_bwd_reduce, dfd_dwconv_bwd) take a BnBwdFinDesc the same way (what dfd_bn_bwd_finalize does). NULL: no finalisation. */
/* Small-K variant (Cin = 16 / 24 / 32 pointwise convs and their input gradients): `pack` consecutive rows of A are read
 * as one row of pack*K values against the block-diagonal weight Bd[pack*N, pack*K] built by dfd_blockdiag_weights; the
 * result is byte-identical row-major C[M,N], statistics are folded back onto the N channels. Requires M % pack == 0. */
int dfd_gemm_tn_rowpack(const void* A, const void* Bd, void* C, long long M, int N, int K, int pack, int dt,
                        double* dsum, double* dsq, const void* fin, void* stream);
/* table: device array of { const void* src; void* dst; int N; int K; int pack; int _pad; } */
int dfd_blockdiag_weights(const void* table, int count, int dt, void* stream);
/* same contract on the warp-level mma.sync path (+ optional residual `add` [M,N]); cross-check / fallback */
int dfd_gemm_tn_mma(const void* A, const void* B, void* C, const void* add, long long M, int N, int K, int dt,
                    double* dsum, double* dsq, void* stream);
/* weight gradient dW[Nw,Kw] (fp32, accumulated) += G[M,Nw]^T * X[M,Kw]  (autograd of the conv, train.py:634) */
int dfd_gemm_wgrad_mma(const void* G, const void* X, float* dW, long long M, int Nw, int Kw, int dt, void* stream);
/* the same contract on wgmma: both operands MN-major straight from NHWC memory (TMA 128-byte swizzle boxes), fp32
 * accumulators in registers over a contiguous range of rows per CTA, one red.global.add flush */
int dfd_gemm_wgrad(const void* G, const void* X, float* dW, long long M, int Nw, int Kw, int dt, void* ws, long long ws_bytes,
                   void* stream);
/* ws (optional): ORDER-DETERMINISTIC mode - split z stores its fp32 partial matrix at ws[z][Nw][Kw] with plain stores, dW is
 * not touched, and dfd_ordered_reduce adds the dfd_gemm_wgrad_splits(M, Nw, Kw) partials into dW in split order afterwards
 * (ws_bytes >= splits * Nw * Kw * 4). NULL: red.global.add from every split straight into dW, in arrival order. */
int dfd_gemm_wgrad_splits(long long M, int Nw, int Kw);
/* dst[i] += sum_{p < parts} src[p * stride + i], i < n, partials added in index order. table: device array of
 * { const float* src; float* dst; long long n; long long stride; int parts; int _pad; } (n % 4 == 0, 16-byte aligned);
 * blocks_x = CTAs per entry (a CTA covers 256 float4 per trip of an entry with <= 64 parts, 8 float4 per trip otherwise);
 * first_dst (the lowest gradient address written) is informational for host-side planners. */
int dfd_ordered_reduce(const void* table, int count, const float* first_dst, int blocks_x, void* stream);

/* ---- depthwise k x k convolution: nn.Conv2d(groups=C), efficientnet_blocks.py:152-153,283-285 -------- */
int dfd_dwconv_fwd(const void* x, const float* scale, const float* shift, const float* w, void* out, int N, int H,
                   int W, int C, int k, int stride, int act_in, int dt, double* dsum, double* dsq, const void* fin,
                   void* stream);
int dfd_dwconv_dgrad(const void* gy, const void* yout, const float* cA, const float* cB, const float* cC,
                     const float* w, const void* xin, const float* scale, const float* shift, const float* mean,
                     const float* rstd, const void* add, void* gx, int N, int H, int W, int C, int k, int stride,
                     int mode, int dt, double* s1, double* s2, void* stream);
int dfd_dwconv_wgrad(const void* x, const float* scale, const float* shift, const void* gy, const void* yout,
                     const float* cA, const float* cB, const float* cC, float* dW, int N, int H, int W, int C, int k,
                     int stride, int dt, void* stream);
/* dfd_dwconv_dgrad + dfd_dwconv_wgrad of one depthwise stage in a single pass over dy: the autograd backward of conv_dw
 * (+ bn1/act1 behind it when scale != NULL, efficientnet_blocks.py:283-285, 277-281; scale == NULL: DS block,
 * efficientnet_blocks.py:152-153, gx = dgrad (+ add)), dW accumulated into `dW` */
int dfd_dwconv_bwd(const void* gy, const void* yout, const float* cA, const float* cB, const float* cC,
                   const float* w, const void* xin, const float* scale, const float* shift, const float* mean,
                   const float* rstd, const void* add, void* gx, float* dW, int N, int H, int W, int C, int k,
                   int stride, int dt, double* s1, double* s2, void* ws, long long ws_bytes, const void* fin, void* stream);
/* ws (optional): ORDER-DETERMINISTIC dW - CTA (tile x, channel block y, image group z) stores its partial at
 * ws[y][x * groups + z][B * k*k] laid out like dW[By .. By+B)[k*k], B = dfd_dwconv_block_channels(C), and
 * dfd_ordered_reduce adds the dfd_dwconv_bwd_parts(...) = tiles * groups partials of every channel block into dW in slot order
 * afterwards (ws_bytes >= ceil(C/B) * parts * B*k*k * 4). NULL: fp32 atomics into dW. */
int dfd_dwconv_bwd_parts(int N, int H, int W, int C, int k, int stride);
/* channels per CTA of the depthwise kernels for a layer of C channels (64, or 32 / 16 where 64-channel blocks would leave a
 * fifth or more of the lanes idle): the slot width and the channel-block size of the ws layout above */
int dfd_dwconv_block_channels(int C);
/* TF "SAME" padding (Conv2dSame, layers/conv2d_same.py; the tf_efficientnet_* models): dfd_dwconv_fwd / dfd_dwconv_bwd with
 * pad_t zero rows above and pad_l zero columns left of the image. Each is (k-1)/2, or (k-1)/2 - 1 at stride 2 over an even
 * extent; the output extent is ceil(extent / stride) either way (the end side gets the rest). The asymmetric backward takes
 * the stride-2 stage of an inverted-residual block only (scale and cA non-NULL). Symmetric pads run exactly the kernels of
 * the entry points above. */
int dfd_dwconv_fwd_pad(const void* x, const float* scale, const float* shift, const float* w, void* out, int N, int H,
                       int W, int C, int k, int stride, int pad_t, int pad_l, int act_in, int dt, double* dsum, double* dsq,
                       const void* fin, void* stream);
/* dfd_dwconv_bwd of a depthwise stage whose input passes a ReLU (Xception's separable convolutions; k = 3, stride 1, cA NULL):
 * scale != NULL: input relu(scale*xin + shift), gx = dgrad * 1[relu > 0] plus the BN-backward sums s1 / s2 of gx;
 * scale == NULL: input relu(xin), gx = dgrad * 1[xin > 0] (+ add). The masks test the staged 16-bit value. */
int dfd_dwconv_bwd_relu(const void* gy, const void* yout, const float* cA, const float* cB, const float* cC,
                        const float* w, const void* xin, const float* scale, const float* shift, const float* mean,
                        const float* rstd, const void* add, void* gx, float* dW, int N, int H, int W, int C, int k,
                        int stride, int dt, double* s1, double* s2, void* ws, long long ws_bytes, const void* fin, void* stream);
int dfd_dwconv_bwd_pad(const void* gy, const void* yout, const float* cA, const float* cB, const float* cC,
                       const float* w, const void* xin, const float* scale, const float* shift, const float* mean,
                       const float* rstd, const void* add, void* gx, float* dW, int N, int H, int W, int C, int k,
                       int stride, int pad_t, int pad_l, int dt, double* s1, double* s2, void* ws, long long ws_bytes,
                       const void* fin, void* stream);

/* ---- stem convolution: conv_stem 3x3 s2 (efficientnet.py:275,321) / conv1 7x7 s2 (resnet.py:379,451) ---- */
int dfd_stem_fwd(const void* x_nchw, const float* w, void* out_nhwc, int N, int Cin, int H, int W, int Cout, int k,
                 int stride, int pad, int dt, double* dsum, double* dsq, void* stream);
int dfd_stem_wgrad(const void* x_nchw, const void* g, const void* y, const float* cA, const float* cB,
                   const float* cC, float* dW, int N, int Cin, int H, int W, int Cout, int k, int stride, int pad,
                   int dt, void* stream);

/* stem as a GEMM (round-1 perf path): im2col of the NCHW image, column order (ci,kh,kw) == OIHW flattening, K padded to
 * Kp % 8 == 0; weights padded to [Cout, Kp]; fp32 gradient un-padded (accumulating) into the OIHW arena */
int dfd_stem_im2col(const void* x_nchw, void* cols, int N, int Cin, int H, int W, int k, int stride, int pad, int Kp, int dt,
                    void* stream);
/* the same with TF "SAME" padding: Ho = ceil(H/stride), Wo = ceil(W/stride); pad_t / pad_l must be the begin sides,
 * total // 2 of total = max((ceil(i/s) - 1)*s + k - i, 0) (layers/padding.py) */
int dfd_stem_im2col_pad(const void* x_nchw, void* cols, int N, int Cin, int H, int W, int k, int stride, int pad_t, int pad_l,
                        int Kp, int dt, void* stream);
int dfd_pad_weight(const void* src16, void* dst16, int O, int taps, int Kp, int dt, void* stream);
int dfd_unpad_grad(const float* g_padded, float* g_accum, int O, int taps, int Kp, void* stream);

/* ---- dense k x k convolution, max-pool, ReLU tail (ResNet: resnet.py:129-136,150-175,195-260,379-382,450-468).
 *      Product path: the IMPLICIT GEMMs further down (dfd_conv_tc, dfd_conv_wgrad_tc, dfd_conv_dgrad_s2_tc,
 *      dfd_conv1x1_dgrad_add) for every 3x3 and strided 1x1 convolution; the materialised formulation below (conv = im2col ->
 *      dfd_gemm_tn; dgrad = dfd_gemm_tn -> col2im; wgrad on the im2col matrix) serves the 7x7 stem, channel counts that are
 *      not multiples of 64, and the bit-exact cross-checks in the tests.
 *      Column order of the im2col matrix / packed weights: (kh, kw, ci). ------------------------------------------- */
int dfd_im2col(const void* x, void* cols, int N, int H, int W, int C, int k, int stride, int pad, int dt, void* stream);
int dfd_col2im(const void* dcols, const void* add, void* dx, int N, int H, int W, int C, int k, int stride, int pad, int dt,
               void* stream);
/* table: device array of { const void* src_OIHW16; void* dst_OHWI16; void* dstT_HWI_O16; void* dstD_IH'W'O16 (flipped taps);
 *                          int O; int I; int k; int pad; }  - dstT / dstD may be null */
int dfd_repack_weights(const void* table, int count, int dt, void* stream);
/* Dense k x k convolution, stride 1, padding (k-1)/2, as an IMPLICIT GEMM on wgmma (no im2col matrix in memory): the TMA
 * producer loads, per tap and 64-channel block, the NHWC input box shifted by the tap through a 4-D tensor map; out-of-image
 * rows arrive as zeros (= the padding). Replaces nn.Conv2d 3x3 stride 1 of BasicBlock / Bottleneck (resnet.py:129-136,195-197):
 *   forward: x = input [N,H,W,Cin],  wpk = dst_OHWI16,             y [N,H,W,Cout]; dsum/dsq = BatchNorm statistics of y
 *   dgrad  : x = dY    [N,H,W,Cout], wpk = dstD (flipped, [Cin]..), y = dX [N,H,W,Cin]  (call with Cin/Cout exchanged)
 * Cin % 64 == 0, Cout % 64 == 0. H, W = INPUT extents; stride 1 or 2 (2: the TMA box walks the input with element strides
 * {1, 2, 2, 1}; forward / weight gradient only - the strided input gradient stays dfd_gemm_tn + dfd_col2im); k = 1 with
 * stride 2 is the strided 1x1 downsample convolution (resnet.py:249-260) without its gather. */
int dfd_conv_tc(const void* x, const void* wpk, void* y, int N, int H, int W, int Cin, int Cout, int k, int stride, int dt,
                double* dsum, double* dsq, const void* fin, void* stream);
/* Weight gradient of the same convolution, also an implicit GEMM (MN-major wgmma operands straight from the NHWC tensors,
 * one pipeline stage = one patch of <= 64 output pixels, its input box shifted by the tap): dW_OHWI fp32 [Cout][kh][kw][Cin]
 * += sum_pixels dY[pixel, co] * x[pixel + tap, ci]. `ws` / `ws_bytes` as for dfd_gemm_wgrad: when given, the split partials
 * (dfd_conv_wgrad_splits x Cout x k*k*Cin floats) are written there for dfd_ordered_reduce and dW is left alone. */
int dfd_conv_wgrad_tc(const void* dy, const void* x, float* dW_ohwi, int N, int H, int W, int Cin, int Cout, int k, int stride,
                      int dt, void* ws, long long ws_bytes, void* stream);
int dfd_conv_wgrad_splits(int N, int H, int W, int Cin, int Cout, int k, int stride);
/* Input gradient of a 3x3, stride-2, padding-1 convolution (the autograd dgrad of resnet.py:195-197 with stride 2) as four
 * implicit GEMMs, one per parity class of the input pixels (1, 2, 2 and 4 taps), each storing through a strided tensor-map
 * view of dx: dx [N,H,W,Cin] is written exactly once, no column matrix, no col2im. dy [N,Ho,Wo,Cout]; wpkD = the tap-flipped
 * [Cin][kh'][kw'][Cout] layout of dfd_repack_weights. Cin % 64 == 0, Cout % 64 == 0. */
int dfd_conv_dgrad_s2_tc(const void* dy, const void* wpkD, void* dx, int N, int H, int W, int Cin, int Cout, int dt, void* stream);
/* Input gradient of a 1x1 convolution with stride 1 or 2 (downsample branch, resnet.py:249-260) ADDED into dx [N,H,W,Cin],
 * which already holds the main-path gradient: dx[n, s*a, s*b, :] += dY[n,a,b,:] * W - an implicit GEMM whose output map is
 * the stride-s pixel view of dx and whose epilogue is a TMA reduction store (16-bit add in L2). wT = transposed [Cin][Cout]
 * weight (dfd_transpose_weights). Replaces dfd_gemm_tn + dfd_col2im / dfd_add_inplace. */
int dfd_conv1x1_dgrad_add(const void* dy, const void* wT, void* dx, int N, int H, int W, int Cin, int Cout, int stride, int dt,
                          void* stream);
int dfd_unpack_grad(const float* g_ohwi, float* g_oihw_accum, int O, int I, int k, void* stream);
int dfd_maxpool_fwd(const void* x, void* out, void* argmax_u8, int N, int H, int W, int C, int dt, void* stream);
int dfd_maxpool_bwd(const void* gy, const void* argmax_u8, void* gx, int N, int H, int W, int C, int dt, void* stream);
/* nn.MaxPool2d(3, 2, ceil_mode=True) without padding (SENet's stem pool, senet.py:297-299): Ho = ceil((H - 3) / 2) + 1 (less
 * one if the last window would start outside the input), so the last window of an even extent is clipped; H, W >= 3 are the
 * INPUT extents for both directions. Arg-max byte and first-maximum tie-break as dfd_maxpool_fwd / dfd_maxpool_bwd. */
int dfd_maxpool_ceil_fwd(const void* x, void* out, void* argmax_u8, int N, int H, int W, int C, int dt, void* stream);
int dfd_maxpool_ceil_bwd(const void* gy, const void* argmax_u8, void* gx, int N, int H, int W, int C, int dt, void* stream);
int dfd_relu_bwd(const void* g, const void* out, void* gm, long long numel, int dt, void* stream);
int dfd_pool_bwd(const float* dpooled, void* dout, int N, long long hw, int C, int dt, void* stream);
/* backward of dfd_global_pool on a stored tensor (ResNet): dout[n,hw,c] = round16(g_avg[n,c] / HW + (hw == argmax[n,c]) *
 * g_max[n,c]), with g_avg / g_max taken from dpooled [N, P] by pool_type (MAX: 0 / dpooled; AVGMAX: both 0.5 * dpooled;
 * CATAVGMAX: dpooled[:, :C] / dpooled[:, C:]). pool_type != DFD_POOL_AVG (that is dfd_pool_bwd). */
int dfd_gpool_bwd(const float* dpooled, const int* argmax, void* dout, int N, long long hw, int C, int pool_type, int dt,
                  void* stream);

/* ---- BatchNorm2d (train + eval), Swish, SE gating, residual, global pool and their backward:
 *      efficientnet_blocks.py:104-110,154,166,180-194,280-348; layers/activations.py:19-33;
 *      efficientnet.py:323-343; resnet.py:154-173 ---------------------------------------------------- */
int dfd_colstats(const void* y, int n, long long hw, int C, int dt, double* dsum, double* dsq, void* stream);
int dfd_bn_finalize(const double* dsum, const double* dsq, double count, const float* gamma, const float* beta,
                    float* running_mean, float* running_var, long long* num_batches_tracked, float momentum,
                    float eps, int training, int C, float* scale, float* shift, float* mean, float* rstd,
                    void* stream);
int dfd_bn_act(const void* y, const float* scale, const float* shift, const float* gate, const void* res, void* out,
               int n, long long hw, int C, int act, int res_mode, int dt, void* stream);
/* pooled[n,c] = mean_hw act(scale*y + shift). `partial` (optional, max_chunks * n * C floats): when the batch alone cannot
 * fill the GPU, every image is reduced by up to max_chunks CTAs whose partial sums are added in a fixed order (the
 * forward stays bit-reproducible); NULL / max_chunks <= 1: one CTA per image */
int dfd_pool(const void* y, const float* scale, const float* shift, float* pooled, int n, long long hw, int C,
             int act, int dt, float* partial, int max_chunks, void* stream);
/* Selectable global pool of a = act(scale*y + shift) (fp32 on load, never stored; scale / shift NULL: a = y) in one pass:
 *   AVG: pooled[n,c] = mean_hw a        MAX: pooled[n,c] = max_hw a        AVGMAX: 0.5f * (mean + max)
 *   CATAVGMAX: pooled[n, 0:C] = mean, pooled[n, C:2C] = max           (pooled is [n, P])
 * argmax [n, C] int32 (optional) receives the hw index of the max under torch's adaptive_max_pool2d rule: a value replaces
 * the running max when it is strictly greater or NaN (ties -> first index in row-major order, NaN propagates). The mean is
 * summed in exactly dfd_pool's order and chunk geometry, so it is bit-identical to dfd_pool's result; chunk maxima are
 * combined in chunk order, so max and argmax do not depend on the chunking. */
int dfd_global_pool(const void* y, const float* scale, const float* shift, float* pooled, int* argmax, int n, long long hw,
                    int C, int act, int pool_type, int dt, int max_chunks, void* stream);
int dfd_bn_bwd_reduce(const void* g, const void* y, const void* out, const float* mean, const float* rstd, int n,
                      long long hw, int C, int dt, double* s1, double* s2, const void* fin, void* stream);
/* ReLU backward (and the residual add of the block above: g2 optional) fused into the reduction (ResNet block tail):
 * gm = round16(g + g2) * (out > 0) is stored and reduced in one pass */
int dfd_relu_bn_bwd_reduce(const void* g, const void* g2, const void* y, const void* out, void* gm, const float* mean,
                           const float* rstd, int n, long long hw, int C, int dt, double* s1, double* s2, void* stream);
int dfd_bn_bwd_finalize(const double* s1, const double* s2, double count, const float* gamma, const float* mean,
                        const float* rstd, float* dgamma, float* dbeta, float* cA, float* cB, float* cC, int C,
                        void* stream);
int dfd_bn_bwd_apply(const void* g, const void* y, const void* out, const float* cA, const float* cB,
                     const float* cC, void* dy, int n, long long hw, int C, int dt, void* stream);
int dfd_se_bwd_reduce(const void* da, const void* y, const float* scale, const float* shift, float* draw, int n,
                      long long hw, int C, int dt, void* stream);
int dfd_act_bwd(const void* da, const void* y, const float* scale, const float* shift, const float* mean,
                const float* rstd, const float* gate, const float* dpool, void* gu, int n, long long hw, int C,
                int act, int dt, double* s1, double* s2, const void* fin, void* stream);
/* dfd_act_bwd with no da and the gradient of dfd_global_pool instead of dpool (EfficientNet head: act = Swish; Xception: ReLU):
 *   gu = (g_avg[n,c] / hw + (hw == argmax[n,c]) * g_max[n,c]) * act'(u), g_avg / g_max from dpooled [n, P] as in
 * dfd_gpool_bwd; the BN backward sums and `fin` as in dfd_act_bwd. pool_type != DFD_POOL_AVG. */
int dfd_act_bwd_gpool(const void* y, const float* scale, const float* shift, const float* mean, const float* rstd,
                      const float* dpooled, const int* argmax, void* gu, int n, long long hw, int C, int act, int pool_type,
                      int dt, double* s1, double* s2, const void* fin, void* stream);
int dfd_add_inplace(void* a, const void* b, long long numel, int dt, void* stream);
/* 2x2 / stride-2 average pool of the ResNet-D shortcut, nn.AvgPool2d(2, 2, ceil_mode=True, count_include_pad=False)
 * (resnet.py:263-277), NHWC 16-bit: x [N,H,W,C] -> y [N,ceil(H/2),ceil(W/2),C]. Each output is the fp32 sum of the in-image
 * values of its window, in row-major order, times 1 / count (count 4, 2 or 1: a window clipped by an odd extent averages
 * the values it holds), rounded once. C % 8 == 0, C <= 8192. */
int dfd_avgpool2_fwd(const void* x, void* y, int N, int H, int W, int C, int dt, void* stream);
/* its input gradient, added to a second source: dx[n,y,x,c] = round16(add[n,y,x,c] + dy[n,y/2,x/2,c] / count(y/2, x/2)).
 * add may be NULL (zero) or dx itself. Elementwise, no atomics. H, W = INPUT extents. */
int dfd_avgpool2_bwd_add(const void* dy, const void* add, void* dx, int N, int H, int W, int C, int dt, void* stream);
/* tail of a strided Xception block (xception.py:110-124): out[N, Ho, Wo, C] = maxpool3x3s2p1(scale*y + shift) + scale_s*ys +
 * shift_s, Ho = (H - 1) / 2 + 1, rounded once; windows padded with -inf, the first maximum in row-major window order wins.
 * idx (NULL: not written): the arg-max tap (0..8), one byte per output. */
int dfd_bn_maxpool_add(const void* y, const float* scale, const float* shift, const void* ys, const float* scale_s,
                       const float* shift_s, void* out, void* idx, int N, int H, int W, int C, int dt, void* stream);
/* its backward through the pool: gx[N, H, W, C] = round16(sum of gy over the windows whose arg-max is the pixel), no atomics,
 * and the BN-backward sums s1 += gx, s2 += gx * (y - mean) * rstd (accumulated). H, W = INPUT extents. */
int dfd_maxpool_bn_bwd_reduce(const void* gy, const void* idx, const void* y, const float* mean, const float* rstd, void* gx,
                              int N, int H, int W, int C, int dt, double* s1, double* s2, void* stream);

/* ---- squeeze-excite FCs: SqueezeExcite.forward, efficientnet_blocks.py:104-110 ------------------------ */
int dfd_se_fc_fwd(const float* pooled, const float* Wr, const float* br, const float* We, const float* be,
                  float* gate, int N, int C, int Cse, void* stream);
int dfd_se_fc_bwd(const float* draw, const float* pooled, const float* Wr, const float* br, const float* We,
                  const float* be, float* d_e, float* r, float* d_rpre, float* dpool, float* dWr, float* dbr,
                  float* dWe, float* dbe, int N, int C, int Cse, void* stream);

/* SE parameter gradients from the per-image vectors of the backward chain: dWe += d_e^T r, dbe += sum d_e,
 * dWr += d_rpre^T pooled, dbr += sum d_rpre (split partials in fixed slots, added in order) */
int dfd_se_fc_wgrad(const float* d_e, const float* r, const float* d_rpre, const float* pooled, float* dWr, float* dbr,
                    float* dWe, float* dbe, int N, int C, int Cse, void* stream);
/* Fused forms (one launch each; the CTA that completes an image's reduction carries on with that image's FC chain, which is
 * latency-bound and hides in the tail of the streaming kernel):
 *   dfd_pool_se      = dfd_pool + dfd_se_fc_fwd            (squeeze + excite gate)
 *   dfd_se_bwd_chain = dfd_se_bwd_reduce + the per-image part of dfd_se_fc_bwd   (dfd_se_fc_wgrad follows) */
int dfd_pool_se(const void* y, const float* scale, const float* shift, float* pooled, const float* Wr, const float* br,
                const float* We, const float* be, float* gate, int n, long long hw, int C, int Cse, int act, int dt,
                int max_chunks, void* stream);
int dfd_se_bwd_chain(const void* da, const void* y, const float* scale, const float* shift, float* draw, const float* pooled,
                     const float* Wr, const float* br, const float* We, const float* be, float* d_e, float* r, float* d_rpre,
                     float* dpool, int n, long long hw, int C, int Cse, int dt, void* stream);
/* SENet's SEModule (senet.py:67-86: avg-pool, fc1 + bias, ReLU, fc2 + bias, sigmoid) on a = act(scale*y + shift), act NONE
 * (SEResNetBottleneck: the bare bn3 output) or RELU (SEResNetBlock, :213-215): pooled[n,c] = mean_hw a, gate[n,:] =
 * sigmoid(We relu(Wr pooled[n,:] + br) + be), fp32 [n, C]. Chunking for small batches as dfd_pool (max_chunks), the FC chain in
 * the CTA that completes the image. The block tail is dfd_bn_act(y, scale, shift, gate, res, act, res_mode 2). */
int dfd_pool_se_relu(const void* y, const float* scale, const float* shift, float* pooled, const float* Wr, const float* br,
                     const float* We, const float* be, float* gate, int n, long long hw, int C, int Cse, int act, int dt,
                     int max_chunks, void* stream);
/* Backward of the SE-ResNet block tail out = relu(a * gate[n,c] + res), a = act(scale*y + shift) (senet.py:111-112,220-221), in
 * one pass over the block output: gm = round16(g + g2) * (out > 0) is stored (g2 optional, as dfd_relu_bn_bwd_reduce),
 * draw[n,c] = sum_hw gm * a (fp32, chunk partials in fixed slots), and the CTA completing image n runs the SE backward chain
 * with the ReLU inner activation: d_e [n,C], r [n,Cse], d_rpre [n,Cse] for dfd_se_fc_wgrad and dpool [n,C] = dL/dpooled.
 * The last BatchNorm's input gradient is then gz = (gm * gate + dpool / hw) * act'(u): dfd_act_bwd (act, da = gm, gate, dpool). */
int dfd_relu_se_bwd_reduce(const void* g, const void* g2, const void* y, const void* out, const float* scale, const float* shift,
                           void* gm, float* draw, const float* pooled, const float* Wr, const float* br, const float* We,
                           const float* be, float* d_e, float* r, float* d_rpre, float* dpool, int n, long long hw, int C,
                           int Cse, int act, int dt, void* stream);

/* ---- classifier + loss + accuracy: nn.Linear (efficientnet.py:348, resnet.py:467), LabelSmoothing /
 *      SoftTarget / nn.CrossEntropyLoss (loss/cross_entropy.py:20-36, train.py:509-520), accuracy
 *      (utils.py:170-186).  Any K >= 1.  K == 2: one CTA per image, softmax-CE computed as sigmoid-BCE on z1 - z0
 *      (exactly equal); the backward splits the batch into fixed scratch slots added in order.  Every other K: fp32
 *      tiled SIMT GEMMs for logits / dpooled / dW (each output reduced by one thread in a fixed order, no split, no
 *      scratch) and a per-image max-subtracted log-sum-exp pass for loss, top-1 and dlogits; there a hard label outside
 *      [0, K) gives that image a NaN loss and a zero dlogits row.  Loss and correct count are added in image order:
 *      both heads are run-to-run bit-identical. ----- */
int dfd_head_fwd(const float* pooled, const float* W, const float* b, float* logits, int N, int F, int K,
                 const long long* target_i64, const float* target_soft, float smoothing, float loss_scale,
                 const float* loss_scale_dev, float* loss_acc, float* correct_acc, float* dlogits, void* stream);
int dfd_head_bwd(const float* dlogits, const float* pooled, const float* W, float* dW, float* db, float* dpooled,
                 int N, int F, int K, void* stream);

/* ---- the step's non-activation inputs (csrc/input.cu) ------------------------------------------------------------ */
/* PrefetchLoader.__iter__, dfd/timm/data/loader.py:243-256: uint8 NCHW batch -> 16-bit NCHW, (x - mean255[c]) / std255[c]
 * in fp32 with one rounding (mean255 / std255: device float[C] = mean*255 / std*255 repeated per frame, loader.py:229-230) */
int dfd_input_normalize(const void* x_u8, const float* mean255, const float* std255, void* out, int N, int C, int H, int W,
                        int dt, void* stream);
/* drop_path (layers/drop.py:84-100) and F.dropout (efficientnet.py:346-347) masks, already divided by keep_prob.
 * table: device array of { float* out; long long rows; int width; float keep_prob; int stream; int _pad; } - one random
 * draw per row, replicated over `width`; state: device int64 [seed, step] of the counter-based generator */
int dfd_rng_masks(const void* table, int count, const long long* state, void* stream);
int dfd_rng_tick(long long* state, void* stream);
int dfd_mul_f32(float* a, const float* b, long long n, void* stream);
/* DropBlock block masks of drop_block_2d (layers/drop.py:24-63), one launch for every site of the step.
 * table: device array of { unsigned char* mask; float* noise; unsigned long long* kept; double gamma; int N, H, W, C;
 * int cb; int stream; int _pad[2]; } (64 bytes). mask [N, H, W, C] = the min-pool over cb x cb (cb odd, <= 7) of the seeds
 * (2 - gamma - valid + u >= 1, u uniform per element); kept (zero on entry) receives the number of ones; noise (optional)
 * receives u. state: the [seed, step] of dfd_rng_masks; stream ids must differ from that table's. */
int dfd_drop_block_masks(const void* table, int count, const long long* state, void* stream);
/* DropBlock on the ResNet BatchNorm outputs (resnet.py:153-162,218-233): ms = mask ? numel / (float(*kept) + 1e-7) : 0.
 * res_mode 0: out = relu((scale*y + shift) * ms [* gate[n,c]]); res_mode 2: out = relu((scale*y + shift) * ms [* gate[n,c]]
 * + res). mask == NULL: dfd_bn_act with ReLU (res_mode 0) or the block tail (res_mode 2) */
int dfd_bn_act_drop(const void* y, const float* scale, const float* shift, const unsigned char* mask,
                    const unsigned long long* kept, long long numel, const float* gate, const void* res, void* out, int n,
                    long long hw, int C, int res_mode, int dt, void* stream);
/* gu = round16(da * ms) * (scale*y + shift > 0), stored, and the BN backward sums of gu */
int dfd_act_bwd_drop(const void* da, const void* y, const float* scale, const float* shift, const float* mean,
                     const float* rstd, const unsigned char* mask, const unsigned long long* kept, long long numel, void* gu,
                     int n, long long hw, int C, int dt, double* s1, double* s2, void* stream);
/* dfd_relu_bn_bwd_reduce for a block tail with DropBlock (mask) and / or drop path (gate [n, C]): gm = round16(g + g2) *
 * (out > 0) is stored unmasked; gd = round16(gm * ms * gate[n,c]) is stored and reduced */
int dfd_relu_bn_bwd_reduce_drop(const void* g, const void* g2, const void* y, const void* out, void* gm,
                                const unsigned char* mask, const unsigned long long* kept, long long numel, const float* gate,
                                void* gd, const float* mean, const float* rstd, int n, long long hw, int C, int dt, double* s1,
                                double* s2, void* stream);

/* ---- optimizers over the flat fp32 parameter arena: create_optimizer, optim_factory.py:26-100;
 *      RMSpropTF rmsprop_tf.py:57-122; AdamW adamw.py:55-117; apex AMP loss scaling train.py:353,632-634 ---- */
/* effective gradient scale = grad_scale * (*gscale_dev if non-null): 1/world for the DDP mean, 1/loss_scale on device.
 * lr_dev (optional, device float): when non-null it overrides `lr` - the schedulers mutate param_groups[i]['lr'] every
 * update (scheduler/scheduler.py:81-85), and a device-resident value lets one captured CUDA graph survive that.
 * step_dev (optional, device int): Adam's step count for the bias corrections, advanced by dfd_opt_tick. */
int dfd_sgd_step(float* p, const float* g, float* m, long long n, float lr, float momentum, float wd, int nesterov,
                 float grad_scale, const float* gscale_dev, const int* skip, void* p16, int dt, const float* lr_dev,
                 void* stream);
int dfd_adam_step(float* p, const float* g, float* m, float* v, long long n, float lr, float b1, float b2, float eps,
                  float wd, int decoupled, int step, float grad_scale, const float* gscale_dev, const int* skip, void* p16,
                  int dt, const float* lr_dev, const int* step_dev, void* stream);
int dfd_rmsprop_tf_step(float* p, const float* g, float* sq, float* mom, long long n, float lr, float alpha,
                        float eps, float wd, float momentum, float grad_scale, const float* gscale_dev, const int* skip,
                        void* p16, int dt, const float* lr_dev, void* stream);
/* ---- the other optimizers of create_optimizer (csrc/optim_ext.cu), same conventions; step_dev is required where named ---- */
/* RAdam, dfd/timm/optim/radam.py:10-82 (factory optim_factory.py:57-59): exp_avg m, exp_avg_sq v; N_sma and the step size from
 * *step_dev and *lr0_dev (group 0's lr: the reference caches them in self.buffer, shared by all groups, :54-70), in double;
 * decoupled decay p -= wd * lr * p first (:73-74) with the range's own lr; N_sma < 5: p -= step_size * m (:79-80) */
int dfd_radam_step(float* p, const float* g, float* m, float* v, long long n, float lr, double b1, double b2, float eps,
                   float wd, float grad_scale, const float* gscale_dev, const int* skip, void* p16, int dt,
                   const float* lr_dev, const float* lr0_dev, const int* step_dev, void* stream);
/* torch.optim.Adadelta(rho, eps, weight_decay) as built by optim_factory.py:63-65: square_avg sq, acc_delta acc, L2 decay */
int dfd_adadelta_step(float* p, const float* g, float* sq, float* acc, long long n, float lr, float rho, float eps, float wd,
                      float grad_scale, const float* gscale_dev, const int* skip, void* p16, int dt, const float* lr_dev,
                      void* stream);
/* torch.optim.RMSprop(alpha, eps, momentum, weight_decay), optim_factory.py:66-69: square_avg sq from zeros, eps outside the
 * sqrt, momentum_buffer mom (may be NULL when momentum == 0), lr applied at the weight update */
int dfd_rmsprop_step(float* p, const float* g, float* sq, float* mom, long long n, float lr, float alpha, float eps, float wd,
                     float momentum, float grad_scale, const float* gscale_dev, const int* skip, void* p16, int dt,
                     const float* lr_dev, void* stream);
/* Layer-wise norms of NovoGrad / NvNovoGrad (novograd.py:35,59; nvnovograd.py:94): sumsq[t] = sum over tensor t of
 * (g * grad_scale * *gscale_dev)^2. table: device array of { long long off; int len; int tensor; } (16 bytes), chunks of one
 * tensor each, in arena order; chunk0[t] .. chunk0[t+1] are tensor t's chunks (n_tensors + 1 ints); partial: n_chunks
 * doubles of scratch. Partials in fixed slots, fp64, added in a fixed order: bit-reproducible. Nothing written if *skip. */
int dfd_tensor_sumsq(const float* g, const void* table, int n_chunks, const int* chunk0, int n_tensors, double* partial,
                     float* sumsq, float grad_scale, const float* gscale_dev, const int* skip, void* stream);
/* NovoGrad, dfd/timm/optim/novograd.py:12-77, per-tensor part (one CTA): v, grad_ema [n_tensors]; state[0] = initialised flag
 * (the first applied step re-initialises every tensor, :30-46, and restarts *step_dev at 1), state[1] = this step
 * initialised; coef [2 * n_tensors] for dfd_novograd_step. ||g/(sqrt(grad_ema)+eps)||^2 is ||g||^2/(sqrt(grad_ema)+eps)^2. */
int dfd_novograd_prepare(const float* sumsq, float* v, float* grad_ema, float* coef, int* state, int* step_dev, int n_tensors,
                         float b2, float eps, const int* skip, void* stream);
/* NovoGrad elementwise part over the chunks [table, table + n_chunks) of one range: m, then p -= lr sqrt(1-b2^t)/(1-b1^t) m
 * (:65-72); wd is the constructor's decay (self._wd, :20,41,69) */
int dfd_novograd_step(float* p, const float* g, float* m, const void* table, int n_chunks, const float* coef, const int* state,
                      float lr, double b1, double b2, float wd, float grad_scale, const float* gscale_dev, const int* skip,
                      void* p16, int dt, const float* lr_dev, const int* step_dev, void* stream);
/* NvNovoGrad, dfd/timm/optim/nvnovograd.py:13-117, per tensor: exp_avg_sq = sumsq while it is 0, EMA after (:96-99);
 * denom = sqrt(exp_avg_sq) + eps */
int dfd_nvnovograd_prepare(const float* sumsq, float* exp_avg_sq, float* denom, int n_tensors, float b2, float eps,
                           const int* skip, void* stream);
/* NvNovoGrad elementwise part: exp_avg = b1 exp_avg + g / denom + wd p (the group's decay), p -= lr exp_avg (:108-115) */
int dfd_nvnovograd_step(float* p, const float* g, float* m, const void* table, int n_chunks, const float* denom, float lr,
                        float b1, float wd, float grad_scale, const float* gscale_dev, const int* skip, void* p16, int dt,
                        const float* lr_dev, void* stream);
/* *step_dev += 1 unless *skip (fp16 overflow): a skipped step does not advance Adam's bias correction (apex semantics) */
int dfd_opt_tick(int* step_dev, const int* skip, void* stream);
/* dst[0..n) = v0..v(n-1), n <= 8: host scalars (learning rates) to device memory, values carried in the launch itself */
int dfd_set_floats(float* dst, int n, float v0, float v1, float v2, float v3, float v4, float v5, float v6, float v7,
                   void* stream);
/* ModelEma.update (dfd/timm/utils.py:329-340) over the flat parameter / buffer arenas: ema = ema*decay + (1-decay)*model;
 * the int64 num_batches_tracked entries follow the reference's float arithmetic + truncating copy_ */
int dfd_ema_update(float* ema, const float* p, long long n, long long* ema_i64, const long long* p_i64, int n_i64,
                   float decay, void* stream);
int dfd_cast_arena(const float* p, void* p16, long long n, int dt, void* stream);
int dfd_check_finite(const float* g, long long n, int* flag, void* stream);
int dfd_update_loss_scale(int* flag, float* scale, int* good_steps, int interval, float* inv_scale_out,
                          void* stream);
/* table: device array of { const void* src; void* dst; int O; int I; } — dst[I,O] = transpose(src[O,I]) */
int dfd_transpose_weights(const void* table, int count, int dt, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DFD_B200_H */
