// Depthwise k x k convolution (k in {3,5}, stride in {1,2}) forward, input-gradient and weight-gradient,
// NHWC 16-bit activations, fp32 accumulation.   Reference: nn.Conv2d(groups=C) built by
// dfd/timm/models/layers/create_conv2d.py:11-30 at dfd/timm/models/efficientnet_blocks.py:152-153,283-285
// with symmetric padding (k-1)//2 (layers/padding.py:12-14), or, through the `_pad` entry points, with the TensorFlow
// "SAME" padding of the tf_efficientnet_* models (Conv2dSame, layers/conv2d_same.py): at stride 2 over an even extent the
// begin side (top / left) gets one element less, (k-1)/2 - 1, and the output extent stays ceil(H/2).
//
// Design: these layers are HBM-bound with k*k-fold reuse of every input element, and the preceding
// BN + Swish is fused into the load, so:
//   * a CTA stages an input tile (+halo) for 64 channels in shared memory ONCE, applying BN scale/shift and the
//     activation exactly once per element (sigmoid = one MUFU tanh), stored as packed 16-bit pairs;
//   * lane l of every warp owns channel pair (2l, 2l+1): shared-memory reads are 32 consecutive 4-byte words
//     (conflict free), global stores are 128 contiguous bytes per pixel;
//   * each warp computes strips of P=8 consecutive output columns with the k*k weights of its two channels
//     held in registers (sliding-window reuse: (P-1)*s+k smem reads feed P*k FMAs per kernel row);
//   * per-channel BN statistics of the (rounded) outputs are reduced in the epilogue: one fp64 atomic per
//     channel per CTA.
#include <stdlib.h>

#include "common.cuh"
#include "bn_finalize.cuh"

namespace {

constexpr int CB = 64;       // channels per CTA of the split (diagnostic) kernels and the default of the hot ones
// Lane mapping of the hot kernels (forward, fused backward): CPW channel PAIRS per sub-strip, 32 / CPW sub-strips per warp.
// CPW = 32: a lane is a channel pair, a warp works on one strip of 64 channels (every layer whose channel count fills
// 64-channel blocks). CPW = 16 / 8: a CTA covers 32 / 16 channels and the lanes of a warp split into 2 / 4 sub-strips on
// consecutive tile rows - so that C = 32, 96 or 144 (the three LARGEST layers of EfficientNet-B0, which left half or a
// quarter of every warp idle in the last 64-channel block) keep all 32 lanes busy. The staged tile is [pixel][CPW words];
// an odd tile width puts the sub-strips of a warp on disjoint shared-memory banks.
constexpr int P = 8;         // output columns per strip
constexpr int NTHREADS = 256;            // largest CTA (sizes the static reduction buffer); see dw_nt() for the per-k choice
constexpr int DW_MAX_SMEM = 200 * 1024;


struct DwGeom {
    int N, H, W, C, Ho, Wo, pad;     // pad: the symmetric (k-1)/2 (TF "SAME" pads: template parameters DT / DL below)
    int TH, TW;              // output tile (TW multiple of 8)
    int IH, IW;              // staged input tile
    int tiles_x, tiles_y;
    int dbg;                 // diagnostics (DFD_DW_DBG): 1 = skip the strip math, 2 = skip tile staging (fused backward only)
    // order-deterministic weight gradient of the fused backward (part != NULL): CTA (tile x, block y, group z) stores its
    // k*k x 64 partial at part[y][x * gz + z][64 * k*k] in dW's own (channel, tap) order with plain stores and leaves dW alone;
    // dfd_ordered_reduce adds the partials of every channel block in slot order later. NULL: fp32 atomics into dW.
    float* part;
};

__device__ __forceinline__ void load_chan_params(const float* p, int cbase, int C, float* out, float dflt) {
#pragma unroll
    for (int i = 0; i < 8; i++) out[i] = (p && cbase + i < C) ? p[cbase + i] : dflt;
}

// Stage act(scale*x+shift) for rows [iy0, iy0+IH) x cols [ix0, ix0+IW) x channels [c0, c0+64) of image `img`
// (zero outside the image / beyond C) into tile[(r*IW + c)*32 + word].
// UNR independent 16-byte loads are issued per thread before any is consumed (memory-level parallelism: with one
// load in flight per thread the kernel is latency-bound at ~1/3 of HBM speed).
constexpr int UNR = 4;
template <typename T, int ACT, bool AFFINE, int CPW = 32>
__device__ __forceinline__ void stage_input_tile(uint32_t* tile, const T* __restrict__ img, int H, int W, int C,
                                                 int c0, int iy0, int ix0, int IH, int IW,
                                                 const float* __restrict__ scale, const float* __restrict__ shift) {
    constexpr int VPP = CPW / 4;                 // 16-byte vectors (8 channels) per pixel
    const int v = threadIdx.x % VPP;
    const int cbase = c0 + v * 8;
    const bool cvalid = cbase < C;
    float sc[8], sh[8];
    if (AFFINE) { load_chan_params(scale, cbase, C, sc, 1.f); load_chan_params(shift, cbase, C, sh, 0.f); }
    const int npix = IH * IW;
    const int PSTEP = blockDim.x / VPP;
    // (row, col) of the visited pixels advance by PSTEP each: kept incrementally (an integer division per pixel cost
    // more issue slots than the activation it feeds)
    const int dq = PSTEP / IW, dr = PSTEP - dq * IW;
    int r = (threadIdx.x / VPP) / IW, c = (threadIdx.x / VPP) - r * IW;
    for (int base = threadIdx.x / VPP; base < npix; base += PSTEP * UNR) {
        uint4 raw[UNR];
        bool ok[UNR];
#pragma unroll
        for (int u = 0; u < UNR; u++) {
            const int pix = base + u * PSTEP;
            const int iy = iy0 + r, ix = ix0 + c;
            ok[u] = pix < npix && cvalid && iy >= 0 && iy < H && ix >= 0 && ix < W;
            if (ok[u]) raw[u] = ldg16(img + (uint32_t)((iy * W + ix) * C + cbase));      // in-image offsets fit 32 bits
            r += dq; c += dr;
            if (c >= IW) { c -= IW; r++; }
        }
#pragma unroll
        for (int u = 0; u < UNR; u++) {
            int pix = base + u * PSTEP;
            if (pix >= npix) break;
            uint4 o = make_uint4(0, 0, 0, 0);
            if (ok[u]) {
                if (AFFINE || ACT != DFD_ACT_NONE) {
                    float f[8];
                    unpack8<T>(raw[u], f);
#pragma unroll
                    for (int i = 0; i < 8; i++) {
                        float uu = AFFINE ? fmaf(f[i], sc[i], sh[i]) : f[i];
                        f[i] = act_fwd<ACT>(uu);
                    }
                    o = pack8<T>(f);
                } else {
                    o = raw[u];
                }
            }
            *reinterpret_cast<uint4*>(tile + pix * CPW + v * 4) = o;
        }
    }
}

// Stage the output gradient dy = A*g + B*y + C (BN backward folded into the load): tile pixel (r, c) <-> dy[oy0 + r,
// ox0 + c], zero outside [0,Ho) x [0,Wo).  (Compact: the stride-2 input-gradient kernel indexes it by parity, nothing is
// zero-upsampled.)
template <typename T, bool AFFINE, int UG_ = 0, int CPW = 32>
__device__ __forceinline__ void stage_grad_tile(uint32_t* tile, const T* __restrict__ g, const T* __restrict__ y,
                                                int Ho, int Wo, int C, int c0, int oy0, int ox0, int IH, int IW,
                                                const float* __restrict__ cA, const float* __restrict__ cB,
                                                const float* __restrict__ cC) {
    constexpr int VPP = CPW / 4;
    const int v = threadIdx.x % VPP;
    const int cbase = c0 + v * 8;
    const bool cvalid = cbase < C;
    float A[8], B[8], Cc[8];
    if (AFFINE) { load_chan_params(cA, cbase, C, A, 1.f); load_chan_params(cB, cbase, C, B, 0.f); load_chan_params(cC, cbase, C, Cc, 0.f); }
    const int npix = IH * IW;
    const int PSTEP = blockDim.x / VPP;
    constexpr int UG = UG_ ? UG_ : (AFFINE ? 2 : 4);     // two tensors are read when the BN backward is folded in
    const int dq = PSTEP / IW, dr = PSTEP - dq * IW;          // incremental (row, col), see stage_input_tile
    int r = (threadIdx.x / VPP) / IW, c = (threadIdx.x / VPP) - r * IW;
    for (int base = threadIdx.x / VPP; base < npix; base += PSTEP * UG) {
        uint4 graw[UG], yraw[UG];
        bool ok[UG];
#pragma unroll
        for (int u = 0; u < UG; u++) {
            const int pix = base + u * PSTEP;
            const int oy = oy0 + r, ox = ox0 + c;
            ok[u] = pix < npix && cvalid && oy >= 0 && oy < Ho && ox >= 0 && ox < Wo;
            if (ok[u]) {
                const uint32_t off = (uint32_t)((oy * Wo + ox) * C + cbase);
                graw[u] = ldg16(g + off);
                if (AFFINE) yraw[u] = ldg16(y + off);
            }
            r += dq; c += dr;
            if (c >= IW) { c -= IW; r++; }
        }
#pragma unroll
        for (int u = 0; u < UG; u++) {
            int pix = base + u * PSTEP;
            if (pix >= npix) break;
            uint4 o = make_uint4(0, 0, 0, 0);
            if (ok[u]) {
                if (AFFINE) {
                    float gg[8], yy[8];
                    unpack8<T>(graw[u], gg);
                    unpack8<T>(yraw[u], yy);
#pragma unroll
                    for (int i = 0; i < 8; i++) gg[i] = fmaf(A[i], gg[i], fmaf(B[i], yy[i], Cc[i]));
                    o = pack8<T>(gg);
                } else {
                    o = graw[u];
                }
            }
            *reinterpret_cast<uint4*>(tile + pix * CPW + v * 4) = o;
        }
    }
}

// stride-2 input gradient of one strip of P input columns (ix0 even) in input row `sy` (relative to the even tile
// origin): ga[p] = sum over taps with (sy+pad-kh) and (p+pad-kw) even of dy[(sy+pad-kh)/2, (sx+p+pad-kw)/2] * w[kh,kw].
// The compact dy tile starts at (y0/2 - 1, x0/2 - 1). Symmetric padding only (the diagnostic split kernel).
template <typename T, int K>
__device__ __forceinline__ void strip_dgrad_s2(const uint32_t* __restrict__ tile, int IW, int sy, int sx, int lane,
                                               const float (&w)[K * K][2], float (&acc)[P][2]) {
    constexpr int PAD = (K - 1) / 2;
#pragma unroll
    for (int kh = 0; kh < K; kh++) {
        const int q = sy + PAD - kh;
        if (q & 1) continue;                          // warp-uniform
        const int row = (q >> 1) + 1;
        const uint32_t* rp = tile + (row * IW + (sx >> 1)) * 32 + lane;
        float2 vv[P / 2 + 2];
#pragma unroll
        for (int j = 0; j < P / 2 + 2; j++) vv[j] = unpack2<T>(rp[j * 32]);
#pragma unroll
        for (int p = 0; p < P; p++) {
#pragma unroll
            for (int kw = 0; kw < K; kw++) {
                const int e = p + PAD - kw;
                if (((e % 2) + 2) % 2 == 0) {
                    const int col = (e + 2) / 2;      // e/2 + 1 with e >= -2
                    acc[p][0] = fmaf(vv[col].x, w[kh * K + kw][0], acc[p][0]);
                    acc[p][1] = fmaf(vv[col].y, w[kh * K + kw][1], acc[p][1]);
                }
            }
        }
    }
}

// acc[p][:] += sum_{kh,kw} tile[r0+kh][c0 + p*S + kw] * w[kh*K+kw]
template <typename T, int K, int S, int CPW = 32>
__device__ __forceinline__ void strip_conv(const uint32_t* __restrict__ tile, int IW, int r0, int c0, int lane,
                                           const float (&w)[K * K][2], float (&acc)[P][2]) {
#pragma unroll
    for (int kh = 0; kh < K; kh++) {
        const uint32_t* row = tile + ((r0 + kh) * IW + c0) * CPW + lane;      // `lane`: the channel-pair index in [0, CPW)
#pragma unroll
        for (int j = 0; j < (P - 1) * S + K; j++) {
            float2 x = unpack2<T>(row[j * CPW]);
#pragma unroll
            for (int kw = 0; kw < K; kw++) {
                int pj = j - kw;
                if (pj >= 0 && (pj % S) == 0 && pj / S < P) {
                    acc[pj / S][0] = fmaf(x.x, w[kh * K + kw][0], acc[pj / S][0]);
                    acc[pj / S][1] = fmaf(x.y, w[kh * K + kw][1], acc[pj / S][1]);
                }
            }
        }
    }
}

// block reduction of per-thread channel-pair values across the 8 warps, then fn(channel_in_block, value)
// (CPW < 32: the lanes cp, cp + CPW, ... of a warp hold the same channel pair on different sub-strips and are added first)
template <int CPW = 32, typename F>
__device__ __forceinline__ void reduce_warps_emit(float* sm, float a, float b, F fn) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
    for (int o = CPW; o < 32; o <<= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, o);
        b += __shfl_xor_sync(0xffffffffu, b, o);
    }
    if (lane < CPW) {
        sm[warp * 64 + lane * 2] = a;
        sm[warp * 64 + lane * 2 + 1] = b;
    }
    __syncthreads();
    if (threadIdx.x < 2 * CPW) {
        float s = 0.f;
#pragma unroll
        for (int w = 0; w < (int)(blockDim.x >> 5); w++) s += sm[w * 64 + threadIdx.x];
        fn(threadIdx.x, s);
    }
    __syncthreads();
}

// ---------------------------------------------------------------------------------------------
// forward
// ---------------------------------------------------------------------------------------------
// DT / DL: the top / left pad is g.pad - DT / g.pad - DL (TF "SAME" over an even extent at stride 2: DT, DL = 1)
template <typename T, int K, int S, int ACT, bool AFFINE, int NT, int CPW = 32, int DT = 0, int DL = 0>
__global__ void __launch_bounds__(NT)
dwconv_fwd_kernel(const T* __restrict__ x, const float* __restrict__ scale, const float* __restrict__ shift,
                  const float* __restrict__ wgt, T* __restrict__ out, double* __restrict__ dsum,
                  double* __restrict__ dsq, const BnFinDesc* __restrict__ fin, DwGeom g) {
    extern __shared__ __align__(16) uint32_t tile[];
    __shared__ float red[NTHREADS / 32 * 64];
    constexpr int SUB = 32 / CPW;               // sub-strips (consecutive tile rows) per warp
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int cp = lane % CPW, sub = lane / CPW;
    const int tx = blockIdx.x % g.tiles_x, ty = blockIdx.x / g.tiles_x;
    const int c0 = blockIdx.y * (2 * CPW), n = blockIdx.z;
    const int oy0 = ty * g.TH, ox0 = tx * g.TW;
    const T* img = x + (size_t)n * g.H * g.W * g.C;
    stage_input_tile<T, ACT, AFFINE, CPW>(tile, img, g.H, g.W, g.C, c0, oy0 * S - (g.pad - DT), ox0 * S - (g.pad - DL), g.IH, g.IW, scale, shift);

    const int ch = c0 + cp * 2;
    const bool chv = ch < g.C;
    float w[K * K][2];
#pragma unroll
    for (int i = 0; i < K * K; i++) {
        w[i][0] = chv ? wgt[(size_t)ch * K * K + i] : 0.f;
        w[i][1] = chv ? wgt[(size_t)(ch + 1) * K * K + i] : 0.f;
    }
    __syncthreads();

    float s0 = 0.f, s1 = 0.f, q0 = 0.f, q1 = 0.f;
    const int strips_x = g.TW / P;              // TW in {8,16,32}, P in {4,8}: a power of two
    const int xsh = 31 - __clz(strips_x);
    const int nstrips = ((g.TH + SUB - 1) / SUB) * strips_x;
    T* oimg = out + (size_t)n * g.Ho * g.Wo * g.C;
    for (int s = warp; s < nstrips; s += (int)(blockDim.x >> 5)) {
        const int sy = (s >> xsh) * SUB + sub, sx = (s & (strips_x - 1)) * P;
        int oy = oy0 + sy, ox = ox0 + sx;
        if (sy >= g.TH || oy >= g.Ho || ox >= g.Wo) continue;
        float acc[P][2];
#pragma unroll
        for (int p = 0; p < P; p++) { acc[p][0] = 0.f; acc[p][1] = 0.f; }
        strip_conv<T, K, S, CPW>(tile, g.IW, sy * S, sx * S, cp, w, acc);
        if (chv) {
#pragma unroll
            for (int p = 0; p < P; p++) {
                if (ox + p < g.Wo) {
                    uint32_t pk = pack2<T>(acc[p][0], acc[p][1]);
                    *reinterpret_cast<uint32_t*>(oimg + (uint32_t)((oy * g.Wo + ox + p) * g.C + ch)) = pk;
                    float2 r = unpack2<T>(pk);
                    s0 += r.x; s1 += r.y;
                    q0 = fmaf(r.x, r.x, q0); q1 = fmaf(r.y, r.y, q1);
                }
            }
        }
    }
    if (dsum) {
        double* ps = stat_slot(dsum, g.C);
        double* pq = stat_slot(dsq, g.C);
        reduce_warps_emit<CPW>(red, s0, s1, [&](int c, float v) { if (c0 + c < g.C) atomicAdd(ps + c0 + c, (double)v); });
        reduce_warps_emit<CPW>(red, q0, q1, [&](int c, float v) { if (c0 + c < g.C) atomicAdd(pq + c0 + c, (double)v); });
    }
    bn_finalize_tail(fin, threadIdx.x, NT);
}

// ---------------------------------------------------------------------------------------------
// input gradient.  Tile is in INPUT pixel space (H x W); the staged operand is the zero-upsampled dy.
//   ga[h,w] = sum_{kh',kw'} U[h - p' + kh', w - p' + kw'] * wflip[kh',kw'],  p' = K-1-pad
// MODE 0: dx = ga (+ add)                                   (DS block: dw conv reads the block input directly)
// MODE 1: gu = ga * act'(scale*xin + shift); BN-backward reductions s1 += gu, s2 += gu*xhat
// ---------------------------------------------------------------------------------------------
template <typename T, int K, int S, int MODE, bool AFFINE, int NT>
__global__ void __launch_bounds__(NT)
dwconv_dgrad_kernel(const T* __restrict__ gy, const T* __restrict__ yout, const float* __restrict__ cA,
                    const float* __restrict__ cB, const float* __restrict__ cC, const float* __restrict__ wgt,
                    const T* __restrict__ xin, const float* __restrict__ scale, const float* __restrict__ shift,
                    const float* __restrict__ mean, const float* __restrict__ rstd, const T* __restrict__ add,
                    T* __restrict__ gx, double* __restrict__ ds1, double* __restrict__ ds2, DwGeom g) {
    extern __shared__ __align__(16) uint32_t tile[];
    __shared__ float red[NTHREADS / 32 * 64];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tx = blockIdx.x % g.tiles_x, ty = blockIdx.x / g.tiles_x;
    const int c0 = blockIdx.y * CB, n = blockIdx.z;
    const int y0 = ty * g.TH, x0 = tx * g.TW;           // input-space tile origin
    const int pp = K - 1 - g.pad;
    const size_t ooff = (size_t)n * g.Ho * g.Wo * g.C;
    // stride 1: the dy tile is the input tile shifted by the flipped padding; stride 2: compact tile at (y0/2-1, x0/2-1)
    stage_grad_tile<T, AFFINE>(tile, gy + ooff, AFFINE ? yout + ooff : nullptr, g.Ho, g.Wo, g.C, c0,
                               S == 1 ? y0 - pp : (y0 >> 1) - 1, S == 1 ? x0 - pp : (x0 >> 1) - 1, g.IH, g.IW, cA, cB, cC);
    const int ch = c0 + lane * 2;
    const bool chv = ch < g.C;
    float w[K * K][2];
#pragma unroll
    for (int i = 0; i < K * K; i++) {       // stride 1: flipped taps (correlation form); stride 2: direct taps
        const int src = S == 1 ? (K * K - 1 - i) : i;
        w[i][0] = chv ? wgt[(size_t)ch * K * K + src] : 0.f;
        w[i][1] = chv ? wgt[(size_t)(ch + 1) * K * K + src] : 0.f;
    }
    float sc0 = 1.f, sc1 = 1.f, sh0 = 0.f, sh1 = 0.f, mu0 = 0.f, mu1 = 0.f, rs0 = 0.f, rs1 = 0.f;
    if (MODE == 1 && chv) {
        sc0 = scale[ch]; sc1 = scale[ch + 1]; sh0 = shift[ch]; sh1 = shift[ch + 1];
        mu0 = mean[ch]; mu1 = mean[ch + 1]; rs0 = rstd[ch]; rs1 = rstd[ch + 1];
    }
    __syncthreads();

    float a0 = 0.f, a1 = 0.f, b0 = 0.f, b1 = 0.f;
    const int strips_x = g.TW / P;              // TW in {8,16,32}, P in {4,8}: a power of two
    const int xsh = 31 - __clz(strips_x);
    const int nstrips = g.TH * strips_x;
    const size_t ioff = (size_t)n * g.H * g.W * g.C;
    for (int s = warp; s < nstrips; s += (int)(blockDim.x >> 5)) {
        const int sy = s >> xsh, sx = (s & (strips_x - 1)) * P;
        int iy = y0 + sy, ix = x0 + sx;
        if (iy >= g.H || ix >= g.W) continue;
        // issue the strip's global reads (pre-activation input / residual gradient) BEFORE the conv math so that
        // their latency hides behind it instead of serialising with the stores
        uint32_t pre[P];
        const size_t off0 = ioff + ((size_t)iy * g.W + ix) * g.C + ch;
        if (chv && (MODE == 1 || add)) {
            const T* src = MODE == 1 ? xin : add;
#pragma unroll
            for (int p = 0; p < P; p++) pre[p] = (ix + p < g.W) ? __ldg(reinterpret_cast<const uint32_t*>(src + off0 + (size_t)p * g.C)) : 0u;
        }
        float acc[P][2];
#pragma unroll
        for (int p = 0; p < P; p++) { acc[p][0] = 0.f; acc[p][1] = 0.f; }
        if (S == 1) strip_conv<T, K, 1>(tile, g.IW, sy, sx, lane, w, acc);
        else strip_dgrad_s2<T, K>(tile, g.IW, sy, sx, lane, w, acc);
        if (chv) {
#pragma unroll
            for (int p = 0; p < P; p++) {
                if (ix + p < g.W) {
                    size_t off = off0 + (size_t)p * g.C;
                    float v0 = acc[p][0], v1 = acc[p][1];
                    if (MODE == 1) {
                        float2 xi = unpack2<T>(pre[p]);
                        v0 *= act_bwd<DFD_ACT_SWISH>(fmaf(xi.x, sc0, sh0));
                        v1 *= act_bwd<DFD_ACT_SWISH>(fmaf(xi.y, sc1, sh1));
                        uint32_t pk = pack2<T>(v0, v1);
                        *reinterpret_cast<uint32_t*>(gx + off) = pk;
                        float2 r = unpack2<T>(pk);
                        a0 += r.x; a1 += r.y;
                        b0 = fmaf(r.x, (xi.x - mu0) * rs0, b0);
                        b1 = fmaf(r.y, (xi.y - mu1) * rs1, b1);
                    } else {
                        if (add) {
                            float2 ad = unpack2<T>(pre[p]);
                            v0 += ad.x; v1 += ad.y;
                        }
                        *reinterpret_cast<uint32_t*>(gx + off) = pack2<T>(v0, v1);
                    }
                }
            }
        }
    }
    if (MODE == 1) {
        double* p1 = stat_slot(ds1, g.C);
        double* p2 = stat_slot(ds2, g.C);
        reduce_warps_emit(red, a0, a1, [&](int c, float v) { if (c0 + c < g.C) atomicAdd(p1 + c0 + c, (double)v); });
        reduce_warps_emit(red, b0, b1, [&](int c, float v) { if (c0 + c < g.C) atomicAdd(p2 + c0 + c, (double)v); });
    }
}

// ---------------------------------------------------------------------------------------------
// weight gradient: dW[c,kh,kw] += sum_{n,oy,ox} dy[n,oy,ox,c] * a[n, oy*S-pad+kh, ox*S-pad+kw, c]
// a = act(scale*x+shift) is re-staged like the forward; dy = A*g + B*y + C is formed per strip.
// gridDim.z image groups: each CTA loops over images z, z+gridDim.z, ... to bound the number of atomics.
// ---------------------------------------------------------------------------------------------
template <typename T, int K, int S, int ACT, bool AFFINE_IN, bool AFFINE_G, int NT>
__global__ void __launch_bounds__(NT)
dwconv_wgrad_kernel(const T* __restrict__ x, const float* __restrict__ scale, const float* __restrict__ shift,
                    const T* __restrict__ gy, const T* __restrict__ yout, const float* __restrict__ cA,
                    const float* __restrict__ cB, const float* __restrict__ cC, float* __restrict__ dW, DwGeom g) {
    extern __shared__ __align__(16) uint32_t tile[];
    __shared__ float red[NTHREADS / 32 * 64];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tx = blockIdx.x % g.tiles_x, ty = blockIdx.x / g.tiles_x;
    const int c0 = blockIdx.y * CB;
    const int oy0 = ty * g.TH, ox0 = tx * g.TW;
    const int ch = c0 + lane * 2;
    const bool chv = ch < g.C;
    float A0 = 1.f, A1 = 1.f, B0 = 0.f, B1 = 0.f, C0 = 0.f, C1 = 0.f;
    if (AFFINE_G && chv) { A0 = cA[ch]; A1 = cA[ch + 1]; B0 = cB[ch]; B1 = cB[ch + 1]; C0 = cC[ch]; C1 = cC[ch + 1]; }
    float wacc[K * K][2];
#pragma unroll
    for (int i = 0; i < K * K; i++) { wacc[i][0] = 0.f; wacc[i][1] = 0.f; }
    const int strips_x = g.TW / P;              // TW in {8,16,32}, P in {4,8}: a power of two
    const int xsh = 31 - __clz(strips_x);
    const int nstrips = g.TH * strips_x;

    for (int n = blockIdx.z; n < g.N; n += gridDim.z) {
        const T* img = x + (size_t)n * g.H * g.W * g.C;
        const size_t ooff = (size_t)n * g.Ho * g.Wo * g.C;
        // software pipeline: the raw gradient operands of a strip are fetched one strip ahead (the first one before
        // the tile is staged) so that their global latency overlaps staging / the previous strip's FMAs
        uint32_t gq[P], yq[P];
        auto prefetch = [&](int s) {
            const int sy = s >> xsh, sx = (s & (strips_x - 1)) * P;
            int oy = oy0 + sy, ox = ox0 + sx;
            const bool rowok = chv && oy < g.Ho;
            const size_t off0 = ooff + ((size_t)oy * g.Wo + ox) * g.C + ch;
#pragma unroll
            for (int p = 0; p < P; p++) {
                const bool ok = rowok && ox + p < g.Wo;
                gq[p] = ok ? __ldg(reinterpret_cast<const uint32_t*>(gy + off0 + (size_t)p * g.C)) : 0u;
                if (AFFINE_G) yq[p] = ok ? __ldg(reinterpret_cast<const uint32_t*>(yout + off0 + (size_t)p * g.C)) : 0u;
            }
        };
        if (warp < nstrips) prefetch(warp);
        __syncthreads();    // previous image's tile fully consumed
        stage_input_tile<T, ACT, AFFINE_IN>(tile, img, g.H, g.W, g.C, c0, oy0 * S - g.pad, ox0 * S - g.pad, g.IH, g.IW, scale, shift);
        __syncthreads();
        for (int s = warp; s < nstrips; s += (int)(blockDim.x >> 5)) {
            const int sy = s >> xsh, sx = (s & (strips_x - 1)) * P;
            int oy = oy0 + sy, ox = ox0 + sx;
            float dy[P][2];
#pragma unroll
            for (int p = 0; p < P; p++) {
                float2 gg = unpack2<T>(gq[p]);
                const bool ok = chv && oy < g.Ho && ox + p < g.Wo;
                if (AFFINE_G) {
                    float2 yy = unpack2<T>(yq[p]);
                    // round like the staged operand of the dgrad kernel so both see the same dy
                    gg = unpack2<T>(pack2<T>(fmaf(A0, gg.x, fmaf(B0, yy.x, C0)), fmaf(A1, gg.y, fmaf(B1, yy.y, C1))));
                }
                dy[p][0] = ok ? gg.x : 0.f;
                dy[p][1] = ok ? gg.y : 0.f;
            }
            if (s + (int)(blockDim.x >> 5) < nstrips) prefetch(s + (int)(blockDim.x >> 5));
            if (oy >= g.Ho || ox >= g.Wo || !chv) continue;
#pragma unroll
            for (int kh = 0; kh < K; kh++) {
                const uint32_t* row = tile + ((sy * S + kh) * g.IW + sx * S) * 32 + lane;
#pragma unroll
                for (int j = 0; j < (P - 1) * S + K; j++) {
                    float2 a = unpack2<T>(row[j * 32]);
#pragma unroll
                    for (int kw = 0; kw < K; kw++) {
                        int pj = j - kw;
                        if (pj >= 0 && (pj % S) == 0 && pj / S < P) {
                            wacc[kh * K + kw][0] = fmaf(a.x, dy[pj / S][0], wacc[kh * K + kw][0]);
                            wacc[kh * K + kw][1] = fmaf(a.y, dy[pj / S][1], wacc[kh * K + kw][1]);
                        }
                    }
                }
            }
        }
    }
    // reduce the 8 warps' partial sums, one tap at a time, then one fp32 atomic per (channel, tap) per CTA
#pragma unroll
    for (int i = 0; i < K * K; i++) {
        reduce_warps_emit(red, wacc[i][0], wacc[i][1], [&](int c, float v) {
            if (c0 + c < g.C) atomicAdd(dW + (size_t)(c0 + c) * K * K + i, v);
        });
    }
}

// ---------------------------------------------------------------------------------------------
// fused backward of an MBConv depthwise stage: the input gradient of MODE 1 above AND the weight gradient in one pass.
// Both are sums over the same (input pixel x, tap t) pairs of the staged dy tile:
//     ga[x] += dy[o(x,t)] * w[t]            dW[t] += dy[o(x,t)] * a[x],   a = swish(scale*xin + shift)
// so the pass that owns input pixel x (this kernel's tiling) feeds two FMAs from every shared-memory read, the dy
// operand (two tensors when the BN backward is folded in) is fetched and formed once instead of twice, and the
// sigmoid of the input pixel serves both a and swish'.  A CTA walks images blockIdx.z, +gridDim.z, ... so that its
// k*k weight-gradient partials (registers) are reduced and flushed once, not once per image.
// ---------------------------------------------------------------------------------------------
// PT / PL: the zero rows above / columns left of the image, (K-1)/2 (symmetric) or (K-1)/2 - 1 (TF "SAME" over an even
// extent). Either way the taps that reach input row sy read dy rows (sy + PT - kh)/2 >= -1 and <= (TH+1)/2 - 1 of the tile
// (columns likewise): the compact tile at (y0/2 - 1, x0/2 - 1) with (TH+1)/2 + 2 rows and TW/2 + 2 columns covers both
// pads; only the tap parity classes change.
template <typename T, int K, bool WG, int P, int CPW = 32, int PT = (K - 1) / 2, int PL = (K - 1) / 2>
__device__ __forceinline__ void strip_bwd_s2(const uint32_t* __restrict__ tile, int IW, int sy, int sx, int lane,
                                             const float (&w)[K * K][2], float (&acc)[P][2],
                                             const float (&av)[P][2], float (&wacc)[K * K][2]) {
#pragma unroll
    for (int kh = 0; kh < K; kh++) {
        const int q = sy + PT - kh;
        if (q & 1) continue;                          // warp-uniform: the sub-strips of a warp sit on rows of one parity
        const int row = (q >> 1) + 1;
        const uint32_t* rp = tile + (row * IW + (sx >> 1)) * CPW + lane;
        float2 vv[P / 2 + 2];
#pragma unroll
        for (int j = 0; j < P / 2 + 2; j++) vv[j] = unpack2<T>(rp[j * CPW]);
#pragma unroll
        for (int p = 0; p < P; p++) {
#pragma unroll
            for (int kw = 0; kw < K; kw++) {
                const int e = p + PL - kw;
                if (((e % 2) + 2) % 2 == 0) {
                    const int col = (e + 2) / 2;
                    acc[p][0] = fmaf(vv[col].x, w[kh * K + kw][0], acc[p][0]);
                    acc[p][1] = fmaf(vv[col].y, w[kh * K + kw][1], acc[p][1]);
                    if (WG) {
                        wacc[kh * K + kw][0] = fmaf(vv[col].x, av[p][0], wacc[kh * K + kw][0]);
                        wacc[kh * K + kw][1] = fmaf(vv[col].y, av[p][1], wacc[kh * K + kw][1]);
                    }
                }
            }
        }
    }
}

template <typename T, int K, int P, int CPW = 32>
__device__ __forceinline__ void strip_bwd_s1(const uint32_t* __restrict__ tile, int IW, int r0, int c0, int lane,
                                             const float (&w)[K * K][2], float (&acc)[P][2],
                                             const float (&av)[P][2], float (&wacc)[K * K][2]) {
#pragma unroll
    for (int kh = 0; kh < K; kh++) {
        const uint32_t* row = tile + ((r0 + kh) * IW + c0) * CPW + lane;
#pragma unroll
        for (int j = 0; j < P - 1 + K; j++) {
            float2 x = unpack2<T>(row[j * CPW]);
#pragma unroll
            for (int kw = 0; kw < K; kw++) {
                const int pj = j - kw;
                if (pj >= 0 && pj < P) {
                    acc[pj][0] = fmaf(x.x, w[kh * K + kw][0], acc[pj][0]);
                    acc[pj][1] = fmaf(x.y, w[kh * K + kw][1], acc[pj][1]);
                    wacc[kh * K + kw][0] = fmaf(x.x, av[pj][0], wacc[kh * K + kw][0]);
                    wacc[kh * K + kw][1] = fmaf(x.y, av[pj][1], wacc[kh * K + kw][1]);
                }
            }
        }
    }
}

// MODE 1: xin is the pre-BN expand output (a = swish(scale*xin + shift), gx = ga * swish', BN-backward sums);
// MODE 0: xin is the block input itself (DS block): a = xin, gx = ga (+ add);
// MODE 2: a = relu(scale*xin + shift) (Xception, inside a block): gx = ga * 1[a > 0], BN-backward sums as MODE 1;
// MODE 3: a = relu(xin) (Xception, a block's first separable convolution): gx = ga * 1[xin > 0] (+ add).
// The ReLU masks test the 16-bit value the forward staged, so that torch's (out > 0) rule holds after rounding too.
// DT / DL (stride 2 only): the top / left pad is (K-1)/2 - DT / (K-1)/2 - DL (see strip_bwd_s2).
template <typename T, int K, int S, bool AFFINE, int MODE, int NT, int P, int CPW = 32, int DT = 0, int DL = 0>
#ifndef DW_BWD_OCC3
#define DW_BWD_OCC3 4
#endif
__global__ void __launch_bounds__(NT, K == 3 ? (P == 4 ? DW_BWD_OCC3 : 3) : 2)
dwconv_bwd_kernel(const T* __restrict__ gy, const T* __restrict__ yout, const float* __restrict__ cA,
                  const float* __restrict__ cB, const float* __restrict__ cC, const float* __restrict__ wgt,
                  const T* __restrict__ xin, const float* __restrict__ scale, const float* __restrict__ shift,
                  const float* __restrict__ mean, const float* __restrict__ rstd, const T* __restrict__ add,
                  T* __restrict__ gx,
                  float* __restrict__ dW, double* __restrict__ ds1, double* __restrict__ ds2,
                  const BnBwdFinDesc* __restrict__ fin, DwGeom g) {
    extern __shared__ __align__(16) uint32_t tile[];
    __shared__ float red[NTHREADS / 32 * 64];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    constexpr int NW = NT / 32;
    constexpr int SUB = 32 / CPW;           // sub-strips per warp (see the lane mapping note at the top)
    constexpr int CW = 2 * CPW;             // channels per CTA
    const int cp = lane % CPW, sub = lane / CPW;
    const int tx = blockIdx.x % g.tiles_x, ty = blockIdx.x / g.tiles_x;
    const int c0 = blockIdx.y * CW;
    const int y0 = ty * g.TH, x0 = tx * g.TW;           // input-space tile origin
    const int pp = K - 1 - g.pad;
    const int ch = c0 + cp * 2;
    const bool chv = ch < g.C;
    float w[K * K][2], wacc[K * K][2];
#pragma unroll
    for (int i = 0; i < K * K; i++) {       // stride 1: flipped taps (correlation form); stride 2: direct taps
        const int src = S == 1 ? (K * K - 1 - i) : i;
        w[i][0] = chv ? wgt[(size_t)ch * K * K + src] : 0.f;
        w[i][1] = chv ? wgt[(size_t)(ch + 1) * K * K + src] : 0.f;
        wacc[i][0] = 0.f; wacc[i][1] = 0.f;
    }
    float sc0 = 1.f, sc1 = 1.f, sh0 = 0.f, sh1 = 0.f, mu0 = 0.f, mu1 = 0.f, rs0 = 0.f, rs1 = 0.f;
    if ((MODE == 1 || MODE == 2) && chv) {
        sc0 = scale[ch]; sc1 = scale[ch + 1]; sh0 = shift[ch]; sh1 = shift[ch + 1];
        mu0 = mean[ch]; mu1 = mean[ch + 1]; rs0 = rstd[ch]; rs1 = rstd[ch + 1];
    }
    const float nm0 = -mu0 * rs0, nm1 = -mu1 * rs1;
    float a0 = 0.f, a1 = 0.f, b0 = 0.f, b1 = 0.f;
    const int strips_x = g.TW / P;              // TW in {8,16,32}, P in {4,8}: a power of two
    const int xsh = 31 - __clz(strips_x);
    // A warp visits SUB tile rows at once. Stride 1: rows g*SUB + sub. Stride 2: the taps of an input row depend on its
    // parity, so a warp's rows share one parity - rows 2*(g*SUB + sub) + par, all even groups first, then the odd ones.
    const int row_groups = S == 1 ? (g.TH + SUB - 1) / SUB : ((g.TH + 1) / 2 + SUB - 1) / SUB;
    const int nstrips = (S == 1 ? row_groups : 2 * row_groups) * strips_x;
    auto strip_row = [&](int s) {
        const int r = s >> xsh;
        if (S == 1) return r * SUB + sub;
        const int par = r >= row_groups ? 1 : 0;
        return 2 * ((r - par * row_groups) * SUB + sub) + par;
    };

    for (int n = blockIdx.z; n < g.N; n += gridDim.z) {
        const size_t ooff = (size_t)n * g.Ho * g.Wo * g.C;
        const size_t ioff = (size_t)n * g.H * g.W * g.C;
        const T* xin_n = xin + ioff;        // per-image bases: offsets inside an image fit 32 bits
        T* gx_n = gx + ioff;
        // the strip's pre-activation inputs are an OPERAND here (a = swish(bn(xin))): fetched one strip ahead, the
        // first one before the tile is staged, so their latency hides behind staging / the previous strip's FMAs
        uint32_t pre[P];
        auto prefetch = [&](int s) {
            const int sy = strip_row(s), sx = (s & (strips_x - 1)) * P;
            const int iy = y0 + sy, ix = x0 + sx;
            const bool rowok = chv && sy < g.TH && iy < g.H;
            const uint32_t off0 = (uint32_t)((iy * g.W + ix) * g.C + ch);
#pragma unroll
            for (int p = 0; p < P; p++)
                pre[p] = (rowok && ix + p < g.W) ? __ldg(reinterpret_cast<const uint32_t*>(xin_n + off0 + (uint32_t)(p * g.C))) : 0u;
        };
        if (warp < nstrips) prefetch(warp);
        __syncthreads();    // previous image's tile fully consumed
        // staging batch (16-byte loads in flight per thread and tensor): 4 for k = 5 (two CTAs per SM either way), 2 for k = 3
        // where the deeper batch costs the third resident CTA; both chosen on the GPU this code was first tuned on, not
        // re-measured on the H100
        if (!(g.dbg & 2))
            stage_grad_tile<T, AFFINE, (K == 5 ? 4 : 2), CPW>(tile, gy + ooff, AFFINE ? yout + ooff : nullptr, g.Ho, g.Wo, g.C, c0,
                                   S == 1 ? y0 - pp : (y0 >> 1) - 1, S == 1 ? x0 - pp : (x0 >> 1) - 1, g.IH, g.IW, cA, cB, cC);
        __syncthreads();
        if (!(g.dbg & 1))
        for (int s = warp; s < nstrips; s += NW) {
            const int sy = strip_row(s), sx = (s & (strips_x - 1)) * P;
            const int iy = y0 + sy, ix = x0 + sx;
            float av[P][2], da[P][2], xh[P][2];
            // interior strips need no per-pixel masking: lanes beyond C compute garbage that is never stored, reduced or
            // flushed (pre[] is zero for rows outside the tile / image)
            const bool interior = sy < g.TH && iy < g.H && ix + P <= g.W;
#pragma unroll
            for (int p = 0; p < P; p++) {
                const float2 xi = unpack2<T>(pre[p]);
                if (MODE == 1) {
                    const float u0 = fmaf(xi.x, sc0, sh0), u1 = fmaf(xi.y, sc1, sh1);
                    const float g0 = sigmoid_fast(u0), g1 = sigmoid_fast(u1);
                    // the forward staged a = swish(u) as a 16-bit value: the weight gradient sees the same rounding
                    const float2 ar = unpack2<T>(pack2<T>(u0 * g0, u1 * g1));
                    av[p][0] = ar.x;
                    av[p][1] = ar.y;
                    da[p][0] = fmaf(g0, fmaf(-u0, g0, u0), g0);       // == act_bwd<SWISH>(u)
                    da[p][1] = fmaf(g1, fmaf(-u1, g1, u1), g1);
                    xh[p][0] = fmaf(xi.x, rs0, nm0);                  // (x - mean) * rstd
                    xh[p][1] = fmaf(xi.y, rs1, nm1);
                } else if (MODE == 2) {
                    const float2 ar = unpack2<T>(pack2<T>(fmaxf(fmaf(xi.x, sc0, sh0), 0.f), fmaxf(fmaf(xi.y, sc1, sh1), 0.f)));
                    av[p][0] = ar.x;
                    av[p][1] = ar.y;
                    da[p][0] = ar.x > 0.f ? 1.f : 0.f;
                    da[p][1] = ar.y > 0.f ? 1.f : 0.f;
                    xh[p][0] = fmaf(xi.x, rs0, nm0);
                    xh[p][1] = fmaf(xi.y, rs1, nm1);
                } else if (MODE == 3) {
                    av[p][0] = fmaxf(xi.x, 0.f);     // zero outside the image and beyond C already
                    av[p][1] = fmaxf(xi.y, 0.f);
                    da[p][0] = xi.x > 0.f ? 1.f : 0.f;
                    da[p][1] = xi.y > 0.f ? 1.f : 0.f;
                    xh[p][0] = xh[p][1] = 0.f;
                } else {
                    av[p][0] = xi.x;                 // pre[] is zero outside the image and beyond C already
                    av[p][1] = xi.y;
                    da[p][0] = da[p][1] = 1.f;
                    xh[p][0] = xh[p][1] = 0.f;
                }
            }
            if ((MODE == 1 || MODE == 2) && !interior) {
#pragma unroll
                for (int p = 0; p < P; p++) {
                    const bool ok = sy < g.TH && iy < g.H && ix + p < g.W;
                    av[p][0] = ok ? av[p][0] : 0.f;
                    av[p][1] = ok ? av[p][1] : 0.f;
                }
            }
            if (s + NW < nstrips) prefetch(s + NW);
            if (sy >= g.TH || iy >= g.H || ix >= g.W) continue;
            float acc[P][2];
#pragma unroll
            for (int p = 0; p < P; p++) { acc[p][0] = 0.f; acc[p][1] = 0.f; }
            if (S == 1) strip_bwd_s1<T, K, P, CPW>(tile, g.IW, sy, sx, cp, w, acc, av, wacc);
            else strip_bwd_s2<T, K, true, P, CPW, (K - 1) / 2 - DT, (K - 1) / 2 - DL>(tile, g.IW, sy, sx, cp, w, acc, av, wacc);
            if (chv) {
                const uint32_t off0 = (uint32_t)((iy * g.W + ix) * g.C + ch);
#pragma unroll
                for (int p = 0; p < P; p++) {
                    if (ix + p < g.W) {
                        if (MODE == 1 || MODE == 2) {
                            const uint32_t pk = pack2<T>(acc[p][0] * da[p][0], acc[p][1] * da[p][1]);
                            *reinterpret_cast<uint32_t*>(gx_n + off0 + (uint32_t)(p * g.C)) = pk;
                            const float2 r = unpack2<T>(pk);
                            a0 += r.x; a1 += r.y;
                            b0 = fmaf(r.x, xh[p][0], b0);
                            b1 = fmaf(r.y, xh[p][1], b1);
                        } else {
                            float v0 = acc[p][0], v1 = acc[p][1];
                            if (MODE == 3) { v0 *= da[p][0]; v1 *= da[p][1]; }
                            if (add) {
                                const float2 ad = unpack2<T>(__ldg(reinterpret_cast<const uint32_t*>(add + ioff + off0 + (uint32_t)(p * g.C))));
                                v0 += ad.x; v1 += ad.y;
                            }
                            *reinterpret_cast<uint32_t*>(gx_n + off0 + (uint32_t)(p * g.C)) = pack2<T>(v0, v1);
                        }
                    }
                }
            }
        }
    }
    if (MODE == 1 || MODE == 2) {
        double* p1 = stat_slot(ds1, g.C);
        double* p2 = stat_slot(ds2, g.C);
        reduce_warps_emit<CPW>(red, a0, a1, [&](int c, float v) { if (c0 + c < g.C) atomicAdd(p1 + c0 + c, (double)v); });
        reduce_warps_emit<CPW>(red, b0, b1, [&](int c, float v) { if (c0 + c < g.C) atomicAdd(p2 + c0 + c, (double)v); });
    }
    bn_bwd_finalize_tail(fin, threadIdx.x, NT);      // the last CTA turns the BN-backward sums into dgamma / dbeta / cA,cB,cC
    __syncthreads();      // every warp is done with the dy tile before it is reused
    // weight-gradient partials: the sub-strips of a warp are added first (lanes cp, cp + CPW, ... hold the same channel
    // pair), then all taps go through the (now free) tile memory in one go, [warp][tap][CW channels]
    float* wr = reinterpret_cast<float*>(tile);
#pragma unroll
    for (int i = 0; i < K * K; i++) {
        float v0 = wacc[i][0], v1 = wacc[i][1];
#pragma unroll
        for (int o = CPW; o < 32; o <<= 1) {
            v0 += __shfl_xor_sync(0xffffffffu, v0, o);
            v1 += __shfl_xor_sync(0xffffffffu, v1, o);
        }
        if (lane < CPW) {
            wr[(warp * K * K + i) * CW + cp * 2] = v0;
            wr[(warp * K * K + i) * CW + cp * 2 + 1] = v1;
        }
    }
    __syncthreads();
    constexpr int KKCW = K * K * CW;
    if (!g.part) {
        for (int e = threadIdx.x; e < KKCW; e += NT) {
            const int i = e / CW, c = e % CW;
            if (c0 + c < g.C) {
                float v = 0.f;
#pragma unroll
                for (int q = 0; q < NW; q++) v += wr[(q * K * K + i) * CW + c];
                const int tap = S == 1 ? (K * K - 1 - i) : i;
                atomicAdd(dW + (size_t)(c0 + c) * K * K + tap, v);
            }
        }
        return;
    }
    // ---- order-deterministic mode: this CTA's partial goes to its fixed slot, laid out like dW[c0 .. c0+CW) x taps ----
    float* slot = g.part + ((size_t)blockIdx.y * gridDim.x * gridDim.z + (size_t)blockIdx.x * gridDim.z + blockIdx.z) * KKCW;
    for (int e = threadIdx.x; e < KKCW; e += NT) {
        const int c = e / (K * K), tap = e - c * (K * K);            // consecutive threads -> consecutive slot words
        const int i = S == 1 ? (K * K - 1 - tap) : tap;
        float v = 0.f;
#pragma unroll
        for (int q = 0; q < NW; q++) v += wr[(q * K * K + i) * CW + c];
        slot[e] = v;
    }
}

// channel pairs per sub-strip of the hot kernels for a layer of C channels (see the lane mapping note at the top): 32 unless
// the last 64-channel block would idle a fifth or more of the lanes; then 16 (C = 32, 96, 144: best on the GPU this code
// was first tuned on, not re-measured on the H100; also where 8 would waste nothing), and 8 only where 16 would still idle
// a fifth (C = 16, 48). DFD_DW_CPW forces a value (diagnostics).
static int dw_cpw(int C) {
    static int forced = -1;
    if (forced < 0) { const char* e = getenv("DFD_DW_CPW"); forced = e ? atoi(e) : 0; }
    if (forced == 32 || forced == 16 || forced == 8) return forced;
    const int w32 = (C + 63) / 64 * 64 - C;
    if (w32 * 5 < C) return 32;
    const int w16 = (C + 31) / 32 * 32 - C;
    return w16 * 5 < C ? 16 : 8;
}

static int fill_geom(DwGeom& g, int N, int H, int W, int C, int K, int S, bool input_space, int cpw = 32) {
    // input_space: tiles partition the INPUT pixels (dgrad); the staged tile is then dy: shifted (S=1) or compact (S=2)
    g.N = N; g.H = H; g.W = W; g.C = C; g.pad = (K - 1) / 2;
    g.Ho = (H + 2 * g.pad - K) / S + 1;           // == ceil(H / S): also the extent of TF "SAME" padding
    g.Wo = (W + 2 * g.pad - K) / S + 1;
    int th_dim = input_space ? H : g.Ho, tw_dim = input_space ? W : g.Wo;
    int eff_s = input_space ? 1 : S;
    g.TW = tw_dim <= 8 ? 8 : ((tw_dim <= 16 || eff_s == 2) ? 16 : 32);   // stride-2 tiles stage 2x the columns
    g.TH = th_dim < 8 ? th_dim : 8;
    // forward k = 5 stride 2: an 8-row tile stages 19 x 35 pixels (85 KB) and leaves two 4-warp CTAs per SM; 4 rows double that
    if (!input_space && S == 2 && K == 5 && th_dim >= 8 && !getenv("DFD_DW_TH8")) g.TH = 4;
    if (input_space && S == 2) {
        g.IW = g.TW / 2 + 2;
        g.IH = (g.TH + 1) / 2 + 2;
    } else {
        g.IW = (g.TW - 1) * eff_s + K;
        g.IH = (g.TH - 1) * eff_s + K;
    }
    if (cpw < 32 && !(g.IW & 1)) g.IW++;      // odd tile width: the sub-strips of a warp (consecutive rows) use disjoint banks
    g.tiles_x = (tw_dim + g.TW - 1) / g.TW;
    g.tiles_y = (th_dim + g.TH - 1) / g.TH;
    { const char* e = getenv("DFD_DW_DBG"); g.dbg = e ? atoi(e) : 0; }
    g.part = nullptr;
    return g.IH * g.IW * cpw * (int)sizeof(uint32_t);
}

template <typename KernelT>
static int set_smem(KernelT k, int bytes) {
    cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e != cudaSuccess) return dfd_set_cuda_error(e, __FILE__, __LINE__);
    return DFD_OK;
}

}  // namespace

// CTA size per kernel size: k = 5 holds 50 weight registers per thread, so 128-thread CTAs let four of them (not two)
// share an SM's register file; overridable for experiments with DFD_DW_NT3 / DFD_DW_NT5 (128 or 256).
static int dw_nt(int k) {
    static int nt3 = 0, nt5 = 0;
    if (!nt3) {
        const char* e3 = getenv("DFD_DW_NT3");
        const char* e5 = getenv("DFD_DW_NT5");
        nt3 = (e3 && atoi(e3) == 128) ? 128 : 256;
        nt5 = (e5 && atoi(e5) == 256) ? 256 : 128;
    }
    return k == 5 ? nt5 : nt3;
}
#define DW_NT(K_, ...)                                                            \
    if (dw_nt(K_) == 128) { constexpr int NT = 128; __VA_ARGS__; }                \
    else { constexpr int NT = 256; __VA_ARGS__; }
#define DW_DISPATCH_KS(K_, S_, ...)                                               \
    if (K_ == 3 && S_ == 1) { constexpr int K = 3, S = 1; DW_NT(K_, __VA_ARGS__); }          \
    else if (K_ == 3 && S_ == 2) { constexpr int K = 3, S = 2; DW_NT(K_, __VA_ARGS__); }     \
    else if (K_ == 5 && S_ == 1) { constexpr int K = 5, S = 1; DW_NT(K_, __VA_ARGS__); }     \
    else if (K_ == 5 && S_ == 2) { constexpr int K = 5, S = 2; DW_NT(K_, __VA_ARGS__); }     \
    else return dfd_set_error(DFD_ERR_UNSUPPORTED, "depthwise conv: k in {3,5}, stride in {1,2}");

#define DW_DISPATCH_T(dt, ...)                                           \
    if ((dt) == DFD_DT_BF16) { typedef bf16 T; __VA_ARGS__; }            \
    else if ((dt) == DFD_DT_FP16) { typedef __half T; __VA_ARGS__; }     \
    else return dfd_set_error(DFD_ERR_ARG, "bad dtype");

#define DW_LAUNCH(kern, grid, smem, st, ...)                         \
    do {                                                             \
        auto kfn__ = kern;                                           \
        static bool attr_done__ = false;   /* once per instantiation: a per-launch value would be stale at graph replay */ \
        if (!attr_done__) {                                          \
            int rc__ = set_smem(kfn__, DW_MAX_SMEM);                 \
            if (rc__) return rc__;                                   \
            attr_done__ = true;                                      \
        }                                                            \
        if (smem > DW_MAX_SMEM) return dfd_set_error(DFD_ERR_UNSUPPORTED, "depthwise tile exceeds shared memory"); \
        kfn__<<<grid, NT, smem, st>>>(__VA_ARGS__);                  \
    } while (0)

extern "C" {

// out[N,Ho,Wo,C] = dwconv(act_in(scale*x + shift)); scale == NULL: x is consumed as is (act_in 0) or through a ReLU (act_in
// DFD_ACT_RELU). A BN input takes Swish, or ReLU (k = 3, stride 1, without output statistics).
// dsum/dsq (optional): per-channel sum / sum of squares of the rounded outputs (fp64, accumulated).
// dt_ / dl_: the top / left pad is (k-1)/2 - dt_ / (k-1)/2 - dl_ (TF "SAME", stride 2)
static int dw_fwd(const void* x, const float* scale, const float* shift, const float* w, void* out, int N, int H, int W,
                  int C, int k, int stride, int dt_, int dl_, int act_in, int dt, double* dsum, double* dsq,
                  const void* fin, void* stream) {
    if (C % 8 || N <= 0 || H <= 0 || W <= 0) return dfd_set_error(DFD_ERR_ARG, "dfd_dwconv_fwd: sizes");
    // a ReLU input, after a BN (scale != NULL) or alone: Xception's separable convolutions, k = 3 at stride 1, no BN behind
    const bool relu = act_in == DFD_ACT_RELU;
    if (relu && (k != 3 || stride != 1 || dt_ || dl_ || dsum || dsq || fin))
        return dfd_set_error(DFD_ERR_UNSUPPORTED, "dfd_dwconv_fwd: a ReLU input needs k = 3, stride 1 and no statistics");
    if (!relu && !scale && act_in != DFD_ACT_NONE) return dfd_set_error(DFD_ERR_ARG, "dfd_dwconv_fwd: act without BN");
    if (!relu && scale && act_in != DFD_ACT_SWISH) return dfd_set_error(DFD_ERR_UNSUPPORTED, "dfd_dwconv_fwd: BN input implies Swish");
    DwGeom g;
    const int cpw = dw_cpw(C);
    int smem = fill_geom(g, N, H, W, C, k, stride, false, cpw);
    // TF "SAME" pads: the staged halo (IH x IW) does not depend on the pads, only the tile origin moves. Instantiated for what
    // a plan launches: the stride-2 depthwise conv of an inverted-residual block (BN + Swish input) at the default CTA size
    if (dt_ || dl_) {
        if (stride != 2 || !scale || dw_nt(k) != (k == 5 ? 128 : 256))
            return dfd_set_error(DFD_ERR_UNSUPPORTED, "dfd_dwconv_fwd_pad: asymmetric pads need stride 2, a BN + Swish input and the default CTA size");
        dim3 grid(g.tiles_x * g.tiles_y, (C + 2 * cpw - 1) / (2 * cpw), N);
        cudaStream_t st = (cudaStream_t)stream;
#define FWP1(K_, CPW_, DT_, DL_) do { constexpr int NT = K_ == 5 ? 128 : 256;                                                  \
        DW_LAUNCH((dwconv_fwd_kernel<T, K_, 2, DFD_ACT_SWISH, true, NT, CPW_, DT_, DL_>), grid, smem, st, (const T*)x, scale, shift, w, \
                  (T*)out, dsum, dsq, (const BnFinDesc*)fin, g); } while (0)
#define FWP2(K_, DT_, DL_) do { if (cpw == 32) FWP1(K_, 32, DT_, DL_); else if (cpw == 16) FWP1(K_, 16, DT_, DL_); else FWP1(K_, 8, DT_, DL_); } while (0)
#define FWP(K_) do { if (dt_ && dl_) FWP2(K_, 1, 1); else if (dt_) FWP2(K_, 1, 0); else FWP2(K_, 0, 1); } while (0)
        DW_DISPATCH_T(dt, {
            if (k == 3) FWP(3);
            else if (k == 5) FWP(5);
            else return dfd_set_error(DFD_ERR_UNSUPPORTED, "depthwise conv: k in {3,5}, stride in {1,2}");
        });
#undef FWP
#undef FWP2
#undef FWP1
        DFD_LAUNCH_CHECK();
        return DFD_OK;
    }
    // one CTA per (tile, 2*cpw channels, image): walking several images per CTA (as the fused backward does) was slower
    // here on the GPU this code was first tuned on (not re-measured on the H100) - the forward has no per-CTA state worth amortising and loses the overlap between resident CTAs
    dim3 grid(g.tiles_x * g.tiles_y, (C + 2 * cpw - 1) / (2 * cpw), N);
    cudaStream_t st = (cudaStream_t)stream;
#define FW(ACT_, AFF_, CPW_) DW_LAUNCH((dwconv_fwd_kernel<T, K, S, ACT_, AFF_, NT, CPW_>), grid, smem, st, (const T*)x, scale, shift, w, (T*)out, dsum, dsq, (const BnFinDesc*)fin, g)
#define FWC(ACT_, AFF_) do { if (cpw == 32) FW(ACT_, AFF_, 32); else if (cpw == 16) FW(ACT_, AFF_, 16); else FW(ACT_, AFF_, 8); } while (0)
    if (relu) {
        DW_DISPATCH_T(dt, { constexpr int K = 3, S = 1; DW_NT(3, {
            if (scale) FWC(DFD_ACT_RELU, true);
            else FWC(DFD_ACT_RELU, false);
        }); });
        DFD_LAUNCH_CHECK();
        return DFD_OK;
    }
    DW_DISPATCH_T(dt, DW_DISPATCH_KS(k, stride, {
        if (scale) FWC(DFD_ACT_SWISH, true);
        else FWC(DFD_ACT_NONE, false);
    }));
#undef FWC
#undef FW
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

// TF "SAME" padding check of the `_pad` entry points: stride 1 takes the symmetric (k-1)/2 only; stride 2 also takes
// (k-1)/2 - 1 on a side whose extent is even (the output extent is ceil(extent / 2) either way)
static bool dw_pad_ok(int pad, int extent, int k, int stride) {
    const int sym = (k - 1) / 2;
    return pad == sym || (stride == 2 && pad == sym - 1 && extent % 2 == 0);
}

int dfd_dwconv_fwd(const void* x, const float* scale, const float* shift, const float* w, void* out, int N, int H,
                   int W, int C, int k, int stride, int act_in, int dt, double* dsum, double* dsq, const void* fin,
                   void* stream) {
    return dw_fwd(x, scale, shift, w, out, N, H, W, C, k, stride, 0, 0, act_in, dt, dsum, dsq, fin, stream);
}

// dfd_dwconv_fwd with the zero rows above (pad_t) and columns left (pad_l) of the image given: TF "SAME" padding
int dfd_dwconv_fwd_pad(const void* x, const float* scale, const float* shift, const float* w, void* out, int N, int H,
                       int W, int C, int k, int stride, int pad_t, int pad_l, int act_in, int dt, double* dsum, double* dsq,
                       const void* fin, void* stream) {
    if (!dw_pad_ok(pad_t, H, k, stride) || !dw_pad_ok(pad_l, W, k, stride))
        return dfd_set_error(DFD_ERR_ARG, "dfd_dwconv_fwd_pad: pads are (k-1)/2, or (k-1)/2 - 1 at stride 2 over an even extent");
    const int sym = (k - 1) / 2;
    return dw_fwd(x, scale, shift, w, out, N, H, W, C, k, stride, sym - pad_t, sym - pad_l, act_in, dt, dsum, dsq, fin, stream);
}

// Input gradient of the depthwise conv.
//   gy [N,Ho,Wo,C]: gradient w.r.t. the BN output behind the conv (cA != NULL: dy = cA*gy + cB*yout + cC is formed on load)
//   mode 0: gx = dgrad (+ add)                       (block input consumed directly)
//   mode 1: gx = dgrad * swish'(scale*xin + shift), and s1 += sum gx, s2 += sum gx * (xin-mean)*rstd
int dfd_dwconv_dgrad(const void* gy, const void* yout, const float* cA, const float* cB, const float* cC,
                     const float* w, const void* xin, const float* scale, const float* shift, const float* mean,
                     const float* rstd, const void* add, void* gx, int N, int H, int W, int C, int k, int stride,
                     int mode, int dt, double* s1, double* s2, void* stream) {
    if (C % 8 || N <= 0 || H <= 0 || W <= 0) return dfd_set_error(DFD_ERR_ARG, "dfd_dwconv_dgrad: sizes");
    if (mode == 1 && (!xin || !scale || !s1 || !s2)) return dfd_set_error(DFD_ERR_ARG, "dfd_dwconv_dgrad: mode 1 operands");
    DwGeom g;
    int smem = fill_geom(g, N, H, W, C, k, stride, true);
    dim3 grid(g.tiles_x * g.tiles_y, (C + CB - 1) / CB, N);
    cudaStream_t st = (cudaStream_t)stream;
#define DG(MODE, AFF) DW_LAUNCH((dwconv_dgrad_kernel<T, K, S, MODE, AFF, NT>), grid, smem, st, (const T*)gy, (const T*)yout, cA, cB, cC, w, (const T*)xin, scale, shift, mean, rstd, (const T*)add, (T*)gx, s1, s2, g)
    DW_DISPATCH_T(dt, DW_DISPATCH_KS(k, stride, {
        if (mode == 1) { if (cA) DG(1, true); else DG(1, false); }
        else { if (cA) DG(0, true); else DG(0, false); }
    }));
#undef DG
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

// dW[C,1,k,k] (fp32, accumulated with atomics) of the depthwise conv; operands as in fwd / dgrad.
int dfd_dwconv_wgrad(const void* x, const float* scale, const float* shift, const void* gy, const void* yout,
                     const float* cA, const float* cB, const float* cC, float* dW, int N, int H, int W, int C, int k,
                     int stride, int dt, void* stream) {
    if (C % 8 || N <= 0 || H <= 0 || W <= 0) return dfd_set_error(DFD_ERR_ARG, "dfd_dwconv_wgrad: sizes");
    DwGeom g;
    int smem = fill_geom(g, N, H, W, C, k, stride, false);
    int tiles = g.tiles_x * g.tiles_y, cbs = (C + CB - 1) / CB;
    int gz = (DFD_SMS * 6 + tiles * cbs - 1) / (tiles * cbs);
    if (gz > N) gz = N;
    if (gz < 1) gz = 1;
    dim3 grid(tiles, cbs, gz);
    cudaStream_t st = (cudaStream_t)stream;
#define WG(ACT, AIN, AG) DW_LAUNCH((dwconv_wgrad_kernel<T, K, S, ACT, AIN, AG, NT>), grid, smem, st, (const T*)x, scale, shift, (const T*)gy, (const T*)yout, cA, cB, cC, dW, g)
    DW_DISPATCH_T(dt, DW_DISPATCH_KS(k, stride, {
        if (scale) { if (cA) WG(DFD_ACT_SWISH, true, true); else WG(DFD_ACT_SWISH, true, false); }
        else { if (cA) WG(DFD_ACT_NONE, false, true); else WG(DFD_ACT_NONE, false, false); }
    }));
#undef WG
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

// Fused backward of a depthwise stage: dfd_dwconv_dgrad and dfd_dwconv_wgrad in one pass over the dy tile (operands as
// there; dW accumulated). scale != NULL: the stage input is BN + Swish of `xin` (mode 1: every MBConv block with an
// expansion, `add` unused); scale == NULL: `xin` is consumed as is (mode 0: DS block), gx = dgrad (+ add).
// grid of the fused backward: (tiles, 64-channel blocks, image groups); enough CTAs for ~6 per SM, each walking N / gz images
// (gz a divisor of N keeps them balanced)
static void dw_bwd_grid(const DwGeom& g, int N, int C, int cpw, int& tiles, int& cbs, int& gz) {
    tiles = g.tiles_x * g.tiles_y;
    cbs = (C + 2 * cpw - 1) / (2 * cpw);
    gz = (DFD_SMS * 6 + tiles * cbs - 1) / (tiles * cbs);
    if (gz > N) gz = N;
    while (gz < N && N % gz) gz++;
}
// channels per CTA (= per partial slot / per reduce entry) of the depthwise kernels for a layer of C channels: 64, 32 or 16
int dfd_dwconv_block_channels(int C) { return C > 0 ? 2 * dw_cpw(C) : 0; }

// partial slots per channel block that the order-deterministic mode of dfd_dwconv_bwd writes (tiles x image groups); the
// workspace holds ceil(C / B) x that x B*k*k floats, B = dfd_dwconv_block_channels(C)
int dfd_dwconv_bwd_parts(int N, int H, int W, int C, int k, int stride) {
    if (C % 8 || N <= 0 || H <= 0 || W <= 0 || (k != 3 && k != 5) || (stride != 1 && stride != 2)) return 0;
    DwGeom g;
    const int cpw = dw_cpw(C);
    fill_geom(g, N, H, W, C, k, stride, true, cpw);
    int tiles, cbs, gz;
    dw_bwd_grid(g, N, C, cpw, tiles, cbs, gz);
    return tiles * gz;
}

// dt_ / dl_: the top / left pad is (k-1)/2 - dt_ / (k-1)/2 - dl_ (stride 2 only, see strip_bwd_s2)
static int dw_bwd(const void* gy, const void* yout, const float* cA, const float* cB, const float* cC,
                  const float* w, const void* xin, const float* scale, const float* shift, const float* mean,
                  const float* rstd, const void* add, void* gx, float* dW, int N, int H, int W, int C, int k,
                  int stride, int dt_, int dl_, int dt, double* s1, double* s2, void* ws, long long ws_bytes, const void* fin,
                  void* stream, bool relu = false) {
    if (C % 8 || N <= 0 || H <= 0 || W <= 0) return dfd_set_error(DFD_ERR_ARG, "dfd_dwconv_bwd: sizes");
    if (relu && (k != 3 || stride != 1 || cA || dt_ || dl_))
        return dfd_set_error(DFD_ERR_UNSUPPORTED, "dfd_dwconv_bwd_relu: k = 3, stride 1, the BN backward not folded into gy (cA NULL)");
    if (!xin || !dW) return dfd_set_error(DFD_ERR_ARG, "dfd_dwconv_bwd: operands");
    if (scale && (!shift || !mean || !rstd || !s1 || !s2)) return dfd_set_error(DFD_ERR_ARG, "dfd_dwconv_bwd: mode 1 operands");
    DwGeom g;
    const int cpw = dw_cpw(C);
    int smem = fill_geom(g, N, H, W, C, k, stride, true, cpw);
    constexpr int NT = 128;
    const int red_bytes = (NT / 32) * k * k * 2 * cpw * (int)sizeof(float);
    if (smem < red_bytes) smem = red_bytes;
    int tiles, cbs, gz;
    dw_bwd_grid(g, N, C, cpw, tiles, cbs, gz);
    if (ws) {
        if ((long long)cbs * tiles * gz * k * k * 2 * cpw * 4 > ws_bytes)
            return dfd_set_error(DFD_ERR_ARG, "dfd_dwconv_bwd: workspace too small (blocks x dfd_dwconv_bwd_parts x block_channels*k*k floats)");
        g.part = (float*)ws;
    }
    dim3 grid(tiles, cbs, gz);
    cudaStream_t st = (cudaStream_t)stream;
    // strip width per kernel size: 4 for k = 3 (four CTAs per SM), 8 for k = 5, chosen on the GPU this code was first tuned
    // on (not re-measured on the H100); DFD_DW_PB3 / DFD_DW_PB5 override
    static int pb3 = 0, pb5 = 0;
    if (!pb3) { const char* e3 = getenv("DFD_DW_PB3"); const char* e5 = getenv("DFD_DW_PB5"); pb3 = (e3 && atoi(e3) == 8) ? 8 : 4; pb5 = (e5 && atoi(e5) == 4) ? 4 : 8; }
    const int pb = k == 3 ? pb3 : pb5;
#define BWARGS (const T*)gy, (const T*)yout, cA, cB, cC, w, (const T*)xin, scale, shift, mean, rstd, (const T*)add, (T*)gx, dW, s1, s2, (const BnBwdFinDesc*)fin, g
    // narrow lane groups (cpw 16 / 8) are instantiated for the default strip width of each kernel size only
#define BW1(K_, S_, AFF, MODE_) do {                                                                                          \
        constexpr int PD = K_ == 3 ? 4 : 8;                                                                                   \
        if (cpw == 16) DW_LAUNCH((dwconv_bwd_kernel<T, K_, S_, AFF, MODE_, NT, PD, 16>), grid, smem, st, BWARGS);             \
        else if (cpw == 8) DW_LAUNCH((dwconv_bwd_kernel<T, K_, S_, AFF, MODE_, NT, PD, 8>), grid, smem, st, BWARGS);          \
        else if (pb == 4) DW_LAUNCH((dwconv_bwd_kernel<T, K_, S_, AFF, MODE_, NT, 4>), grid, smem, st, BWARGS);               \
        else DW_LAUNCH((dwconv_bwd_kernel<T, K_, S_, AFF, MODE_, NT, 8>), grid, smem, st, BWARGS);                            \
    } while (0)
#define BW(K_, S_) do { if (scale) { if (cA) BW1(K_, S_, true, 1); else BW1(K_, S_, false, 1); } else { if (cA) BW1(K_, S_, true, 0); else BW1(K_, S_, false, 0); } } while (0)
    // TF "SAME" pads (one side one element short): instantiated for what a plan launches - the stride-2 depthwise stage of an
    // inverted-residual block (BN + Swish input, BN backward folded into dy) at the default strip width of each kernel size
#define BWP1(K_, DT_, DL_) do {                                                                                               \
        constexpr int PD = K_ == 3 ? 4 : 8;                                                                                   \
        if (cpw == 16) DW_LAUNCH((dwconv_bwd_kernel<T, K_, 2, true, 1, NT, PD, 16, DT_, DL_>), grid, smem, st, BWARGS);       \
        else if (cpw == 8) DW_LAUNCH((dwconv_bwd_kernel<T, K_, 2, true, 1, NT, PD, 8, DT_, DL_>), grid, smem, st, BWARGS);    \
        else DW_LAUNCH((dwconv_bwd_kernel<T, K_, 2, true, 1, NT, PD, 32, DT_, DL_>), grid, smem, st, BWARGS);                 \
    } while (0)
#define BWP(K_) do { if (dt_ && dl_) BWP1(K_, 1, 1); else if (dt_) BWP1(K_, 1, 0); else BWP1(K_, 0, 1); } while (0)
    if (dt_ || dl_) {
        if (stride != 2 || !scale || !cA)
            return dfd_set_error(DFD_ERR_UNSUPPORTED, "dfd_dwconv_bwd_pad: asymmetric pads need stride 2, a BN + Swish input and cA");
        DW_DISPATCH_T(dt, {
            if (k == 3) BWP(3);
            else if (k == 5) BWP(5);
            else return dfd_set_error(DFD_ERR_UNSUPPORTED, "depthwise conv: k in {3,5}, stride in {1,2}");
        });
        DFD_LAUNCH_CHECK();
        return DFD_OK;
    }
    if (relu) {
        DW_DISPATCH_T(dt, { if (scale) BW1(3, 1, false, 2); else BW1(3, 1, false, 3); });
        DFD_LAUNCH_CHECK();
        return DFD_OK;
    }
    DW_DISPATCH_T(dt, {
        if (k == 3 && stride == 1) BW(3, 1);
        else if (k == 3 && stride == 2) BW(3, 2);
        else if (k == 5 && stride == 1) BW(5, 1);
        else if (k == 5 && stride == 2) BW(5, 2);
        else return dfd_set_error(DFD_ERR_UNSUPPORTED, "depthwise conv: k in {3,5}, stride in {1,2}");
    });
#undef BWP
#undef BWP1
#undef BW
#undef BW1
#undef BWARGS
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

int dfd_dwconv_bwd(const void* gy, const void* yout, const float* cA, const float* cB, const float* cC,
                   const float* w, const void* xin, const float* scale, const float* shift, const float* mean,
                   const float* rstd, const void* add, void* gx, float* dW, int N, int H, int W, int C, int k,
                   int stride, int dt, double* s1, double* s2, void* ws, long long ws_bytes, const void* fin, void* stream) {
    return dw_bwd(gy, yout, cA, cB, cC, w, xin, scale, shift, mean, rstd, add, gx, dW, N, H, W, C, k, stride, 0, 0, dt, s1, s2,
                  ws, ws_bytes, fin, stream);
}

// dfd_dwconv_bwd of a depthwise stage whose input passes a ReLU (Xception's separable convolutions; k = 3, stride 1, cA NULL):
// scale != NULL: the input is relu(scale*xin + shift), gx = dgrad * 1[relu > 0] with the BN-backward sums s1 / s2 of gx;
// scale == NULL: the input is relu(xin), gx = dgrad * 1[xin > 0] (+ add). dW and the workspace as in dfd_dwconv_bwd.
int dfd_dwconv_bwd_relu(const void* gy, const void* yout, const float* cA, const float* cB, const float* cC,
                        const float* w, const void* xin, const float* scale, const float* shift, const float* mean,
                        const float* rstd, const void* add, void* gx, float* dW, int N, int H, int W, int C, int k,
                        int stride, int dt, double* s1, double* s2, void* ws, long long ws_bytes, const void* fin, void* stream) {
    return dw_bwd(gy, yout, cA, cB, cC, w, xin, scale, shift, mean, rstd, add, gx, dW, N, H, W, C, k, stride, 0, 0, dt, s1, s2,
                  ws, ws_bytes, fin, stream, true);
}

// dfd_dwconv_bwd of a stage padded with pad_t rows above and pad_l columns left of the image (TF "SAME", as in
// dfd_dwconv_fwd_pad); the workspace layout and dfd_dwconv_bwd_parts do not depend on the pads
int dfd_dwconv_bwd_pad(const void* gy, const void* yout, const float* cA, const float* cB, const float* cC,
                       const float* w, const void* xin, const float* scale, const float* shift, const float* mean,
                       const float* rstd, const void* add, void* gx, float* dW, int N, int H, int W, int C, int k,
                       int stride, int pad_t, int pad_l, int dt, double* s1, double* s2, void* ws, long long ws_bytes,
                       const void* fin, void* stream) {
    if (!dw_pad_ok(pad_t, H, k, stride) || !dw_pad_ok(pad_l, W, k, stride))
        return dfd_set_error(DFD_ERR_ARG, "dfd_dwconv_bwd_pad: pads are (k-1)/2, or (k-1)/2 - 1 at stride 2 over an even extent");
    const int sym = (k - 1) / 2;
    return dw_bwd(gy, yout, cA, cB, cC, w, xin, scale, shift, mean, rstd, add, gx, dW, N, H, W, C, k, stride, sym - pad_t,
                  sym - pad_l, dt, s1, s2, ws, ws_bytes, fin, stream);
}

}  // extern "C"
