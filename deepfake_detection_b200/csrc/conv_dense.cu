// ResNet-side kernels: dense k x k convolution as (im2col -> tensor-core GEMM), its backward (GEMM -> col2im, GEMM wgrad
// on the im2col matrix), weight / gradient layout changes between OIHW and the GEMM's [Cout][kh][kw][Cin], 3x3/s2
// max-pool forward/backward, ReLU-mask and global-pool (avg, and max / avgmax / catavgmax by argmax) backward.
//   ResNet.forward            dfd/timm/models/resnet.py:450-468 (conv1 7x7 -> bn -> relu -> maxpool 3x3 s2 p1 :379-382)
//   BasicBlock / Bottleneck   resnet.py:150-175, :215-246 (3x3 convs :129-136,:195-197; downsample 1x1 s2 :249-260)
// Round-1 scope note: the 3x3 convolutions go through a MATERIALISED im2col matrix (9x the activation bytes). It is
// correct and runs on the tensor-core GEMM, but it is not the final design: the implicit-GEMM kernel with TMA im2col
// descriptors replaces im2col/col2im next (DESIGN.md section 6).
#include "common.cuh"

namespace {

// cols[m, (kh*k + kw)*C + c] = x[n, oy*s - pad + kh, ox*s - pad + kw, c]  (zero outside), m = (n, oy, ox)
template <typename T>
__global__ void im2col_kernel(const T* __restrict__ x, T* __restrict__ cols, int N, int H, int W, int C, int k, int s,
                              int pad, int Ho, int Wo) {
    const int V = C / 8;
    const long long total = (long long)N * Ho * Wo * k * k * V;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        int v = (int)(i % V);
        long long t = i / V;
        int tap = (int)(t % (k * k));
        long long m = t / (k * k);
        int ox = (int)(m % Wo);
        long long t2 = m / Wo;
        int oy = (int)(t2 % Ho);
        int n = (int)(t2 / Ho);
        int kh = tap / k, kw = tap - kh * k;
        int iy = oy * s - pad + kh, ix = ox * s - pad + kw;
        uint4 val = make_uint4(0, 0, 0, 0);
        if (iy >= 0 && iy < H && ix >= 0 && ix < W) val = ldg16(x + (((size_t)n * H + iy) * W + ix) * C + v * 8);
        stg16(cols + ((size_t)m * k * k + tap) * C + v * 8, val);
    }
}

// dx[n, iy, ix, c] = sum over (oy, ox, kh, kw) with oy*s - pad + kh == iy, ox*s - pad + kw == ix of dcols[m, tap, c]
// (+ add[n,iy,ix,c]).  Gather form: no atomics, deterministic.
template <typename T>
__global__ void col2im_kernel(const T* __restrict__ dcols, const T* __restrict__ add, T* __restrict__ dx, int N, int H,
                              int W, int C, int k, int s, int pad, int Ho, int Wo) {
    const int V = C / 8;
    const long long total = (long long)N * H * W * V;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        int v = (int)(i % V);
        long long t = i / V;
        int ix = (int)(t % W);
        long long t2 = t / W;
        int iy = (int)(t2 % H);
        int n = (int)(t2 / H);
        float acc[8];
#pragma unroll
        for (int j = 0; j < 8; j++) acc[j] = 0.f;
        if (add) unpack8<T>(ldg16(add + (size_t)t * C + v * 8), acc);
        for (int kh = 0; kh < k; kh++) {
            int a = iy + pad - kh;
            if (a < 0 || a % s) continue;
            int oy = a / s;
            if (oy >= Ho) continue;
            for (int kw = 0; kw < k; kw++) {
                int b = ix + pad - kw;
                if (b < 0 || b % s) continue;
                int ox = b / s;
                if (ox >= Wo) continue;
                size_t m = ((size_t)n * Ho + oy) * Wo + ox;
                float f[8];
                unpack8<T>(ldg16(dcols + (m * k * k + kh * k + kw) * C + v * 8), f);
#pragma unroll
                for (int j = 0; j < 8; j++) acc[j] += f[j];
            }
        }
        stg16(dx + (size_t)t * C + v * 8, pack8<T>(acc));
    }
}

struct RepackDesc {
    const void* src;   // 16-bit [O][I][k][k]  (or fp32 permuted gradient for the inverse)
    void* dst;         // 16-bit [O][k][k][I]
    void* dstT;        // 16-bit [k][k][I][O] = transpose of dst as a [O, k*k*I] matrix (dgrad B operand), may be null
    void* dstD;        // 16-bit [I][k'][k'][O] with flipped taps (kh' = k-1-kh): B operand of the implicit-GEMM dgrad, may be null
    int O, I, k, pad_;
};
// weights: OIHW 16-bit -> [O][kh][kw][I] (GEMM B operand), its transpose [(kh,kw,I)][O] and the tap-flipped [I][kh'][kw'][O].
// One pass per destination layout, each walking ITS OWN element order so that the 2-byte stores of a warp are contiguous
// (a single pass in dst order scattered the other two layouts with a stride of O elements); the strided source reads of the later passes hit L2.
template <typename T>
__global__ void repack_weights_kernel(const RepackDesc* __restrict__ table) {
    RepackDesc d = table[blockIdx.y];
    const T* src = (const T*)d.src;
    T* dst = (T*)d.dst;
    T* dstT = (T*)d.dstT;
    T* dstD = (T*)d.dstD;
    const int kk = d.k * d.k;
    const long long total = (long long)d.O * d.I * kk;
    const long long step = (long long)gridDim.x * blockDim.x, i0 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (dst) {
#pragma unroll 4
        for (long long i = i0; i < total; i += step) {          // i = (o*kk + tap)*I + ci
            const int ci = (int)(i % d.I);
            const long long t = i / d.I;
            const int tap = (int)(t % kk), o = (int)(t / kk);
            dst[i] = src[((size_t)o * d.I + ci) * kk + tap];
        }
    }
    if (dstT) {
#pragma unroll 4
        for (long long i = i0; i < total; i += step) {          // i = (tap*I + ci)*O + o
            const int o = (int)(i % d.O);
            const long long t = i / d.O;
            const int ci = (int)(t % d.I), tap = (int)(t / d.I);
            dstT[i] = src[((size_t)o * d.I + ci) * kk + tap];
        }
    }
    if (dstD) {
#pragma unroll 4
        for (long long i = i0; i < total; i += step) {          // i = (ci*kk + tap')*O + o, tap' = kk-1-tap
            const int o = (int)(i % d.O);
            const long long t = i / d.O;
            const int tapf = (int)(t % kk), ci = (int)(t / kk);
            dstD[i] = src[((size_t)o * d.I + ci) * kk + (kk - 1 - tapf)];
        }
    }
}
// gradients: fp32 [O][kh][kw][I] (wgrad GEMM output) accumulated into the OIHW fp32 arena
__global__ void unpack_grad_kernel(const float* __restrict__ gperm, float* __restrict__ g_oihw, int O, int I, int k) {
    const int kk = k * k;
    const long long total = (long long)O * I * kk;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        int tap = (int)(i % kk);
        long long t = i / kk;
        int ci = (int)(t % I);
        int o = (int)(t / I);
        g_oihw[i] += gperm[((size_t)o * kk + tap) * I + ci];
    }
}

// 3x3 stride-2 max-pool WITHOUT padding in ceil mode (SENet's layer0.pool, senet.py:297-299: nn.MaxPool2d(3, 2,
// ceil_mode=True)): Ho = ceil((H - 3) / 2) + 1, so over an even extent the last window starts at H - 2 and is clipped to two
// rows. Arg-max byte and first-maximum tie-break as maxpool_fwd_kernel.
template <typename T>
__global__ void maxpool_ceil_fwd_kernel(const T* __restrict__ x, T* __restrict__ out, unsigned char* __restrict__ idx, int N,
                                        int H, int W, int C, int Ho, int Wo) {
    const int V = C / 8;
    const long long total = (long long)N * Ho * Wo * V;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        int v = (int)(i % V);
        long long t = i / V;
        int ox = (int)(t % Wo);
        long long t2 = t / Wo;
        int oy = (int)(t2 % Ho);
        int n = (int)(t2 / Ho);
        float best[8];
        unsigned char bi[8];
#pragma unroll
        for (int j = 0; j < 8; j++) { best[j] = -INFINITY; bi[j] = 0; }
        for (int kh = 0; kh < 3; kh++) {
            int iy = oy * 2 + kh;
            if (iy >= H) break;
            for (int kw = 0; kw < 3; kw++) {
                int ix = ox * 2 + kw;
                if (ix >= W) break;
                float f[8];
                unpack8<T>(ldg16(x + (((size_t)n * H + iy) * W + ix) * C + v * 8), f);
#pragma unroll
                for (int j = 0; j < 8; j++)
                    if (f[j] > best[j]) { best[j] = f[j]; bi[j] = (unsigned char)(kh * 3 + kw); }
            }
        }
        stg16(out + (size_t)t * C + v * 8, pack8<T>(best));
        uint2 pk;
        pk.x = bi[0] | (bi[1] << 8) | (bi[2] << 16) | (bi[3] << 24);
        pk.y = bi[4] | (bi[5] << 8) | (bi[6] << 16) | (bi[7] << 24);
        *reinterpret_cast<uint2*>(idx + (size_t)t * C + v * 8) = pk;
    }
}
// its gradient, gathered per input pixel (no atomics): gx[iy, ix] = sum of gy over the windows (oy, ox) with iy = 2 oy + kh,
// ix = 2 ox + kw whose arg-max is (kh, kw)
template <typename T>
__global__ void maxpool_ceil_bwd_kernel(const T* __restrict__ gy, const unsigned char* __restrict__ idx, T* __restrict__ gx,
                                        int N, int H, int W, int C, int Ho, int Wo) {
    const int V = C / 8;
    const long long total = (long long)N * H * W * V;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        int v = (int)(i % V);
        long long t = i / V;
        int ix = (int)(t % W);
        long long t2 = t / W;
        int iy = (int)(t2 % H);
        int n = (int)(t2 / H);
        float acc[8];
#pragma unroll
        for (int j = 0; j < 8; j++) acc[j] = 0.f;
        for (int kh = 0; kh < 3; kh++) {
            int a = iy - kh;
            if (a < 0 || (a & 1)) continue;
            int oy = a >> 1;
            if (oy >= Ho) continue;
            for (int kw = 0; kw < 3; kw++) {
                int b = ix - kw;
                if (b < 0 || (b & 1)) continue;
                int ox = b >> 1;
                if (ox >= Wo) continue;
                size_t o = (((size_t)n * Ho + oy) * Wo + ox) * C + v * 8;
                uint2 pk = *reinterpret_cast<const uint2*>(idx + o);
                float g[8];
                unpack8<T>(ldg16(gy + o), g);
                const unsigned char want = (unsigned char)(kh * 3 + kw);
#pragma unroll
                for (int j = 0; j < 8; j++) {
                    unsigned char bj = (unsigned char)(((j < 4 ? pk.x : pk.y) >> ((j & 3) * 8)) & 0xff);
                    if (bj == want) acc[j] += g[j];
                }
            }
        }
        stg16(gx + (size_t)t * C + v * 8, pack8<T>(acc));
    }
}

// 3x3 stride-2 pad-1 max-pool; the arg-max (first maximum in row-major window order, as ATen's CPU/CUDA kernels) is kept
// in one byte per output so that backward routes ties (frequent after ReLU) exactly like the reference.
template <typename T>
__global__ void maxpool_fwd_kernel(const T* __restrict__ x, T* __restrict__ out, unsigned char* __restrict__ idx, int N,
                                   int H, int W, int C, int Ho, int Wo) {
    const int V = C / 8;
    const long long total = (long long)N * Ho * Wo * V;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        int v = (int)(i % V);
        long long t = i / V;
        int ox = (int)(t % Wo);
        long long t2 = t / Wo;
        int oy = (int)(t2 % Ho);
        int n = (int)(t2 / Ho);
        float best[8];
        unsigned char bi[8];
#pragma unroll
        for (int j = 0; j < 8; j++) { best[j] = -INFINITY; bi[j] = 0; }
        for (int kh = 0; kh < 3; kh++) {
            int iy = oy * 2 - 1 + kh;
            if (iy < 0 || iy >= H) continue;
            for (int kw = 0; kw < 3; kw++) {
                int ix = ox * 2 - 1 + kw;
                if (ix < 0 || ix >= W) continue;
                float f[8];
                unpack8<T>(ldg16(x + (((size_t)n * H + iy) * W + ix) * C + v * 8), f);
#pragma unroll
                for (int j = 0; j < 8; j++)
                    if (f[j] > best[j]) { best[j] = f[j]; bi[j] = (unsigned char)(kh * 3 + kw); }
            }
        }
        stg16(out + (size_t)t * C + v * 8, pack8<T>(best));
        uint2 pk;
        pk.x = bi[0] | (bi[1] << 8) | (bi[2] << 16) | (bi[3] << 24);
        pk.y = bi[4] | (bi[5] << 8) | (bi[6] << 16) | (bi[7] << 24);
        *reinterpret_cast<uint2*>(idx + (size_t)t * C + v * 8) = pk;
    }
}
template <typename T>
__global__ void maxpool_bwd_kernel(const T* __restrict__ gy, const unsigned char* __restrict__ idx, T* __restrict__ gx,
                                   int N, int H, int W, int C, int Ho, int Wo) {
    const int V = C / 8;
    const long long total = (long long)N * H * W * V;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        int v = (int)(i % V);
        long long t = i / V;
        int ix = (int)(t % W);
        long long t2 = t / W;
        int iy = (int)(t2 % H);
        int n = (int)(t2 / H);
        float acc[8];
#pragma unroll
        for (int j = 0; j < 8; j++) acc[j] = 0.f;
        for (int kh = 0; kh < 3; kh++) {
            int a = iy + 1 - kh;
            if (a < 0 || (a & 1)) continue;
            int oy = a >> 1;
            if (oy >= Ho) continue;
            for (int kw = 0; kw < 3; kw++) {
                int b = ix + 1 - kw;
                if (b < 0 || (b & 1)) continue;
                int ox = b >> 1;
                if (ox >= Wo) continue;
                size_t o = (((size_t)n * Ho + oy) * Wo + ox) * C + v * 8;
                uint2 pk = *reinterpret_cast<const uint2*>(idx + o);
                float g[8];
                unpack8<T>(ldg16(gy + o), g);
                const unsigned char want = (unsigned char)(kh * 3 + kw);
#pragma unroll
                for (int j = 0; j < 8; j++) {
                    unsigned char bj = (unsigned char)(((j < 4 ? pk.x : pk.y) >> ((j & 3) * 8)) & 0xff);
                    if (bj == want) acc[j] += g[j];
                }
            }
        }
        stg16(gx + (size_t)t * C + v * 8, pack8<T>(acc));
    }
}

// gm = g * (out > 0): gradient through the ReLU that follows the residual add (resnet.py:173,244)
template <typename T>
__global__ void relu_bwd_kernel(const T* __restrict__ g, const T* __restrict__ out, T* __restrict__ gm, size_t nvec) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (size_t)gridDim.x * blockDim.x) {
        float a[8], o[8];
        unpack8<T>(ldg16(g + i * 8), a);
        unpack8<T>(ldg16(out + i * 8), o);
#pragma unroll
        for (int j = 0; j < 8; j++) a[j] = o[j] > 0.f ? a[j] : 0.f;
        stg16(gm + i * 8, pack8<T>(a));
    }
}
// dout[n, hw, c] = dpooled[n, c] / HW   (backward of the global average pool that feeds the classifier)
template <typename T>
__global__ void pool_bwd_kernel(const float* __restrict__ dpooled, T* __restrict__ dout, int N, long long hw, int C) {
    const int V = C / 8;
    const long long total = (long long)N * hw * V;
    const float inv = 1.f / (float)hw;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        int v = (int)(i % V);
        long long t = i / V;
        int n = (int)(t / hw);
        float f[8];
#pragma unroll
        for (int j = 0; j < 8; j++) f[j] = dpooled[(size_t)n * C + v * 8 + j] * inv;
        stg16(dout + (size_t)t * C + v * 8, pack8<T>(f));
    }
}
// dout[n, hw, c] = g_avg[n, c] / HW + (hw == argmax[n, c]) * g_max[n, c]   (backward of the max / avgmax / catavgmax global
// pool; g_avg / g_max are read from dpooled [N, P] by pool type, as dfd_act_bwd_gpool does)
template <typename T>
__global__ void gpool_bwd_kernel(const float* __restrict__ dpooled, const int* __restrict__ argmax, T* __restrict__ dout, int N,
                                 long long hw, int C, int pool_type) {
    const int V = C / 8;
    const long long total = (long long)N * hw * V;
    const float inv = 1.f / (float)hw;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        int v = (int)(i % V);
        long long t = i / V;
        int n = (int)(t / hw);
        const long long p = t - (long long)n * hw;
        float f[8];
#pragma unroll
        for (int j = 0; j < 8; j++) {
            const int c = v * 8 + j;
            float ga, gm;
            if (pool_type == DFD_POOL_CATAVGMAX) {
                ga = dpooled[(size_t)n * 2 * C + c];
                gm = dpooled[(size_t)n * 2 * C + C + c];
            } else {
                const float d = dpooled[(size_t)n * C + c];
                ga = pool_type == DFD_POOL_AVGMAX ? 0.5f * d : 0.f;
                gm = pool_type == DFD_POOL_AVGMAX ? 0.5f * d : d;
            }
            const float a = ga * inv;
            f[j] = p == (long long)argmax[(size_t)n * C + c] ? a + gm : a;
        }
        stg16(dout + (size_t)t * C + v * 8, pack8<T>(f));
    }
}

// ---- stem as a GEMM: im2col of the NCHW image in (ci, kh, kw) column order (== OIHW flattening), K padded to a multiple of 8.
// One CTA per output row: the Cin x k input rows it needs are staged (zero-padded) in shared memory with coalesced reads,
// then every thread assembles 16-byte column groups from it (a per-thread 2-byte gather from global is request-bound).
// pad_t / pad_l: zero rows above / columns left of the image; WP: staged (padded) row width, >= (Wo - 1) * s + k.
template <typename T>
__device__ __forceinline__ void stem_im2col_body(const T* __restrict__ x, T* __restrict__ cols, int N, int Cin, int H, int W,
                                                 int k, int s, int pad_t, int pad_l, int WP, int Ho, int Wo, int Kp) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int taps = Cin * k * k;
    T* rows = reinterpret_cast<T*>(smem_raw);        // [Cin][k][WP]
    int* offs = reinterpret_cast<int*>(smem_raw + (((size_t)Cin * k * WP * sizeof(T) + 15) & ~(size_t)15));   // [Kp]
    const int oy = blockIdx.x % Ho, n = blockIdx.x / Ho;
    const T* img = x + (size_t)n * Cin * H * W;
    for (int i = threadIdx.x; i < Cin * k * WP; i += blockDim.x) {
        const int px = i % WP, r = i / WP;           // r = ci * k + kh
        const int kh = r % k, ci = r / k;
        const int iy = oy * s - pad_t + kh, ix = px - pad_l;
        rows[i] = (iy >= 0 && iy < H && ix >= 0 && ix < W) ? img[((size_t)ci * H + iy) * W + ix] : from_f<T>(0.f);
    }
    for (int t = threadIdx.x; t < Kp; t += blockDim.x) {
        int o = -1;
        if (t < taps) {
            const int ci = t / (k * k), r = t - ci * k * k;
            const int kh = r / k, kw = r - kh * k;
            o = (ci * k + kh) * WP + kw;
        }
        offs[t] = o;
    }
    __syncthreads();
    const int G = Kp / 8;
    T* out = cols + ((size_t)n * Ho + oy) * Wo * Kp;
    for (int i = threadIdx.x; i < Wo * G; i += blockDim.x) {
        const int g = i % G, ox = i / G;
        T vals[8];
#pragma unroll
        for (int j = 0; j < 8; j++) {
            const int o = offs[g * 8 + j];
            vals[j] = o >= 0 ? rows[o + ox * s] : from_f<T>(0.f);
        }
        stg16(out + (size_t)ox * Kp + g * 8, *reinterpret_cast<const uint4*>(vals));
    }
}
// symmetric padding (the EfficientNet and ResNet stems)
template <typename T>
__global__ void stem_im2col_kernel(const T* __restrict__ x, T* __restrict__ cols, int N, int Cin, int H, int W, int k, int s,
                                   int pad, int Ho, int Wo, int Kp) {
    stem_im2col_body(x, cols, N, Cin, H, W, k, s, pad, pad, W + 2 * pad, Ho, Wo, Kp);
}
// TF "SAME" padding (dfd_stem_im2col_pad)
template <typename T>
__global__ void stem_im2col_same_kernel(const T* __restrict__ x, T* __restrict__ cols, int N, int Cin, int H, int W, int k,
                                        int s, int pad_t, int pad_l, int WP, int Ho, int Wo, int Kp) {
    stem_im2col_body(x, cols, N, Cin, H, W, k, s, pad_t, pad_l, WP, Ho, Wo, Kp);
}
// 16-bit weight [O][taps] -> [O][Kp] (zero padded), and the inverse for the fp32 gradient (accumulating)
template <typename T>
__global__ void pad_weight_kernel(const T* __restrict__ src, T* __restrict__ dst, int O, int taps, int Kp) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= O * Kp) return;
    int o = i / Kp, t = i - o * Kp;
    dst[i] = t < taps ? src[(size_t)o * taps + t] : from_f<T>(0.f);
}
__global__ void unpad_grad_kernel(const float* __restrict__ gp, float* __restrict__ g, int O, int taps, int Kp) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= O * taps) return;
    int o = i / taps, t = i - o * taps;
    g[i] += gp[(size_t)o * Kp + t];
}

static int nblocks(long long total) {
    long long b = (total + 255) / 256;
    if (b > DFD_SMS * 32) b = DFD_SMS * 32;
    if (b < 1) b = 1;
    return (int)b;
}

}  // namespace

#define CD_T(dt, ...)                                                    \
    if ((dt) == DFD_DT_BF16) { typedef bf16 T; __VA_ARGS__; }            \
    else if ((dt) == DFD_DT_FP16) { typedef __half T; __VA_ARGS__; }     \
    else return dfd_set_error(DFD_ERR_ARG, "bad dtype");

extern "C" {

int dfd_im2col(const void* x, void* cols, int N, int H, int W, int C, int k, int stride, int pad, int dt, void* stream) {
    if (C % 8 || N <= 0) return dfd_set_error(DFD_ERR_ARG, "dfd_im2col: C%8");
    int Ho = (H + 2 * pad - k) / stride + 1, Wo = (W + 2 * pad - k) / stride + 1;
    long long total = (long long)N * Ho * Wo * k * k * (C / 8);
    CD_T(dt, (im2col_kernel<T><<<nblocks(total), 256, 0, (cudaStream_t)stream>>>((const T*)x, (T*)cols, N, H, W, C, k, stride, pad, Ho, Wo)));
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

int dfd_col2im(const void* dcols, const void* add, void* dx, int N, int H, int W, int C, int k, int stride, int pad, int dt,
               void* stream) {
    if (C % 8 || N <= 0) return dfd_set_error(DFD_ERR_ARG, "dfd_col2im: C%8");
    int Ho = (H + 2 * pad - k) / stride + 1, Wo = (W + 2 * pad - k) / stride + 1;
    long long total = (long long)N * H * W * (C / 8);
    CD_T(dt, (col2im_kernel<T><<<nblocks(total), 256, 0, (cudaStream_t)stream>>>((const T*)dcols, (const T*)add, (T*)dx, N, H, W, C, k, stride, pad, Ho, Wo)));
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

// table: device array of { const void* src; void* dst; void* dstT; void* dstD; int O, I, k; int pad_; }
int dfd_repack_weights(const void* table, int count, int dt, void* stream) {
    if (count <= 0) return DFD_OK;
    dim3 grid(DFD_SMS * 8, count);       // latency-bound gather: many short grid-stride loops
    CD_T(dt, (repack_weights_kernel<T><<<grid, 256, 0, (cudaStream_t)stream>>>((const RepackDesc*)table)));
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

int dfd_unpack_grad(const float* gperm, float* g_oihw, int O, int I, int k, void* stream) {
    long long total = (long long)O * I * k * k;
    unpack_grad_kernel<<<nblocks(total), 256, 0, (cudaStream_t)stream>>>(gperm, g_oihw, O, I, k);
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

int dfd_maxpool_fwd(const void* x, void* out, void* idx, int N, int H, int W, int C, int dt, void* stream) {
    if (C % 8 || N <= 0) return dfd_set_error(DFD_ERR_ARG, "dfd_maxpool_fwd: C%8");
    int Ho = (H + 2 - 3) / 2 + 1, Wo = (W + 2 - 3) / 2 + 1;
    long long total = (long long)N * Ho * Wo * (C / 8);
    CD_T(dt, (maxpool_fwd_kernel<T><<<nblocks(total), 256, 0, (cudaStream_t)stream>>>((const T*)x, (T*)out, (unsigned char*)idx, N, H, W, C, Ho, Wo)));
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

int dfd_maxpool_bwd(const void* gy, const void* idx, void* gx, int N, int H, int W, int C, int dt, void* stream) {
    if (C % 8 || N <= 0) return dfd_set_error(DFD_ERR_ARG, "dfd_maxpool_bwd: C%8");
    int Ho = (H + 2 - 3) / 2 + 1, Wo = (W + 2 - 3) / 2 + 1;
    long long total = (long long)N * H * W * (C / 8);
    CD_T(dt, (maxpool_bwd_kernel<T><<<nblocks(total), 256, 0, (cudaStream_t)stream>>>((const T*)gy, (const unsigned char*)idx, (T*)gx, N, H, W, C, Ho, Wo)));
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

// output extent of nn.MaxPool2d(3, 2, padding=0, ceil_mode=True) over an input extent h >= 3 (torch's pooling_output_shape:
// ceil((h - 3) / 2) + 1, less one when the last window would start outside the input)
static int ceil_pool_out(int h) {
    int o = (h - 3 + 1) / 2 + 1;
    if ((o - 1) * 2 >= h) o--;
    return o;
}

int dfd_maxpool_ceil_fwd(const void* x, void* out, void* idx, int N, int H, int W, int C, int dt, void* stream) {
    if (C % 8 || C <= 0 || N <= 0 || H < 3 || W < 3) return dfd_set_error(DFD_ERR_ARG, "dfd_maxpool_ceil_fwd: C%8, sizes");
    int Ho = ceil_pool_out(H), Wo = ceil_pool_out(W);
    long long total = (long long)N * Ho * Wo * (C / 8);
    CD_T(dt, (maxpool_ceil_fwd_kernel<T><<<nblocks(total), 256, 0, (cudaStream_t)stream>>>((const T*)x, (T*)out, (unsigned char*)idx, N, H, W, C, Ho, Wo)));
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

int dfd_maxpool_ceil_bwd(const void* gy, const void* idx, void* gx, int N, int H, int W, int C, int dt, void* stream) {
    if (C % 8 || C <= 0 || N <= 0 || H < 3 || W < 3) return dfd_set_error(DFD_ERR_ARG, "dfd_maxpool_ceil_bwd: C%8, sizes");
    int Ho = ceil_pool_out(H), Wo = ceil_pool_out(W);
    long long total = (long long)N * H * W * (C / 8);
    CD_T(dt, (maxpool_ceil_bwd_kernel<T><<<nblocks(total), 256, 0, (cudaStream_t)stream>>>((const T*)gy, (const unsigned char*)idx, (T*)gx, N, H, W, C, Ho, Wo)));
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

int dfd_relu_bwd(const void* g, const void* out, void* gm, long long numel, int dt, void* stream) {
    if (numel % 8) return dfd_set_error(DFD_ERR_ARG, "dfd_relu_bwd: numel%8");
    size_t nvec = (size_t)(numel / 8);
    CD_T(dt, (relu_bwd_kernel<T><<<nblocks((long long)nvec), 256, 0, (cudaStream_t)stream>>>((const T*)g, (const T*)out, (T*)gm, nvec)));
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

int dfd_pool_bwd(const float* dpooled, void* dout, int N, long long hw, int C, int dt, void* stream) {
    if (C % 8 || N <= 0) return dfd_set_error(DFD_ERR_ARG, "dfd_pool_bwd: C%8");
    long long total = (long long)N * hw * (C / 8);
    CD_T(dt, (pool_bwd_kernel<T><<<nblocks(total), 256, 0, (cudaStream_t)stream>>>(dpooled, (T*)dout, N, hw, C)));
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

int dfd_gpool_bwd(const float* dpooled, const int* argmax, void* dout, int N, long long hw, int C, int pool_type, int dt,
                  void* stream) {
    if (C % 8 || N <= 0 || hw <= 0) return dfd_set_error(DFD_ERR_ARG, "dfd_gpool_bwd: C%8, sizes");
    if (!dpooled || !argmax) return dfd_set_error(DFD_ERR_ARG, "dfd_gpool_bwd: operands");
    if (pool_type != DFD_POOL_MAX && pool_type != DFD_POOL_AVGMAX && pool_type != DFD_POOL_CATAVGMAX)
        return dfd_set_error(DFD_ERR_ARG, "dfd_gpool_bwd: pool_type (avg: dfd_pool_bwd)");
    long long total = (long long)N * hw * (C / 8);
    CD_T(dt, (gpool_bwd_kernel<T><<<nblocks(total), 256, 0, (cudaStream_t)stream>>>(dpooled, argmax, (T*)dout, N, hw, C, pool_type)));
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

static int stem_im2col(const void* x_nchw, void* cols, int N, int Cin, int H, int W, int k, int stride, int pad_t, int pad_l,
                       int Ho, int Wo, int WP, int Kp, int dt, void* stream) {
    if (Kp % 8 || Kp < Cin * k * k) return dfd_set_error(DFD_ERR_ARG, "dfd_stem_im2col: Kp");
    size_t smem = (((size_t)Cin * k * WP * 2 + 15) & ~(size_t)15) + (size_t)Kp * sizeof(int);
    if (smem > 48 * 1024) return dfd_set_error(DFD_ERR_UNSUPPORTED, "dfd_stem_im2col: input rows exceed shared memory");
    // symmetric pads (every ResNet / EfficientNet stem, and a TF "SAME" stem over odd extents) run the symmetric kernel
    if (pad_t == pad_l && WP == W + 2 * pad_t && Ho == (H + 2 * pad_t - k) / stride + 1 && Wo == (W + 2 * pad_t - k) / stride + 1) {
        CD_T(dt, (stem_im2col_kernel<T><<<N * Ho, 256, smem, (cudaStream_t)stream>>>((const T*)x_nchw, (T*)cols, N, Cin, H, W, k, stride, pad_t, Ho, Wo, Kp)));
    } else {
        CD_T(dt, (stem_im2col_same_kernel<T><<<N * Ho, 256, smem, (cudaStream_t)stream>>>((const T*)x_nchw, (T*)cols, N, Cin, H, W, k, stride, pad_t, pad_l, WP, Ho, Wo, Kp)));
    }
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

int dfd_stem_im2col(const void* x_nchw, void* cols, int N, int Cin, int H, int W, int k, int stride, int pad, int Kp, int dt,
                    void* stream) {
    int Ho = (H + 2 * pad - k) / stride + 1, Wo = (W + 2 * pad - k) / stride + 1;
    return stem_im2col(x_nchw, cols, N, Cin, H, W, k, stride, pad, pad, Ho, Wo, W + 2 * pad, Kp, dt, stream);
}

// TF "SAME" padding: Ho = ceil(H / stride), Wo = ceil(W / stride), pad_t rows above and pad_l columns left of the image,
// the rest of each total pad max((ceil(i/s) - 1) * s + k - i, 0) below / right (layers/padding.py `pad_same`)
int dfd_stem_im2col_pad(const void* x_nchw, void* cols, int N, int Cin, int H, int W, int k, int stride, int pad_t, int pad_l,
                        int Kp, int dt, void* stream) {
    if (stride <= 0 || N <= 0 || H <= 0 || W <= 0) return dfd_set_error(DFD_ERR_ARG, "dfd_stem_im2col_pad: sizes");
    const int Ho = (H + stride - 1) / stride, Wo = (W + stride - 1) / stride;
    const int tot_h = (Ho - 1) * stride + k - H, tot_w = (Wo - 1) * stride + k - W;
    if (pad_t != (tot_h > 0 ? tot_h / 2 : 0) || pad_l != (tot_w > 0 ? tot_w / 2 : 0))
        return dfd_set_error(DFD_ERR_ARG, "dfd_stem_im2col_pad: pads are the begin sides of TF SAME padding");
    return stem_im2col(x_nchw, cols, N, Cin, H, W, k, stride, pad_t, pad_l, Ho, Wo, (Wo - 1) * stride + k, Kp, dt, stream);
}

int dfd_pad_weight(const void* src, void* dst, int O, int taps, int Kp, int dt, void* stream) {
    CD_T(dt, (pad_weight_kernel<T><<<cdiv((long long)O * Kp, 256), 256, 0, (cudaStream_t)stream>>>((const T*)src, (T*)dst, O, taps, Kp)));
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

int dfd_unpad_grad(const float* gp, float* g, int O, int taps, int Kp, void* stream) {
    unpad_grad_kernel<<<cdiv((long long)O * taps, 256), 256, 0, (cudaStream_t)stream>>>(gp, g, O, taps, Kp);
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

}  // extern "C"
