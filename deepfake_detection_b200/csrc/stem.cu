// Stem convolution: dense k x k, stride 2, tiny Cin (3 RGB / 12 = 4 frames), NCHW 16-bit image in,
// NHWC 16-bit feature map out, plus its weight gradient (the image needs no gradient).
//   EfficientNet conv_stem 3x3 s2 p1 : dfd/timm/models/efficientnet.py:275,321
//   ResNet conv1 7x7 s2 p3           : dfd/timm/models/resnet.py:379,451
// K = Cin*k*k is 27..147: far too skinny for a tensor-core tile and <1% of the step's FLOPs, so this is a
// direct CUDA-core convolution: weights in shared memory as [tap][cout] fp32, one thread = one output pixel x
// 8 output channels (16-byte NHWC store), image reads served from L1 (the NCHW->NHWC layout change is free).
#include "common.cuh"

namespace {

template <typename T, int K>
__global__ void __launch_bounds__(256)
stem_fwd_kernel(const T* __restrict__ x, const float* __restrict__ w, T* __restrict__ out, int N, int Cin, int H,
                int W, int Cout, int Ho, int Wo, int stride, int pad, double* __restrict__ dsum,
                double* __restrict__ dsq) {
    extern __shared__ float sw[];            // [Cin*K*K][Cout]
    const int taps = Cin * K * K;
    for (int i = threadIdx.x; i < taps * Cout; i += blockDim.x) {
        int t = i / Cout, co = i - t * Cout;           // w is OIHW: [co][ci][kh][kw] -> tap t = (ci*K + kh)*K + kw
        sw[i] = w[(size_t)co * taps + t];
    }
    __syncthreads();
    const int G = Cout / 8;
    const int g = threadIdx.x % G;
    const int pix_per_block = blockDim.x / G;
    const long long total = (long long)N * Ho * Wo;
    long long pix = (long long)blockIdx.x * pix_per_block + threadIdx.x / G;
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; i++) acc[i] = 0.f;
    float s[8], q[8];
#pragma unroll
    for (int i = 0; i < 8; i++) { s[i] = 0.f; q[i] = 0.f; }
    const bool active = (threadIdx.x / G) < pix_per_block && pix < total;
    if (active) {
        int ox = (int)(pix % Wo);
        long long t2 = pix / Wo;
        int oy = (int)(t2 % Ho);
        int n = (int)(t2 / Ho);
        const T* img = x + (size_t)n * Cin * H * W;
        for (int ci = 0; ci < Cin; ci++) {
#pragma unroll
            for (int kh = 0; kh < K; kh++) {
                int iy = oy * stride - pad + kh;
                if (iy < 0 || iy >= H) continue;
#pragma unroll
                for (int kw = 0; kw < K; kw++) {
                    int ix = ox * stride - pad + kw;
                    if (ix < 0 || ix >= W) continue;
                    float xv = to_f<T>(img[((size_t)ci * H + iy) * W + ix]);
                    const float4* wp = reinterpret_cast<const float4*>(sw + (size_t)((ci * K + kh) * K + kw) * Cout + g * 8);
                    float4 w0 = wp[0], w1 = wp[1];
                    acc[0] = fmaf(xv, w0.x, acc[0]); acc[1] = fmaf(xv, w0.y, acc[1]);
                    acc[2] = fmaf(xv, w0.z, acc[2]); acc[3] = fmaf(xv, w0.w, acc[3]);
                    acc[4] = fmaf(xv, w1.x, acc[4]); acc[5] = fmaf(xv, w1.y, acc[5]);
                    acc[6] = fmaf(xv, w1.z, acc[6]); acc[7] = fmaf(xv, w1.w, acc[7]);
                }
            }
        }
        uint4 pk = pack8<T>(acc);
        stg16(out + (size_t)pix * Cout + g * 8, pk);
        float r[8];
        unpack8<T>(pk, r);
#pragma unroll
        for (int i = 0; i < 8; i++) { s[i] = r[i]; q[i] = r[i] * r[i]; }
    }
    if (dsum) {
        // block reduce over the pixels that share a channel group, then one fp64 atomic per channel per CTA
        __syncthreads();
        __shared__ float red2[256 * 8];
        double* ps = stat_slot(dsum, Cout);
        double* pq = stat_slot(dsq, Cout);
#pragma unroll
        for (int i = 0; i < 8; i++) red2[threadIdx.x * 8 + i] = s[i];
        __syncthreads();
        if (threadIdx.x < Cout) {
            int gg = threadIdx.x / 8, i = threadIdx.x % 8;
            float t = 0.f;
            for (int p = 0; p < pix_per_block; p++) t += red2[(p * G + gg) * 8 + i];
            atomicAdd(ps + threadIdx.x, (double)t);
        }
        __syncthreads();
#pragma unroll
        for (int i = 0; i < 8; i++) red2[threadIdx.x * 8 + i] = q[i];
        __syncthreads();
        if (threadIdx.x < Cout) {
            int gg = threadIdx.x / 8, i = threadIdx.x % 8;
            float t = 0.f;
            for (int p = 0; p < pix_per_block; p++) t += red2[(p * G + gg) * 8 + i];
            atomicAdd(pq + threadIdx.x, (double)t);
        }
    }
}

// dW[co][ci][kh][kw] += sum_pix dy[pix][co] * x[n][ci][oy*s-p+kh][ox*s-p+kw],  dy = cA*g + cB*y + cC.
// A CTA stages dy for PIX consecutive output pixels in smem (fp32), then every thread owns IPT (tap, 8-cout
// group) items and walks the pixels; partial sums leave through fp32 atomics (taps*Cout per CTA).
template <typename T, int K, int IPT>
__global__ void __launch_bounds__(256)
stem_wgrad_kernel(const T* __restrict__ x, const T* __restrict__ g, const T* __restrict__ y,
                  const float* __restrict__ cA, const float* __restrict__ cB, const float* __restrict__ cC,
                  float* __restrict__ dW, int N, int Cin, int H, int W, int Cout, int Ho, int Wo, int stride, int pad,
                  int pix_per_block) {
    extern __shared__ float sdy[];           // [PIX][Cout] dy, then int2[PIX] pixel coordinates
    constexpr int PIX = 64;
    int2* spix = reinterpret_cast<int2*>(sdy + (size_t)PIX * Cout);    // {image base offset, (iy0 << 16) | (ix0 & 0xffff)}
    const int taps = Cin * K * K;
    const int G = Cout / 8;
    const int items = taps * G;
    // when items < blockDim, several thread groups share the item set and split the pixels between them
    const int groups = IPT == 1 ? max(1, (int)blockDim.x / items) : 1;
    const int grp = IPT == 1 ? threadIdx.x / items : 0;
    const long long total = (long long)N * Ho * Wo;
    const long long p_begin = (long long)blockIdx.x * pix_per_block;
    long long p_end = p_begin + pix_per_block;
    if (p_end > total) p_end = total;
    float acc[IPT][8];
    int it_ci_off[IPT], it_kh[IPT], it_kw[IPT], it_g[IPT];
#pragma unroll
    for (int a = 0; a < IPT; a++) {
#pragma unroll
        for (int i = 0; i < 8; i++) acc[a][i] = 0.f;
        int item = (IPT == 1 ? threadIdx.x % items : threadIdx.x) + a * blockDim.x;
        bool valid = item < items && grp < groups;
        int t = valid ? item / G : 0;
        it_g[a] = valid ? item - t * G : -1;
        int ci = t / (K * K), r = t - ci * K * K;
        it_kh[a] = r / K;
        it_kw[a] = r - it_kh[a] * K;
        it_ci_off[a] = ci * H * W;
    }

    for (long long p0 = p_begin; p0 < p_end; p0 += PIX) {
        int np = (int)((p_end - p0 < PIX) ? (p_end - p0) : PIX);
        __syncthreads();
        if (threadIdx.x < np) {
            long long pix = p0 + threadIdx.x;
            int ox = (int)(pix % Wo);
            long long t2 = pix / Wo;
            int oy = (int)(t2 % Ho);
            int n = (int)(t2 / Ho);
            int iy0 = oy * stride - pad, ix0 = ox * stride - pad;
            spix[threadIdx.x] = make_int2(n * Cin * H * W, (iy0 << 16) | (ix0 & 0xffff));
        }
        for (int i = threadIdx.x; i < np * G; i += blockDim.x) {
            int pp = i / G, gg = i - pp * G;
            size_t off = (size_t)(p0 + pp) * Cout + gg * 8;
            float gv[8], yv[8];
            unpack8<T>(ldg16(g + off), gv);
            unpack8<T>(ldg16(y + off), yv);
#pragma unroll
            for (int k = 0; k < 8; k++) {
                int c = gg * 8 + k;
                sdy[(size_t)pp * Cout + c] = fmaf(cA[c], gv[k], fmaf(cB[c], yv[k], cC[c]));
            }
        }
        __syncthreads();
#pragma unroll
        for (int a = 0; a < IPT; a++) {
            if (it_g[a] < 0) continue;
            const int kh = it_kh[a], kw = it_kw[a], cio = it_ci_off[a], gg = it_g[a];
#pragma unroll 4
            for (int pp = grp; pp < np; pp += groups) {
                int2 pc = spix[pp];
                int iy = (pc.y >> 16) + kh, ix = (int)(short)(pc.y & 0xffff) + kw;
                if (iy < 0 || iy >= H || ix < 0 || ix >= W) continue;
                float xv = to_f<T>(x[(size_t)pc.x + cio + iy * W + ix]);
                const float4* dp = reinterpret_cast<const float4*>(sdy + (size_t)pp * Cout + gg * 8);
                float4 d0 = dp[0], d1 = dp[1];
                acc[a][0] = fmaf(xv, d0.x, acc[a][0]); acc[a][1] = fmaf(xv, d0.y, acc[a][1]);
                acc[a][2] = fmaf(xv, d0.z, acc[a][2]); acc[a][3] = fmaf(xv, d0.w, acc[a][3]);
                acc[a][4] = fmaf(xv, d1.x, acc[a][4]); acc[a][5] = fmaf(xv, d1.y, acc[a][5]);
                acc[a][6] = fmaf(xv, d1.z, acc[a][6]); acc[a][7] = fmaf(xv, d1.w, acc[a][7]);
            }
        }
    }
#pragma unroll
    for (int a = 0; a < IPT; a++) {
        if (it_g[a] < 0) continue;
        int item = (IPT == 1 ? threadIdx.x % items : threadIdx.x) + a * blockDim.x;
        int t = item / G;
#pragma unroll
        for (int i = 0; i < 8; i++) atomicAdd(dW + (size_t)(it_g[a] * 8 + i) * taps + t, acc[a][i]);
    }
}

}  // namespace

#define STEM_T(dt, ...)                                                  \
    if ((dt) == DFD_DT_BF16) { typedef bf16 T; __VA_ARGS__; }            \
    else if ((dt) == DFD_DT_FP16) { typedef __half T; __VA_ARGS__; }     \
    else return dfd_set_error(DFD_ERR_ARG, "bad dtype");

extern "C" {

// x: [N,Cin,H,W] (NCHW, 16-bit) ; w: [Cout,Cin,k,k] fp32 ; out: [N,Ho,Wo,Cout] (NHWC, 16-bit)
int dfd_stem_fwd(const void* x, const float* w, void* out, int N, int Cin, int H, int W, int Cout, int k, int stride,
                 int pad, int dt, double* dsum, double* dsq, void* stream) {
    if (Cout % 8 || Cout > 256 || (k != 3 && k != 7))
        return dfd_set_error(DFD_ERR_UNSUPPORTED, "dfd_stem_fwd: Cout % 8 == 0, Cout <= 256, k in {3,7}");
    int Ho = (H + 2 * pad - k) / stride + 1, Wo = (W + 2 * pad - k) / stride + 1;
    int G = Cout / 8, ppb = 256 / G;
    const int nthreads = G * ppb;            // whole pixels only (e.g. Cout = 48: 6 groups x 42 pixels = 252 threads)
    long long total = (long long)N * Ho * Wo;
    int blocks = cdiv(total, ppb);
    size_t smem = (size_t)Cin * k * k * Cout * sizeof(float);
    cudaStream_t st = (cudaStream_t)stream;
    STEM_T(dt, {
        if (k == 3) {
            auto kf = stem_fwd_kernel<T, 3>;
            if (smem > 48 * 1024) cudaFuncSetAttribute(kf, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            kf<<<blocks, nthreads, smem, st>>>((const T*)x, w, (T*)out, N, Cin, H, W, Cout, Ho, Wo, stride, pad, dsum, dsq);
        } else {
            auto kf = stem_fwd_kernel<T, 7>;
            if (smem > 48 * 1024) cudaFuncSetAttribute(kf, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            kf<<<blocks, nthreads, smem, st>>>((const T*)x, w, (T*)out, N, Cin, H, W, Cout, Ho, Wo, stride, pad, dsum, dsq);
        }
    });
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

// dW [Cout,Cin,k,k] fp32 += ; g, y: [N,Ho,Wo,Cout] ; dy = cA*g + cB*y + cC (BN backward folded in)
int dfd_stem_wgrad(const void* x, const void* g, const void* y, const float* cA, const float* cB, const float* cC,
                   float* dW, int N, int Cin, int H, int W, int Cout, int k, int stride, int pad, int dt,
                   void* stream) {
    if (Cout % 8 || (k != 3 && k != 7)) return dfd_set_error(DFD_ERR_UNSUPPORTED, "dfd_stem_wgrad: Cout%8, k in {3,7}");
    int Ho = (H + 2 * pad - k) / stride + 1, Wo = (W + 2 * pad - k) / stride + 1;
    long long total = (long long)N * Ho * Wo;
    int items = Cin * k * k * (Cout / 8);
    int ipt = (items + 255) / 256;
    int blocks = DFD_SMS * 4;
    long long ppb = (total + blocks - 1) / blocks;
    ppb = ((ppb + 63) / 64) * 64;
    blocks = cdiv(total, ppb);
    size_t smem = (size_t)64 * Cout * sizeof(float) + 64 * sizeof(int2);
    if ((long long)N * Cin * H * W >= (1ll << 31)) return dfd_set_error(DFD_ERR_UNSUPPORTED, "dfd_stem_wgrad: image tensor >= 2^31 elements");
    cudaStream_t st = (cudaStream_t)stream;
#define WG(KK, IPT)                                                                                               \
    do {                                                                                                          \
        auto kf = stem_wgrad_kernel<T, KK, IPT>;                                                                  \
        if (smem > 48 * 1024) cudaFuncSetAttribute(kf, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);   \
        kf<<<blocks, 256, smem, st>>>((const T*)x, (const T*)g, (const T*)y, cA, cB, cC, dW, N, Cin, H, W, Cout, Ho, \
                                      Wo, stride, pad, (int)ppb);                                                 \
    } while (0)
    STEM_T(dt, {
        if (k == 3) {
            if (ipt <= 1) WG(3, 1); else if (ipt <= 2) WG(3, 2); else if (ipt <= 4) WG(3, 4);
            else if (ipt <= 14) WG(3, 14); else return dfd_set_error(DFD_ERR_UNSUPPORTED, "dfd_stem_wgrad: too many taps*Cout");
        } else {
            if (ipt <= 5) WG(7, 5); else if (ipt <= 10) WG(7, 10);
            else return dfd_set_error(DFD_ERR_UNSUPPORTED, "dfd_stem_wgrad: too many taps*Cout");
        }
    });
#undef WG
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

}  // extern "C"
