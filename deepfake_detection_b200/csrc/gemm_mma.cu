// Pointwise (1x1) convolution GEMMs on the legacy warp-level tensor-core path (mma.sync m16n8k16).
//
//   gemm_tn   : C[M,N] = A[M,K] * B[N,K]^T   (both operands K-contiguous)  -> forward (A = activations NHWC,
//               B = conv weight [Cout,Cin]) and input gradient (A = dY, B = W^T stored [Cin,Cout])
//   gemm_wgrad: dW[Nw,Kw] += G[M,Nw]^T * X[M,Kw]   (contraction over the M = N*H*W rows; split over M)
//
// This file is the bring-up / cross-check implementation and the weight-gradient path of round 1; the
// forward/dgrad product path is the wgmma + TMA kernel in gemm_tc.cu.
// Reference ops replaced: nn.Conv2d 1x1 at dfd/timm/models/efficientnet_blocks.py:165,277,299 and
// efficientnet.py:292, ResNet 1x1 at resnet.py:192,199, and their autograd backward (train.py:634-636).
#include "common.cuh"

namespace {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, bool valid) {
    int sz = valid ? 16 : 0;   // src-size 0 => zero fill
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(smem_u32(smem)), "l"(gmem), "r"(sz));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], const void* p) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_u32(p)));
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t (&r)[4], const void* p) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];\n"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_u32(p)));
}
template <typename T> __device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1);
template <> __device__ __forceinline__ void mma16816<bf16>(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
template <> __device__ __forceinline__ void mma16816<__half>(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// =============================================================================================
// gemm_tn: CTA tile 128 x 64 x 32, 8 warps (4 along M x 2 along N), warp tile 32 x 32, 3-stage cp.async.
// smem rows are 64 bytes (32 elements); 16-byte chunks are XOR-swizzled with (row>>1)&3 -> conflict-free ldmatrix.
// =============================================================================================
constexpr int TN_BM = 128, TN_BN = 64, TN_BK = 32, TN_STAGES = 3;
constexpr int TN_CPAD = 8;   // epilogue staging row pitch = 64 + 8 elements

template <typename T>
__global__ void __launch_bounds__(256)
gemm_tn_kernel(const T* __restrict__ A, const T* __restrict__ B, T* __restrict__ C, const T* __restrict__ add,
               int M, int N, int K, double* __restrict__ dsum, double* __restrict__ dsq) {
    __shared__ __align__(128) unsigned char smem_raw[TN_STAGES * (TN_BM + TN_BN) * TN_BK * 2];
    T* sA = reinterpret_cast<T*>(smem_raw);
    T* sB = sA + TN_STAGES * TN_BM * TN_BK;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int wm = warp & 3, wn = warp >> 2;
    const long long m0 = (long long)blockIdx.x * TN_BM;
    const int n0 = blockIdx.y * TN_BN;
    const int ktiles = (K + TN_BK - 1) / TN_BK;

    auto load_stage = [&](int stage, int kt) {
        const int k0 = kt * TN_BK;
        T* a = sA + stage * TN_BM * TN_BK;
        T* b = sB + stage * TN_BN * TN_BK;
#pragma unroll
        for (int i = 0; i < 2; i++) {
            int idx = tid + i * 256;            // 512 chunks of A
            int r = idx >> 2, ch = idx & 3;
            long long gm = m0 + r;
            int gk = k0 + ch * 8;
            bool v = gm < M && gk < K;
            const T* src = v ? A + (size_t)gm * K + gk : A;
            cp_async16(a + r * TN_BK + ((ch ^ ((r >> 1) & 3)) * 8), src, v);
        }
        {
            int r = tid >> 2, ch = tid & 3;     // 256 chunks of B
            int gn = n0 + r, gk = k0 + ch * 8;
            bool v = gn < N && gk < K;
            const T* src = v ? B + (size_t)gn * K + gk : B;
            cp_async16(b + r * TN_BK + ((ch ^ ((r >> 1) & 3)) * 8), src, v);
        }
    };

    float acc[2][4][4];
#pragma unroll
    for (int i = 0; i < 2; i++)
#pragma unroll
        for (int j = 0; j < 4; j++)
#pragma unroll
            for (int k = 0; k < 4; k++) acc[i][j][k] = 0.f;

#pragma unroll
    for (int s = 0; s < TN_STAGES - 1; s++) {
        if (s < ktiles) load_stage(s, s);
        cp_async_commit();
    }
    for (int kt = 0; kt < ktiles; kt++) {
        cp_async_wait<TN_STAGES - 2>();
        __syncthreads();
        {
            int nk = kt + TN_STAGES - 1;
            if (nk < ktiles) load_stage(nk % TN_STAGES, nk);
            cp_async_commit();
        }
        const T* a = sA + (kt % TN_STAGES) * TN_BM * TN_BK;
        const T* b = sB + (kt % TN_STAGES) * TN_BN * TN_BK;
#pragma unroll
        for (int ks = 0; ks < TN_BK / 16; ks++) {
            uint32_t af[2][4], bfr[2][4];
#pragma unroll
            for (int mi = 0; mi < 2; mi++) {
                int r = wm * 32 + mi * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
                int ch = ks * 2 + (lane >> 4);
                ldmatrix_x4(af[mi], a + r * TN_BK + ((ch ^ ((r >> 1) & 3)) * 8));
            }
#pragma unroll
            for (int nj = 0; nj < 2; nj++) {
                int r = wn * 32 + nj * 16 + (lane & 7) + (lane >> 4) * 8;
                int ch = ks * 2 + ((lane >> 3) & 1);
                ldmatrix_x4(bfr[nj], b + r * TN_BK + ((ch ^ ((r >> 1) & 3)) * 8));
            }
#pragma unroll
            for (int mi = 0; mi < 2; mi++)
#pragma unroll
                for (int nj = 0; nj < 2; nj++) {
                    mma16816<T>(acc[mi][nj * 2], af[mi], bfr[nj][0], bfr[nj][1]);
                    mma16816<T>(acc[mi][nj * 2 + 1], af[mi], bfr[nj][2], bfr[nj][3]);
                }
        }
    }
    cp_async_wait<0>();
    __syncthreads();

    // epilogue: accumulators -> smem (rounded to T, padded pitch) -> coalesced 16-byte stores (+add) + column stats
    T* sC = reinterpret_cast<T*>(smem_raw);
    constexpr int PITCH = TN_BN + TN_CPAD;
#pragma unroll
    for (int mi = 0; mi < 2; mi++)
#pragma unroll
        for (int nb = 0; nb < 4; nb++) {
            int r = wm * 32 + mi * 16 + (lane >> 2);
            int c = wn * 32 + nb * 8 + (lane & 3) * 2;
            *reinterpret_cast<uint32_t*>(sC + r * PITCH + c) = pack2<T>(acc[mi][nb][0], acc[mi][nb][1]);
            *reinterpret_cast<uint32_t*>(sC + (r + 8) * PITCH + c) = pack2<T>(acc[mi][nb][2], acc[mi][nb][3]);
        }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 4; i++) {
        int idx = tid + i * 256;       // 1024 chunks: 128 rows x 8
        int r = idx >> 3, ch = idx & 7;
        long long gm = m0 + r;
        int gn = n0 + ch * 8;
        if (gm < M && gn < N) {
            uint4 v = *reinterpret_cast<const uint4*>(sC + r * PITCH + ch * 8);
            if (add) {
                float x[8], z[8];
                unpack8<T>(v, x);
                unpack8<T>(ldg16(add + (size_t)gm * N + gn), z);
#pragma unroll
                for (int k = 0; k < 8; k++) x[k] += z[k];
                v = pack8<T>(x);
                *reinterpret_cast<uint4*>(sC + r * PITCH + ch * 8) = v;   // stats see the stored value
            }
            stg16(C + (size_t)gm * N + gn, v);
        }
    }
    if (dsum) {
        __syncthreads();
        // 256 threads = 64 columns x 4 row quarters
        int c = tid & 63, qd = tid >> 6;
        float s = 0.f, q = 0.f;
        int rmax = (int)((M - m0 < TN_BM) ? (M - m0) : TN_BM);
        for (int r = qd * 32; r < qd * 32 + 32 && r < rmax; r++) {
            float v = to_f<T>(sC[r * PITCH + c]);
            s += v;
            q = fmaf(v, v, q);
        }
        __shared__ float red[2][4][64];
        red[0][qd][c] = s;
        red[1][qd][c] = q;
        __syncthreads();
        if (tid < 64 && n0 + tid < N) {
            float ts = red[0][0][tid] + red[0][1][tid] + red[0][2][tid] + red[0][3][tid];
            float tq = red[1][0][tid] + red[1][1][tid] + red[1][2][tid] + red[1][3][tid];
            atomicAdd(stat_slot(dsum, N) + n0 + tid, (double)ts);
            atomicAdd(stat_slot(dsq, N) + n0 + tid, (double)tq);
        }
    }
}

// =============================================================================================
// gemm_wgrad: dW[Nw,Kw] += sum_m G[m,Nw] * X[m,Kw].  CTA tile 64 (Nw) x 64 (Kw), contraction chunks of 32 rows,
// both operands are "MN-major" w.r.t. the contraction so fragments come from ldmatrix.trans.
// smem rows are 128 bytes (64 elements); chunks XOR-swizzled with row&7.
// grid = (Nw tiles, Kw tiles, M splits); partial tiles are added with fp32 atomics.
// =============================================================================================
constexpr int WG_BN = 64, WG_BK = 64, WG_BM = 32, WG_STAGES = 3;

template <typename T>
__global__ void __launch_bounds__(256)
gemm_wgrad_kernel(const T* __restrict__ G, const T* __restrict__ X, float* __restrict__ dW, long long M, int Nw,
                  int Kw, long long rows_per_split) {
    __shared__ __align__(128) unsigned char smem_raw[WG_STAGES * WG_BM * (WG_BN + WG_BK) * 2];
    T* sG = reinterpret_cast<T*>(smem_raw);
    T* sX = sG + WG_STAGES * WG_BM * WG_BN;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int wi = warp & 3, wj = warp >> 2;        // warp tile: 16 (Nw) x 32 (Kw)
    const int n0 = blockIdx.x * WG_BN, k0 = blockIdx.y * WG_BK;
    const long long mbeg = (long long)blockIdx.z * rows_per_split;
    long long mend = mbeg + rows_per_split;
    if (mend > M) mend = M;
    const int iters = (int)((mend - mbeg + WG_BM - 1) / WG_BM);

    auto load_stage = [&](int stage, int it) {
        const long long mr = mbeg + (long long)it * WG_BM;
        int r = tid >> 3, ch = tid & 7;              // 32 rows x 8 chunks per operand
        long long gm = mr + r;
        bool vr = gm < mend;
        {
            int gc = n0 + ch * 8;
            bool v = vr && gc < Nw;
            const T* src = v ? G + (size_t)gm * Nw + gc : G;
            cp_async16(sG + (stage * WG_BM + r) * WG_BN + ((ch ^ (r & 7)) * 8), src, v);
        }
        {
            int gc = k0 + ch * 8;
            bool v = vr && gc < Kw;
            const T* src = v ? X + (size_t)gm * Kw + gc : X;
            cp_async16(sX + (stage * WG_BM + r) * WG_BK + ((ch ^ (r & 7)) * 8), src, v);
        }
    };

    float acc[4][4];
#pragma unroll
    for (int j = 0; j < 4; j++)
#pragma unroll
        for (int k = 0; k < 4; k++) acc[j][k] = 0.f;

#pragma unroll
    for (int s = 0; s < WG_STAGES - 1; s++) {
        if (s < iters) load_stage(s, s);
        cp_async_commit();
    }
    for (int it = 0; it < iters; it++) {
        cp_async_wait<WG_STAGES - 2>();
        __syncthreads();
        {
            int ni = it + WG_STAGES - 1;
            if (ni < iters) load_stage(ni % WG_STAGES, ni);
            cp_async_commit();
        }
        const T* g = sG + (it % WG_STAGES) * WG_BM * WG_BN;
        const T* x = sX + (it % WG_STAGES) * WG_BM * WG_BK;
#pragma unroll
        for (int ks = 0; ks < WG_BM / 16; ks++) {
            uint32_t af[4], b0[4], b1[4];
            {   // A = G^T fragment: matrices (kk 0-7, i 0-7), (kk 0-7, i 8-15), (kk 8-15, i 0-7), (kk 8-15, i 8-15)
                int kk = ks * 16 + (lane & 7) + (lane >> 4) * 8;
                int ch = wi * 2 + ((lane >> 3) & 1);
                ldmatrix_x4_trans(af, g + kk * WG_BN + ((ch ^ (kk & 7)) * 8));
            }
            {   // B = X fragment: matrices (kk 0-7, j 0-7), (kk 8-15, j 0-7), (kk 0-7, j 8-15), (kk 8-15, j 8-15)
                int kk = ks * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
                int ch = wj * 4 + (lane >> 4);
                ldmatrix_x4_trans(b0, x + kk * WG_BK + ((ch ^ (kk & 7)) * 8));
                ldmatrix_x4_trans(b1, x + kk * WG_BK + (((ch + 2) ^ (kk & 7)) * 8));
            }
            mma16816<T>(acc[0], af, b0[0], b0[1]);
            mma16816<T>(acc[1], af, b0[2], b0[3]);
            mma16816<T>(acc[2], af, b1[0], b1[1]);
            mma16816<T>(acc[3], af, b1[2], b1[3]);
        }
    }
    cp_async_wait<0>();
    // epilogue: fp32 atomics (splits) into dW[Nw][Kw]
#pragma unroll
    for (int nb = 0; nb < 4; nb++) {
        int i = n0 + wi * 16 + (lane >> 2);
        int j = k0 + wj * 32 + nb * 8 + (lane & 3) * 2;
        if (j < Kw) {
            if (i < Nw) {
                atomicAdd(dW + (size_t)i * Kw + j, acc[nb][0]);
                atomicAdd(dW + (size_t)i * Kw + j + 1, acc[nb][1]);
            }
            if (i + 8 < Nw) {
                atomicAdd(dW + (size_t)(i + 8) * Kw + j, acc[nb][2]);
                atomicAdd(dW + (size_t)(i + 8) * Kw + j + 1, acc[nb][3]);
            }
        }
    }
}

}  // namespace

#define GEMM_T(dt, ...)                                                  \
    if ((dt) == DFD_DT_BF16) { typedef bf16 T; __VA_ARGS__; }            \
    else if ((dt) == DFD_DT_FP16) { typedef __half T; __VA_ARGS__; }     \
    else return dfd_set_error(DFD_ERR_ARG, "bad dtype");

extern "C" {

// C[M,N] = A[M,K] * B[N,K]^T (+ add[M,N]); optional per-column statistics of the stored C (fp64 slots [8][N]).
int dfd_gemm_tn_mma(const void* A, const void* B, void* C, const void* add, long long M, int N, int K, int dt,
                    double* dsum, double* dsq, void* stream) {
    if (M <= 0 || N <= 0 || K <= 0 || (N % 8) || (K % 8)) return dfd_set_error(DFD_ERR_ARG, "dfd_gemm_tn_mma: N%8, K%8");
    dim3 grid(cdiv(M, TN_BM), cdiv(N, TN_BN), 1);
    GEMM_T(dt, (gemm_tn_kernel<T><<<grid, 256, 0, (cudaStream_t)stream>>>((const T*)A, (const T*)B, (T*)C, (const T*)add, (int)M, N, K, dsum, dsq)));
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

// dW[Nw,Kw] (fp32) += G[M,Nw]^T * X[M,Kw]
int dfd_gemm_wgrad_mma(const void* G, const void* X, float* dW, long long M, int Nw, int Kw, int dt, void* stream) {
    if (M <= 0 || Nw <= 0 || Kw <= 0 || (Nw % 8) || (Kw % 8)) return dfd_set_error(DFD_ERR_ARG, "dfd_gemm_wgrad_mma: Nw%8, Kw%8");
    int tn = cdiv(Nw, WG_BN), tk = cdiv(Kw, WG_BK);
    long long max_splits = (M + WG_BM * 4 - 1) / (WG_BM * 4);
    long long splits = (DFD_SMS * 4 + tn * tk - 1) / (tn * tk);
    if (splits > max_splits) splits = max_splits;
    if (splits < 1) splits = 1;
    if (splits > 65535) splits = 65535;
    long long rps = (M + splits - 1) / splits;
    rps = ((rps + WG_BM - 1) / WG_BM) * WG_BM;
    splits = (M + rps - 1) / rps;
    dim3 grid(tn, tk, (unsigned)splits);
    GEMM_T(dt, (gemm_wgrad_kernel<T><<<grid, 256, 0, (cudaStream_t)stream>>>((const T*)G, (const T*)X, dW, M, Nw, Kw, rps)));
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

}  // extern "C"
