// Channel-wise streaming kernels: BN statistics / finalise / apply, activation, SE gating, residual,
// global pooling, and their backward passes.  All are HBM-bound single passes over NHWC tensors.
//
// Thread geometry ("row geometry"): blockDim = (V, RY) with V = C/8 channel vectors; a thread owns ONE
// 8-channel vector (its per-channel parameters live in registers) and walks rows r = ty, ty+RY, ...
// Consecutive threads therefore touch consecutive 16-byte chunks (a warp covers >=512 contiguous bytes,
// spanning rows when V < 32 because the row pitch is exactly V*16 bytes).
// grid = (row chunks, images): per-image parameters (SE gate, pooled gradients) index blockIdx.y.
//
// Reference semantics restated here:
//   BN train/eval        torch.nn.BatchNorm2d as constructed at dfd/timm/models/efficientnet_blocks.py:154,166,280,287,300
//   Swish fwd/bwd        dfd/timm/models/layers/activations.py:19-33
//   SE gate, residual    dfd/timm/models/efficientnet_blocks.py:104-110, 343-346
//   global average pool  dfd/timm/models/efficientnet.py:340-343
//   max / avgmax / catavgmax global pool and argmax   dfd/timm/models/layers/adaptive_avgmax_pool.py:24-48
#include <climits>
#include <cmath>

#include "common.cuh"
#include "se_chain.cuh"
#include "bn_finalize.cuh"

namespace {

// scratch of the chunked per-image reductions (library-owned, zero at load; tickets self-reset): when an image is reduced
// by several CTAs their partial sums go to fixed slots [chunk][image][C] and the last CTA of the image to arrive (ticket)
// adds them in chunk order - and then carries on with whatever depends on the completed per-image vector (the SE FCs)
constexpr long long ROWRED_WS_FLOATS = 4LL << 20;
constexpr int ROWRED_TICKETS = 65536;
__device__ float g_rowred_ws[ROWRED_WS_FLOATS];
__device__ int g_rowred_tk[ROWRED_TICKETS];

struct SeFwdArgs {          // squeeze-excite forward chain behind a pooling (Wr == NULL: plain pooling)
    const float *Wr, *br, *We, *be;
    float* gate;            // [n, C]
    int Cse;
};
struct SeBwdArgs {          // squeeze-excite backward chain behind the gate-gradient reduction (Wr == NULL: reduce only)
    const float *pooled, *Wr, *br, *We, *be;
    float *d_e, *r, *d_rpre, *dpool;
    int Cse;
};

// 16-byte load of 4 consecutive floats when the address allows it (every arena array does; plain loads otherwise)
__device__ __forceinline__ float4 ldg_f4(const float* p) {
    if ((reinterpret_cast<uintptr_t>(p) & 15) == 0) return __ldg(reinterpret_cast<const float4*>(p));
    return make_float4(p[0], p[1], p[2], p[3]);
}

// the 8 per-channel operands of a thread (two 16-byte loads instead of eight 4-byte ones: on the small late layers the
// operand prologue was more load instructions than the data itself); p == NULL -> dflt
__device__ __forceinline__ void ldg_f8(const float* p, float* out, float dflt = 0.f) {
    if (!p) {
#pragma unroll
        for (int i = 0; i < 8; i++) out[i] = dflt;
        return;
    }
    const float4 a = ldg_f4(p), b = ldg_f4(p + 4);
    out[0] = a.x; out[1] = a.y; out[2] = a.z; out[3] = a.w;
    out[4] = b.x; out[5] = b.y; out[6] = b.z; out[7] = b.w;
}

struct RowGeom {
    dim3 block;
    dim3 grid;
    int rows_per_block;
};

// hw rows per image, n images; target enough CTAs to fill every SM a few times over
// max_threads: CTA size (256 by default) - target_blocks is scaled so that the resident thread count stays the same.
// 512-thread CTAs helped the two per-image reductions on the large layers (half as many cross-row reductions and tickets
// per image), changed nothing below 28x28 and slowed dfd_bn_act (no reduction to amortise, coarser tail) - on the GPU this code was first tuned on (not re-measured on the H100).
// DFD_ROW_MAXT forces a value for every user (diagnostic).
static int row_maxt(long long hw, bool reduces_per_image) {
    static int v = -1;
    if (v < 0) { const char* e = getenv("DFD_ROW_MAXT"); v = e ? atoi(e) : 0; if (v != 256 && v != 512 && v != 1024) v = 0; }
    if (v) return v;
    return reduces_per_image && hw >= 784 ? 512 : 256;
}
static RowGeom make_geom(int C, long long hw, int n, int target_blocks = DFD_SMS * 6, int max_threads = 256) {
    RowGeom g;
    int V = C / 8;
    int RY = V >= max_threads ? 1 : (max_threads / V);
    if (max_threads > 256 && target_blocks > 1) target_blocks = target_blocks * 256 / max_threads;
    if (RY > 64) RY = 64;
    if ((long long)RY > hw) RY = (int)hw;
    if (RY < 1) RY = 1;
    g.block = dim3(V, RY, 1);
    long long chunks = (target_blocks + n - 1) / n;
    long long max_chunks = (hw + RY - 1) / RY;
    if (chunks > max_chunks) chunks = max_chunks;
    if (chunks < 1) chunks = 1;
    long long rpb = (hw + chunks - 1) / chunks;
    rpb = ((rpb + RY - 1) / RY) * RY;
    chunks = (hw + rpb - 1) / rpb;
    g.rows_per_block = (int)rpb;
    g.grid = dim3((unsigned)chunks, (unsigned)n, 1);
    return g;
}

// block-level reduction of per-thread 8-vectors across threadIdx.y, then `fn(channel, value)` once per channel
// smem: float[RY][V*8] (caller provides dynamic smem)
template <typename F>
__device__ __forceinline__ void reduce_rows_and_emit(float* sm, const float* acc, F fn) {
    const int V = blockDim.x, RY = blockDim.y;
    const int C = V * 8;
    float* mine = sm + (size_t)threadIdx.y * C + threadIdx.x * 8;
#pragma unroll
    for (int i = 0; i < 8; i++) mine[i] = acc[i];
    __syncthreads();
    const int tid = threadIdx.y * V + threadIdx.x;
    for (int c = tid; c < C; c += V * RY) {
        float s = 0.f;
        for (int r = 0; r < RY; r++) s += sm[(size_t)r * C + c];
        fn(c, s);
    }
    __syncthreads();
}

// ---------------------------------------------------------------------------------------------
// column statistics of a [M, C] tensor: dsum[c] += sum_m y, dsq[c] += sum_m y^2   (fp64 atomics)
// ---------------------------------------------------------------------------------------------
template <typename T>
__global__ void colstats_kernel(const T* __restrict__ y, long long hw, int rows_per_block,
                                double* __restrict__ dsum, double* __restrict__ dsq) {
    extern __shared__ float sm[];
    const int V = blockDim.x, C = V * 8;
    const long long r0 = (long long)blockIdx.x * rows_per_block;
    long long r1 = r0 + rows_per_block;
    if (r1 > hw) r1 = hw;
    const T* base = y + (size_t)blockIdx.y * hw * C + threadIdx.x * 8;
    float s[8], q[8];
#pragma unroll
    for (int i = 0; i < 8; i++) { s[i] = 0.f; q[i] = 0.f; }
    for (long long r = r0 + threadIdx.y; r < r1; r += blockDim.y) {
        float f[8];
        unpack8<T>(ldg16(base + (size_t)r * C), f);
#pragma unroll
        for (int i = 0; i < 8; i++) { s[i] += f[i]; q[i] = fmaf(f[i], f[i], q[i]); }
    }
    double* ps = stat_slot(dsum, C);
    double* pq = stat_slot(dsq, C);
    reduce_rows_and_emit(sm, s, [&](int c, float v) { atomicAdd(ps + c, (double)v); });
    reduce_rows_and_emit(sm, q, [&](int c, float v) { atomicAdd(pq + c, (double)v); });
}

// ---------------------------------------------------------------------------------------------
// BN finalise: batch statistics -> (scale, shift, mean, rstd) + running-stat EMA (unbiased var)
// ---------------------------------------------------------------------------------------------
__global__ void bn_finalize_kernel(const double* __restrict__ dsum, const double* __restrict__ dsq, double inv_count,
                                   double unbias,
                                   const float* __restrict__ gamma, const float* __restrict__ beta,
                                   float* __restrict__ running_mean, float* __restrict__ running_var,
                                   long long* __restrict__ nbt, float momentum, float eps, int training, int C,
                                   float* __restrict__ scale, float* __restrict__ shift,
                                   float* __restrict__ mean_out, float* __restrict__ rstd_out) {
    int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c == 0 && training && nbt) *nbt += 1;
    if (c >= C) return;
    float mean, var;
    if (training) {
        // reciprocals come from the host: fp64 divisions are long dependent sequences on this part and these one-block
        // kernels sit on the critical path of every layer
        double m = stat_total(dsum, C, c) * inv_count;
        double v = stat_total(dsq, C, c) * inv_count - m * m;
        if (v < 0) v = 0;
        mean = (float)m;
        var = (float)v;
        double unb = v * unbias;                 // count / (count - 1)
        running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * mean;
        running_var[c] = (1.f - momentum) * running_var[c] + momentum * (float)unb;
    } else {
        // eval: the folded constants rounded once from fp64, so each is within half an fp32 ulp of torch's exact
        // gamma / sqrt(rv + eps) and beta - rm * scale (rsqrtf plus a Newton step in fp32 was up to 1.7 ulp off rstd, and
        // shift inherited scale's error); this runs once per weight state, off the training step's critical path
        const double r = 1.0 / sqrt((double)running_var[c] + (double)eps);
        const double s = (double)gamma[c] * r;
        scale[c] = (float)s;
        shift[c] = (float)((double)beta[c] - (double)running_mean[c] * s);
        mean_out[c] = running_mean[c];
        rstd_out[c] = (float)r;
        return;
    }
    float rstd = rsqrtf(var + eps);
    // rsqrtf is 2 ulp; refine once so that eval-mode folding matches torch's 1/sqrt to fp32 round-off
    rstd = rstd * (1.5f - 0.5f * (var + eps) * rstd * rstd);
    float sc = gamma[c] * rstd;
    scale[c] = sc;
    shift[c] = beta[c] - mean * sc;
    mean_out[c] = mean;
    rstd_out[c] = rstd;
}

// ---------------------------------------------------------------------------------------------
// out = act(scale*y + shift) [* gate[n,c]] [+ res] [relu after the add]
// RES: 0 none, 1 add, 2 add then relu (ResNet block tail, resnet.py:172-173,243-244)
// ---------------------------------------------------------------------------------------------
template <typename T, int ACT, bool GATE, int RES>
__global__ void bn_act_kernel(const T* __restrict__ y, const float* __restrict__ scale,
                              const float* __restrict__ shift, const float* __restrict__ gate,
                              const T* __restrict__ res, T* __restrict__ out, long long hw, int rows_per_block) {
    const int V = blockDim.x, C = V * 8;
    const int c0 = threadIdx.x * 8;
    float sc[8], sh[8], gt[8];
    ldg_f8(scale ? scale + c0 : nullptr, sc, 1.f);
    ldg_f8(shift ? shift + c0 : nullptr, sh, 0.f);
    ldg_f8(GATE ? gate + (size_t)blockIdx.y * C + c0 : nullptr, gt, 1.f);
    const long long r0 = (long long)blockIdx.x * rows_per_block;
    long long r1 = r0 + rows_per_block;
    if (r1 > hw) r1 = hw;
    const size_t img = (size_t)blockIdx.y * hw * C + c0;
    // U rows per trip, all loads issued before any math: a thread with one 16-byte load in flight cannot keep HBM
    // busy at the occupancy these register counts allow (Little's law: tens of KB must be in flight per SM to sustain its share of the HBM rate)
    constexpr int U = RES ? 2 : 4;
    for (long long r = r0 + threadIdx.y; r < r1; r += (long long)U * blockDim.y) {
        uint4 raw[U], rraw[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
            const long long rr = r + (long long)u * blockDim.y;
            if (rr < r1) {
                raw[u] = ldg16(y + img + (size_t)rr * C);
                if (RES) rraw[u] = ldg16(res + img + (size_t)rr * C);
            }
        }
#pragma unroll
        for (int u = 0; u < U; u++) {
            const long long rr = r + (long long)u * blockDim.y;
            if (rr >= r1) break;
            float f[8];
            unpack8<T>(raw[u], f);
#pragma unroll
            for (int i = 0; i < 8; i++) {
                float uu = fmaf(f[i], sc[i], sh[i]);
                f[i] = act_fwd<ACT>(uu);
                if (GATE) f[i] *= gt[i];
            }
            if (RES) {
                float g[8];
                unpack8<T>(rraw[u], g);
#pragma unroll
                for (int i = 0; i < 8; i++) {
                    f[i] += g[i];
                    if (RES == 2) f[i] = fmaxf(f[i], 0.f);
                }
            }
            stg16(out + img + (size_t)rr * C, pack8<T>(f));
        }
    }
}

// ---------------------------------------------------------------------------------------------
// pooled[n,c] = mean_hw act(scale*y + shift)       (one CTA per image: deterministic, no atomics)
// ---------------------------------------------------------------------------------------------
// SE_ACT: inner activation of the squeeze-excite chain behind the pooling (se.Wr != NULL)
template <typename T, int ACT, int SE_ACT = DFD_ACT_SWISH>
__global__ void pool_kernel(const T* __restrict__ y, const float* __restrict__ scale,
                            const float* __restrict__ shift, float* __restrict__ pooled,
                            long long hw, long long rows_per_block, const SeFwdArgs se) {
    extern __shared__ float sm[];
    const int V = blockDim.x, C = V * 8;
    const int c0 = threadIdx.x * 8;
    float sc[8], sh[8], acc[8];
    ldg_f8(scale ? scale + c0 : nullptr, sc, 1.f);
    ldg_f8(shift ? shift + c0 : nullptr, sh, 0.f);
#pragma unroll
    for (int i = 0; i < 8; i++) acc[i] = 0.f;
    const T* base = y + (size_t)blockIdx.y * hw * C + c0;
    // gridDim.x row chunks per image: one (the usual case: the batch alone fills the GPU) stores the mean directly; several
    // write their partial sums to fixed slots of the library scratch and the last of them adds these in chunk order -
    // the forward stays bit-reproducible (no float atomics). 4 independent loads per thread keep HBM busy.
    const long long r0 = (long long)blockIdx.x * rows_per_block;
    long long r1 = r0 + rows_per_block;
    if (r1 > hw) r1 = hw;
    constexpr int U = 4;
    long long r = r0 + threadIdx.y;
    for (; r + (long long)(U - 1) * blockDim.y < r1; r += (long long)U * blockDim.y) {
        uint4 raw[U];
#pragma unroll
        for (int u = 0; u < U; u++) raw[u] = ldg16(base + (size_t)(r + (long long)u * blockDim.y) * C);
#pragma unroll
        for (int u = 0; u < U; u++) {
            float f[8];
            unpack8<T>(raw[u], f);
#pragma unroll
            for (int i = 0; i < 8; i++) acc[i] += act_fwd<ACT>(fmaf(f[i], sc[i], sh[i]));
        }
    }
    for (; r < r1; r += blockDim.y) {
        float f[8];
        unpack8<T>(ldg16(base + (size_t)r * C), f);
#pragma unroll
        for (int i = 0; i < 8; i++) acc[i] += act_fwd<ACT>(fmaf(f[i], sc[i], sh[i]));
    }
    const float inv = 1.f / (float)hw;
    float* dst = pooled + (size_t)blockIdx.y * C;
    float* pv = sm + (size_t)blockDim.y * C;         // [C] the image's pooled vector, [Cse] FC scratch behind it
    const int tid = threadIdx.y * blockDim.x + threadIdx.x, nt = blockDim.x * blockDim.y;
    if (gridDim.x == 1) {
        reduce_rows_and_emit(sm, acc, [&](int c, float v) { dst[c] = v * inv; pv[c] = v * inv; });
    } else {
        // several row chunks per image (the batch alone cannot fill the SMs): fixed-slot partials, added in chunk order by
        // the last chunk to arrive - the forward stays bit-reproducible (no float atomics)
        float* part = g_rowred_ws + ((size_t)blockIdx.x * gridDim.y + blockIdx.y) * C;
        reduce_rows_and_emit(sm, acc, [&](int c, float v) { part[c] = v; });
        __shared__ int s_last;
        __threadfence();
        __syncthreads();
        if (tid == 0) {
            const int t = atomicAdd(g_rowred_tk + blockIdx.y, 1);
            s_last = (t == (int)gridDim.x - 1);
            if (s_last) g_rowred_tk[blockIdx.y] = 0;
        }
        __syncthreads();
        if (!s_last) return;
        __threadfence();
        for (int c = tid; c < C; c += nt) {
            float v = 0.f;
            for (int k = 0; k < (int)gridDim.x; k++) v += __ldcg(g_rowred_ws + ((size_t)k * gridDim.y + blockIdx.y) * C + c);
            dst[c] = v * inv;
            pv[c] = v * inv;
        }
    }
    if (!se.Wr) return;
    __syncthreads();
    // the CTA that completed this image's squeeze carries on with its excite FCs (efficientnet_blocks.py:104-110)
    se_fwd_chain<SE_ACT>(pv, pv + C, se.Wr, se.br, se.We, se.be, se.gate + (size_t)blockIdx.y * C, C, se.Cse, tid, nt);
}

// ---------------------------------------------------------------------------------------------
// selectable global pool (avg / max / avgmax / catavgmax) + argmax, one pass
// ---------------------------------------------------------------------------------------------
// does (m_new, i_new) replace (m_cur, i_cur)?  torch's adaptive_max_pool2d scans row-major and replaces on `v > max || isnan(v)`:
// over any set of (value, index) pairs that gives the last NaN if there is one, else the max with the lowest index. This
// comparison yields exactly that for ANY two disjoint sets, so strided per-thread rows, rows of the CTA and row chunks all
// combine to the sequential result. i_cur == INT_MAX marks an empty set (loses every tie, so an all -inf column -> index 0).
__device__ __forceinline__ bool gp_takes(float m_new, int i_new, float m_cur, int i_cur) {
    if (m_new != m_new) return m_cur == m_cur || i_new > i_cur;
    if (m_cur != m_cur) return false;
    return m_new > m_cur || (m_new == m_cur && i_new < i_cur);
}

// max / argmax partials of the chunked pool, laid out like the sums in g_rowred_ws ([chunk][image][C]) and as large, so that
// dfd_global_pool can always use dfd_pool's chunk geometry (and hence its summation order)
__device__ float g_rowred_max[ROWRED_WS_FLOATS];
__device__ int g_rowred_arg[ROWRED_WS_FLOATS];

template <int PT>
__device__ __forceinline__ void gpool_emit(float* pooled, int* argmax, int n, int C, int c, float sum, float inv, float m, int i) {
    const float a = sum * inv;          // dfd_pool's mean, same operands
    if (PT == DFD_POOL_AVG) pooled[(size_t)n * C + c] = a;
    else if (PT == DFD_POOL_MAX) pooled[(size_t)n * C + c] = m;
    else if (PT == DFD_POOL_AVGMAX) pooled[(size_t)n * C + c] = 0.5f * (a + m);
    else { pooled[(size_t)n * 2 * C + c] = a; pooled[(size_t)n * 2 * C + C + c] = m; }
    if (argmax) argmax[(size_t)n * C + c] = i;
}

// one activation value: the sum term exactly as pool_kernel's `acc += act_fwd(u)` compiles (for Swish the product contracts
// into fma(u, sigmoid(u), acc)), so that the mean keeps dfd_pool's bits; the max sees the rounded act(u)
template <int ACT>
__device__ __forceinline__ float gpool_term(float u, float& acc) {
    if (ACT == DFD_ACT_SWISH) {
        const float s = sigmoid_fast(u);
        acc = fmaf(u, s, acc);
        return u * s;
    }
    const float v = act_fwd<ACT>(u);
    acc += v;
    return v;
}

// pool_kernel's geometry and sum order, plus a running (max, argmax) per thread channel; smem [3][RY][C]
template <typename T, int ACT, int PT>
__global__ void gpool_kernel(const T* __restrict__ y, const float* __restrict__ scale, const float* __restrict__ shift,
                             float* __restrict__ pooled, int* __restrict__ argmax, long long hw, long long rows_per_block) {
    extern __shared__ float sm[];
    const int V = blockDim.x, RY = blockDim.y, C = V * 8;
    const int c0 = threadIdx.x * 8;
    float sc[8], sh[8], acc[8], mx[8];
    int ix[8];
    ldg_f8(scale ? scale + c0 : nullptr, sc, 1.f);
    ldg_f8(shift ? shift + c0 : nullptr, sh, 0.f);
#pragma unroll
    for (int i = 0; i < 8; i++) { acc[i] = 0.f; mx[i] = -INFINITY; ix[i] = INT_MAX; }
    const T* base = y + (size_t)blockIdx.y * hw * C + c0;
    const long long r0 = (long long)blockIdx.x * rows_per_block;
    long long r1 = r0 + rows_per_block;
    if (r1 > hw) r1 = hw;
    constexpr int U = 4;
    long long r = r0 + threadIdx.y;
    for (; r + (long long)(U - 1) * blockDim.y < r1; r += (long long)U * blockDim.y) {
        uint4 raw[U];
#pragma unroll
        for (int u = 0; u < U; u++) raw[u] = ldg16(base + (size_t)(r + (long long)u * blockDim.y) * C);
#pragma unroll
        for (int u = 0; u < U; u++) {
            float f[8];
            unpack8<T>(raw[u], f);
            const int rr = (int)(r + (long long)u * blockDim.y);
#pragma unroll
            for (int i = 0; i < 8; i++) {
                const float v = gpool_term<ACT>(fmaf(f[i], sc[i], sh[i]), acc[i]);
                if (gp_takes(v, rr, mx[i], ix[i])) { mx[i] = v; ix[i] = rr; }
            }
        }
    }
    for (; r < r1; r += blockDim.y) {
        float f[8];
        unpack8<T>(ldg16(base + (size_t)r * C), f);
#pragma unroll
        for (int i = 0; i < 8; i++) {
            const float v = gpool_term<ACT>(fmaf(f[i], sc[i], sh[i]), acc[i]);
            if (gp_takes(v, (int)r, mx[i], ix[i])) { mx[i] = v; ix[i] = (int)r; }
        }
    }
    // rows of the CTA: sums in reduce_rows_and_emit's order, (max, argmax) by gp_takes
    float* rs = sm;
    float* rm = sm + (size_t)RY * C;
    int* ri = reinterpret_cast<int*>(sm + (size_t)2 * RY * C);
    {
        const size_t o = (size_t)threadIdx.y * C + c0;
#pragma unroll
        for (int i = 0; i < 8; i++) { rs[o + i] = acc[i]; rm[o + i] = mx[i]; ri[o + i] = ix[i]; }
    }
    __syncthreads();
    const float inv = 1.f / (float)hw;
    const int tid = threadIdx.y * V + threadIdx.x, nt = V * RY;
    const int n = blockIdx.y;
    const size_t slot = ((size_t)blockIdx.x * gridDim.y + n) * C;
    for (int c = tid; c < C; c += nt) {
        float s = 0.f, m = -INFINITY;
        int im = INT_MAX;
        for (int k = 0; k < RY; k++) {
            s += rs[(size_t)k * C + c];
            const float mk = rm[(size_t)k * C + c];
            const int ik = ri[(size_t)k * C + c];
            if (gp_takes(mk, ik, m, im)) { m = mk; im = ik; }
        }
        if (gridDim.x == 1) gpool_emit<PT>(pooled, argmax, n, C, c, s, inv, m, im);
        else { g_rowred_ws[slot + c] = s; g_rowred_max[slot + c] = m; g_rowred_arg[slot + c] = im; }
    }
    if (gridDim.x == 1) return;
    // several row chunks per image: fixed-slot partials, combined in chunk order by the last chunk to arrive (as pool_kernel)
    __shared__ int s_last;
    __threadfence();
    __syncthreads();
    if (tid == 0) {
        const int t = atomicAdd(g_rowred_tk + n, 1);
        s_last = (t == (int)gridDim.x - 1);
        if (s_last) g_rowred_tk[n] = 0;
    }
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    for (int c = tid; c < C; c += nt) {
        float s = 0.f, m = -INFINITY;
        int im = INT_MAX;
        for (int k = 0; k < (int)gridDim.x; k++) {
            const size_t o = ((size_t)k * gridDim.y + n) * C + c;
            s += __ldcg(g_rowred_ws + o);
            const float mk = __ldcg(g_rowred_max + o);
            const int ik = __ldcg(g_rowred_arg + o);
            if (gp_takes(mk, ik, m, im)) { m = mk; im = ik; }
        }
        gpool_emit<PT>(pooled, argmax, n, C, c, s, inv, m, im);
    }
}

// ---------------------------------------------------------------------------------------------
// BN backward, phase 1: s1[c] += sum g, s2[c] += sum g * xhat, xhat = (y - mean) * rstd
// RELU_MASK: g is first masked by (out > 0) (ResNet: gradient through the post-add ReLU)
// ---------------------------------------------------------------------------------------------
template <typename T, bool RELU_MASK>
__global__ void bn_bwd_reduce_kernel(const T* __restrict__ g, const T* __restrict__ y, const T* __restrict__ out,
                                     const float* __restrict__ mean, const float* __restrict__ rstd,
                                     long long hw, int rows_per_block, double* __restrict__ s1,
                                     double* __restrict__ s2, const BnBwdFinDesc* __restrict__ fin,
                                     T* __restrict__ gm_out = nullptr, const T* __restrict__ g2 = nullptr) {
    extern __shared__ float sm[];
    const int V = blockDim.x, C = V * 8;
    const int c0 = threadIdx.x * 8;
    float mu[8], rs[8], a1[8], a2[8];
#pragma unroll
    for (int i = 0; i < 8; i++) { a1[i] = 0.f; a2[i] = 0.f; }
    ldg_f8(mean + c0, mu);
    ldg_f8(rstd + c0, rs);
    const long long r0 = (long long)blockIdx.x * rows_per_block;
    long long r1 = r0 + rows_per_block;
    if (r1 > hw) r1 = hw;
    const size_t img = (size_t)blockIdx.y * hw * C + c0;
    constexpr int U = 2;
    for (long long r = r0 + threadIdx.y; r < r1; r += (long long)U * blockDim.y) {
        uint4 graw[U], yraw[U], oraw[U], g2raw[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
            const long long rr = r + (long long)u * blockDim.y;
            if (rr < r1) {
                const size_t off = img + (size_t)rr * C;
                graw[u] = ldg16(g + off);
                yraw[u] = ldg16(y + off);
                if (RELU_MASK) oraw[u] = ldg16(out + off);
                if (RELU_MASK && g2) g2raw[u] = ldg16(g2 + off);
            }
        }
#pragma unroll
        for (int u = 0; u < U; u++) {
            if (r + (long long)u * blockDim.y >= r1) break;
            float gg[8], yy[8];
            unpack8<T>(graw[u], gg);
            unpack8<T>(yraw[u], yy);
            if (RELU_MASK && g2) {
                // two-source gradient (main path + identity path of the block above): what dfd_add_inplace would have stored
                float hh[8];
                unpack8<T>(g2raw[u], hh);
#pragma unroll
                for (int i = 0; i < 8; i++) gg[i] = round_t<T>(gg[i] + hh[i]);
            }
            if (RELU_MASK) {
                float oo[8];
                unpack8<T>(oraw[u], oo);
#pragma unroll
                for (int i = 0; i < 8; i++) gg[i] = oo[i] > 0.f ? gg[i] : 0.f;
                // the masked gradient is also the gradient of the block's identity path: stored here, it saves the separate
                // ReLU-backward pass (one read of g and out, one write) over the same tensor
                if (gm_out) stg16(gm_out + img + (size_t)(r + (long long)u * blockDim.y) * C, pack8<T>(gg));
            }
#pragma unroll
            for (int i = 0; i < 8; i++) {
                a1[i] += gg[i];
                a2[i] = fmaf(gg[i], (yy[i] - mu[i]) * rs[i], a2[i]);
            }
        }
    }
    double* p1 = stat_slot(s1, C);
    double* p2 = stat_slot(s2, C);
    reduce_rows_and_emit(sm, a1, [&](int c, float v) { atomicAdd(p1 + c, (double)v); });
    reduce_rows_and_emit(sm, a2, [&](int c, float v) { atomicAdd(p2 + c, (double)v); });
    bn_bwd_finalize_tail(fin, threadIdx.y * blockDim.x + threadIdx.x, blockDim.x * blockDim.y);
}

// BN backward, phase 2 (per channel): parameter gradients and the affine coefficients of
//   dy = A*g + B*y + C  with A = gamma*rstd, B = -gamma*rstd^2*m2, C = -A*m1 - B*mean,
//   m1 = s1/count, m2 = s2/count.
__global__ void bn_bwd_finalize_kernel(const double* __restrict__ s1, const double* __restrict__ s2, double inv_count,
                                       const float* __restrict__ gamma, const float* __restrict__ mean,
                                       const float* __restrict__ rstd, float* __restrict__ dgamma,
                                       float* __restrict__ dbeta, float* __restrict__ cA, float* __restrict__ cB,
                                       float* __restrict__ cC, int C) {
    int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    double sum_g = stat_total(s1, C, c), sum_gx = stat_total(s2, C, c);
    dgamma[c] += (float)sum_gx;
    dbeta[c] += (float)sum_g;
    float m1 = (float)(sum_g * inv_count), m2 = (float)(sum_gx * inv_count);
    float A = gamma[c] * rstd[c];
    float B = -A * rstd[c] * m2;
    cA[c] = A;
    cB[c] = B;
    cC[c] = -A * m1 - B * mean[c];
}

// BN backward, phase 3: dy = A*g*mask + B*y + C  (materialised; the GEMMs consume plain operands)
template <typename T, bool RELU_MASK>
__global__ void bn_bwd_apply_kernel(const T* __restrict__ g, const T* __restrict__ y, const T* __restrict__ out,
                                    const float* __restrict__ cA, const float* __restrict__ cB,
                                    const float* __restrict__ cC, T* __restrict__ dy, long long hw,
                                    int rows_per_block) {
    const int V = blockDim.x, C = V * 8;
    const int c0 = threadIdx.x * 8;
    float A[8], B[8], Cc[8];
#pragma unroll
    for (int i = 0; i < 8; i++) { A[i] = 0.f; }
    ldg_f8(cA + c0, A);
    ldg_f8(cB + c0, B);
    ldg_f8(cC + c0, Cc);
    const long long r0 = (long long)blockIdx.x * rows_per_block;
    long long r1 = r0 + rows_per_block;
    if (r1 > hw) r1 = hw;
    const size_t img = (size_t)blockIdx.y * hw * C + c0;
    constexpr int U = RELU_MASK ? 2 : 4;   // 6-8 independent 16-byte loads in flight per thread (see bn_act_kernel)
    for (long long r = r0 + threadIdx.y; r < r1; r += (long long)U * blockDim.y) {
        uint4 graw[U], yraw[U], oraw[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
            const long long rr = r + (long long)u * blockDim.y;
            if (rr < r1) {
                const size_t off = img + (size_t)rr * C;
                graw[u] = ldg16(g + off);
                yraw[u] = ldg16(y + off);
                if (RELU_MASK) oraw[u] = ldg16(out + off);
            }
        }
#pragma unroll
        for (int u = 0; u < U; u++) {
            const long long rr = r + (long long)u * blockDim.y;
            if (rr >= r1) break;
            float gg[8], yy[8];
            unpack8<T>(graw[u], gg);
            unpack8<T>(yraw[u], yy);
            if (RELU_MASK) {
                float oo[8];
                unpack8<T>(oraw[u], oo);
#pragma unroll
                for (int i = 0; i < 8; i++) gg[i] = oo[i] > 0.f ? gg[i] : 0.f;
            }
#pragma unroll
            for (int i = 0; i < 8; i++) gg[i] = fmaf(A[i], gg[i], fmaf(B[i], yy[i], Cc[i]));
            stg16(dy + img + (size_t)rr * C, pack8<T>(gg));
        }
    }
}

// ---------------------------------------------------------------------------------------------
// SE backward reduce: draw[n,c] = sum_hw da[n,hw,c] * act(scale*y + shift)
// ---------------------------------------------------------------------------------------------
template <typename T, int ACT>
__global__ void se_bwd_reduce_kernel(const T* __restrict__ da, const T* __restrict__ y,
                                     const float* __restrict__ scale, const float* __restrict__ shift,
                                     float* __restrict__ draw, long long hw, long long rows_per_block, const SeBwdArgs se) {
    extern __shared__ float sm[];
    const int V = blockDim.x, C = V * 8;
    const int c0 = threadIdx.x * 8;
    float sc[8], sh[8], acc[8];
#pragma unroll
    for (int i = 0; i < 8; i++) acc[i] = 0.f;
    ldg_f8(scale + c0, sc);
    ldg_f8(shift + c0, sh);
    const size_t img = (size_t)blockIdx.y * hw * C + c0;
    // gridDim.x chunks per image (several when the batch alone cannot fill the SMs): partial sums meet in fp32 atomics on
    // the pre-zeroed output; a single chunk stores directly
    const long long r0 = (long long)blockIdx.x * rows_per_block;
    long long r1 = r0 + rows_per_block;
    if (r1 > hw) r1 = hw;
    for (long long r = r0 + threadIdx.y; r < r1; r += blockDim.y) {
        size_t off = img + (size_t)r * C;
        float d[8], f[8];
        unpack8<T>(ldg16(da + off), d);
        unpack8<T>(ldg16(y + off), f);
#pragma unroll
        for (int i = 0; i < 8; i++) acc[i] = fmaf(d[i], act_fwd<ACT>(fmaf(f[i], sc[i], sh[i])), acc[i]);
    }
    float* dst = draw + (size_t)blockIdx.y * C;
    const int tid = threadIdx.y * blockDim.x + threadIdx.x, nt = blockDim.x * blockDim.y;
    // chain scratch (after the row-reduction area): p [C] | de / draw [C] | rpre, r, drp [Cse] | r_part [nw][Cse]
    float* cs = sm + (size_t)blockDim.y * C;
    if (gridDim.x == 1) {
        reduce_rows_and_emit(sm, acc, [&](int c, float v) { dst[c] = v; cs[C + c] = v; });
    } else {
        // several chunks per image: fixed-slot partials [chunk][image][C] in the library scratch; the last chunk of an image
        // to arrive (ticket) adds them in chunk order - no fp32 atomics, the result does not depend on CTA arrival order
        float* part = g_rowred_ws + ((size_t)blockIdx.x * gridDim.y + blockIdx.y) * C;
        reduce_rows_and_emit(sm, acc, [&](int c, float v) { part[c] = v; });
        __shared__ int s_last;
        __threadfence();
        __syncthreads();
        if (tid == 0) {
            const int t = atomicAdd(g_rowred_tk + blockIdx.y, 1);
            s_last = (t == (int)gridDim.x - 1);
            if (s_last) g_rowred_tk[blockIdx.y] = 0;
        }
        __syncthreads();
        if (!s_last) return;
        __threadfence();
        for (int c = tid; c < C; c += nt) {
            float v = 0.f;
            for (int k = 0; k < (int)gridDim.x; k++) v += __ldcg(g_rowred_ws + ((size_t)k * gridDim.y + blockIdx.y) * C + c);
            dst[c] = v;
            cs[C + c] = v;
        }
    }
    if (!se.Wr) return;
    // the CTA that completed dL/dgate of this image carries on with the backward FC chain of its squeeze-excite
    const size_t n = blockIdx.y;
    for (int c = tid; c < C; c += nt) cs[c] = se.pooled[n * C + c];
    __syncthreads();
    se_bwd_chain(cs, cs + C, se.Wr, se.br, se.We, se.be, se.d_e + n * C, se.r + n * se.Cse, se.d_rpre + n * se.Cse,
                 se.dpool + n * C, C, se.Cse, tid, nt);
}

// ---------------------------------------------------------------------------------------------
// SE-ResNet block tail backward (senet.py:111-112, 220-221: out = relu(a * gate[n,c] + residual), a = act(scale*y + shift),
// act = identity for the bottleneck, ReLU for the basic block, :213-215):
//   gm = round16(g + g2) * (out > 0), stored (the gradient of the residual path and, times the gate, of a)
//   draw[n,c] = sum_hw gm * a                                             (dL/dgate)
// and the CTA that completes an image's draw runs the SEModule's backward FC chain with the ReLU inner activation.
// ---------------------------------------------------------------------------------------------
template <typename T, int ACT>
__global__ void relu_se_bwd_reduce_kernel(const T* __restrict__ g, const T* __restrict__ g2, const T* __restrict__ y,
                                          const T* __restrict__ out, const float* __restrict__ scale,
                                          const float* __restrict__ shift, T* __restrict__ gm, float* __restrict__ draw,
                                          long long hw, long long rows_per_block, const SeBwdArgs se) {
    extern __shared__ float sm[];
    const int V = blockDim.x, C = V * 8;
    const int c0 = threadIdx.x * 8;
    float sc[8], sh[8], acc[8];
#pragma unroll
    for (int i = 0; i < 8; i++) acc[i] = 0.f;
    ldg_f8(scale + c0, sc);
    ldg_f8(shift + c0, sh);
    const size_t img = (size_t)blockIdx.y * hw * C + c0;
    const long long r0 = (long long)blockIdx.x * rows_per_block;
    long long r1 = r0 + rows_per_block;
    if (r1 > hw) r1 = hw;
    constexpr int U = 2;
    for (long long r = r0 + threadIdx.y; r < r1; r += (long long)U * blockDim.y) {
        uint4 graw[U], g2raw[U], yraw[U], oraw[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
            const long long rr = r + (long long)u * blockDim.y;
            if (rr < r1) {
                const size_t off = img + (size_t)rr * C;
                graw[u] = ldg16(g + off);
                if (g2) g2raw[u] = ldg16(g2 + off);
                yraw[u] = ldg16(y + off);
                oraw[u] = ldg16(out + off);
            }
        }
#pragma unroll
        for (int u = 0; u < U; u++) {
            const long long rr = r + (long long)u * blockDim.y;
            if (rr >= r1) break;
            float gg[8], yy[8], oo[8];
            unpack8<T>(graw[u], gg);
            unpack8<T>(yraw[u], yy);
            unpack8<T>(oraw[u], oo);
            if (g2) {
                float hh[8];
                unpack8<T>(g2raw[u], hh);
#pragma unroll
                for (int i = 0; i < 8; i++) gg[i] = round_t<T>(gg[i] + hh[i]);
            }
#pragma unroll
            for (int i = 0; i < 8; i++) {
                gg[i] = oo[i] > 0.f ? gg[i] : 0.f;
                acc[i] = fmaf(gg[i], act_fwd<ACT>(fmaf(yy[i], sc[i], sh[i])), acc[i]);
            }
            stg16(gm + img + (size_t)rr * C, pack8<T>(gg));
        }
    }
    float* dst = draw + (size_t)blockIdx.y * C;
    const int tid = threadIdx.y * blockDim.x + threadIdx.x, nt = blockDim.x * blockDim.y;
    float* cs = sm + (size_t)blockDim.y * C;        // chain scratch, as in se_bwd_reduce_kernel
    if (gridDim.x == 1) {
        reduce_rows_and_emit(sm, acc, [&](int c, float v) { dst[c] = v; cs[C + c] = v; });
    } else {
        // fixed-slot partials [chunk][image][C], added in chunk order by the last chunk of the image to arrive
        float* part = g_rowred_ws + ((size_t)blockIdx.x * gridDim.y + blockIdx.y) * C;
        reduce_rows_and_emit(sm, acc, [&](int c, float v) { part[c] = v; });
        __shared__ int s_last;
        __threadfence();
        __syncthreads();
        if (tid == 0) {
            const int t = atomicAdd(g_rowred_tk + blockIdx.y, 1);
            s_last = (t == (int)gridDim.x - 1);
            if (s_last) g_rowred_tk[blockIdx.y] = 0;
        }
        __syncthreads();
        if (!s_last) return;
        __threadfence();
        for (int c = tid; c < C; c += nt) {
            float v = 0.f;
            for (int k = 0; k < (int)gridDim.x; k++) v += __ldcg(g_rowred_ws + ((size_t)k * gridDim.y + blockIdx.y) * C + c);
            dst[c] = v;
            cs[C + c] = v;
        }
    }
    const size_t n = blockIdx.y;
    for (int c = tid; c < C; c += nt) cs[c] = se.pooled[n * C + c];
    __syncthreads();
    se_bwd_chain<DFD_ACT_RELU>(cs, cs + C, se.Wr, se.br, se.We, se.be, se.d_e + n * C, se.r + n * se.Cse,
                               se.d_rpre + n * se.Cse, se.dpool + n * C, C, se.Cse, tid, nt);
}

// ---------------------------------------------------------------------------------------------
// gradient w.r.t. the BN output u = scale*y + shift behind an activation (+ optional SE gate and pooling):
//   gu = (da * gate[n,c] + dpool[n,c] * inv_hw) * act'(u)        (HAS_DA: da present; dpool may be null)
// plus the BN backward reductions of gu: s1 += sum gu, s2 += sum gu * xhat.
// ---------------------------------------------------------------------------------------------
// The six per-channel operands (BN scale / shift, -mean*rstd, rstd, SE gate, pooled gradient) live in SHARED memory, not in
// registers: with them in registers (48 of 122) only 2 CTAs x 256 threads fit an SM and 4 x 16 bytes in flight per thread
// (32 KB per SM) cannot cover the HBM latency (Little: ~44 KB). Layout [operand][half][V] float4, so that a warp's 16-byte
// reads are consecutive (conflict-free); 12 LDS.128 per row of 8 channels next to ~100 ALU instructions.
#ifndef ACTBWD_U_RELU
#define ACTBWD_U_RELU 3
#endif
// GP (global-pool gradient, no da, no gate): dpool is dpooled [n, P] of dfd_global_pool of type pool_type, the operand slots
// hold g_max (4), g_avg * inv_hw (5) and the argmax (6), and gin = g_avg / hw + (row == argmax) * g_max
template <typename T, int ACT, bool HAS_DA, int MAXT, int OCC, bool GP = false>
__global__ void __launch_bounds__(MAXT, OCC) act_bwd_kernel(const T* __restrict__ da, const T* __restrict__ y, const float* __restrict__ scale,
                               const float* __restrict__ shift, const float* __restrict__ mean,
                               const float* __restrict__ rstd, const float* __restrict__ gate,
                               const float* __restrict__ dpool, float inv_hw, T* __restrict__ gu, long long hw,
                               int rows_per_block, double* __restrict__ s1, double* __restrict__ s2,
                               const BnBwdFinDesc* __restrict__ fin, const int* __restrict__ argmax = nullptr,
                               int pool_type = DFD_POOL_AVG) {
    extern __shared__ __align__(16) float sm[];
    const int V = blockDim.x, C = V * 8;
    const int c0 = threadIdx.x * 8;
    const int tid = threadIdx.y * blockDim.x + threadIdx.x, nt = blockDim.x * blockDim.y;
    float4* ps = reinterpret_cast<float4*>(sm + (size_t)blockDim.y * C);      // behind the [RY][C] reduction scratch
    for (int e = tid; e < (GP ? 14 : 12) * V; e += nt) {
        const int k = e / (2 * V), rem = e - k * 2 * V, h = rem / V, v = rem - h * V;
        const int c = v * 8 + h * 4;
        float4 val;
        if (GP && k >= 4) {
            const size_t nC = (size_t)blockIdx.y * C;
            if (k == 6) {
                const int* a = argmax + nC + c;
                val = make_float4(__int_as_float(a[0]), __int_as_float(a[1]), __int_as_float(a[2]), __int_as_float(a[3]));
            } else if (pool_type == DFD_POOL_CATAVGMAX) {
                val = ldg_f4(dpool + 2 * nC + (k == 4 ? C : 0) + c);
            } else {
                const float4 d = ldg_f4(dpool + nC + c);
                const float f = pool_type == DFD_POOL_AVGMAX ? 0.5f : (k == 4 ? 1.f : 0.f);
                val = make_float4(d.x * f, d.y * f, d.z * f, d.w * f);
            }
            if (k == 5) val = make_float4(val.x * inv_hw, val.y * inv_hw, val.z * inv_hw, val.w * inv_hw);
        } else if (k == 0) val = ldg_f4(scale + c);
        else if (k == 1) val = ldg_f4(shift + c);
        else if (k == 2) {
            const float4 m = ldg_f4(mean + c), r = ldg_f4(rstd + c);
            val = make_float4(-m.x * r.x, -m.y * r.y, -m.z * r.z, -m.w * r.w);
        } else if (k == 3) val = ldg_f4(rstd + c);
        else if (k == 4) val = gate ? ldg_f4(gate + (size_t)blockIdx.y * C + c) : make_float4(1.f, 1.f, 1.f, 1.f);
        else {
            val = make_float4(0.f, 0.f, 0.f, 0.f);
            if (dpool) {
                const float4 d = ldg_f4(dpool + (size_t)blockIdx.y * C + c);
                val = make_float4(d.x * inv_hw, d.y * inv_hw, d.z * inv_hw, d.w * inv_hw);
            }
        }
        ps[e] = val;
    }
    __syncthreads();
    float a1[8], a2[8];
#pragma unroll
    for (int i = 0; i < 8; i++) { a1[i] = 0.f; a2[i] = 0.f; }
    const long long r0 = (long long)blockIdx.x * rows_per_block;
    long long r1 = r0 + rows_per_block;
    if (r1 > hw) r1 = hw;
    const size_t img = (size_t)blockIdx.y * hw * C + c0;
    // independent 16-byte loads in flight per thread: OCC 2 (128 registers, 512 threads per SM) 6; OCC 3 (80 registers) 4
    constexpr int U = OCC == 3 ? 2 : (HAS_DA ? (ACT == 1 ? 3 : ACTBWD_U_RELU) : 4);
    for (long long r = r0 + threadIdx.y; r < r1; r += (long long)U * blockDim.y) {
        uint4 draw_[U], yraw[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
            const long long rr = r + (long long)u * blockDim.y;
            if (rr < r1) {
                const size_t off = img + (size_t)rr * C;
                if (HAS_DA) draw_[u] = ldg16(da + off);
                yraw[u] = ldg16(y + off);
            }
        }
#pragma unroll
        for (int u = 0; u < U; u++) {
            const long long rr = r + (long long)u * blockDim.y;
            if (rr >= r1) break;
            float d[8], f[8];
            if (HAS_DA) unpack8<T>(draw_[u], d);
            unpack8<T>(yraw[u], f);
#pragma unroll
            for (int h = 0; h < 2; h++) {
                if (OCC == 3) asm volatile("" ::: "memory");     // keep one half's operands live at a time
                const float4 sc4 = ps[(0 * 2 + h) * V + threadIdx.x], sh4 = ps[(1 * 2 + h) * V + threadIdx.x];
                const float4 nm4 = ps[(2 * 2 + h) * V + threadIdx.x], rs4 = ps[(3 * 2 + h) * V + threadIdx.x];
                const float4 gt4 = ps[(4 * 2 + h) * V + threadIdx.x], dp4 = ps[(5 * 2 + h) * V + threadIdx.x];
                const float sc[4] = {sc4.x, sc4.y, sc4.z, sc4.w}, sh[4] = {sh4.x, sh4.y, sh4.z, sh4.w};
                const float nm[4] = {nm4.x, nm4.y, nm4.z, nm4.w}, rs[4] = {rs4.x, rs4.y, rs4.z, rs4.w};
                const float gt[4] = {gt4.x, gt4.y, gt4.z, gt4.w}, dp[4] = {dp4.x, dp4.y, dp4.z, dp4.w};
                int am[4] = {0, 0, 0, 0};
                if (GP) {
                    const float4 am4 = ps[(6 * 2 + h) * V + threadIdx.x];
                    am[0] = __float_as_int(am4.x); am[1] = __float_as_int(am4.y);
                    am[2] = __float_as_int(am4.z); am[3] = __float_as_int(am4.w);
                }
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    const int i = h * 4 + j;
                    float uu = fmaf(f[i], sc[j], sh[j]);
                    float gin = HAS_DA ? fmaf(d[i], gt[j], dp[j]) : dp[j];
                    if (GP && rr == (long long)am[j]) gin = dp[j] + gt[j];          // gt holds g_max here
                    float o = gin * act_bwd<ACT>(uu);
                    // the stored (rounded) value is what the consumers see: reduce the rounded value
                    o = round_t<T>(o);
                    d[i] = o;
                    a1[i] += o;
                    a2[i] = fmaf(o, fmaf(f[i], rs[j], nm[j]), a2[i]);      // xhat = (y - mean) * rstd
                }
            }
            stg16(gu + img + (size_t)rr * C, pack8<T>(d));
        }
    }
    double* p1 = stat_slot(s1, C);
    double* p2 = stat_slot(s2, C);
    reduce_rows_and_emit(sm, a1, [&](int c, float v) { atomicAdd(p1 + c, (double)v); });
    reduce_rows_and_emit(sm, a2, [&](int c, float v) { atomicAdd(p2 + c, (double)v); });
    bn_bwd_finalize_tail(fin, tid, nt);
}

// elementwise a += b (residual gradient accumulation) over a flat 16-bit tensor
template <typename T>
__global__ void add_inplace_kernel(T* __restrict__ a, const T* __restrict__ b, size_t nvec) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t stride = (size_t)gridDim.x * blockDim.x;
    for (; i < nvec; i += stride) {
        float x[8], z[8];
        unpack8<T>(ldg16(a + i * 8), x);
        unpack8<T>(ldg16(b + i * 8), z);
#pragma unroll
        for (int k = 0; k < 8; k++) x[k] += z[k];
        stg16(a + i * 8, pack8<T>(x));
    }
}

// ---------------------------------------------------------------------------------------------
// DropBlock (layers/drop.py:24-63) on the ResNet BatchNorm outputs, resnet.py:153-162,218-233: the block mask m (uint8 NHWC,
// dfd_drop_block_masks) and the normalising scale s = numel / (sum m + 1e-7), evaluated as torch evaluates
// `numel / tensor` (reciprocal, then the product) from the exact kept count in device memory - so one captured graph stays
// valid across steps.  ms = m ? s : 0 multiplies the BN output u = scale*y + shift.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float drop_block_scale(const unsigned long long* kept, long long numel) {
    return __fmul_rn(__frcp_rn(__fadd_rn((float)*kept, 1e-7f)), (float)numel);
}

__device__ __forceinline__ void unpack_mask8(const uint2 raw, float s, float* ms) {
#pragma unroll
    for (int i = 0; i < 8; i++) ms[i] = ((i < 4 ? raw.x >> (8 * i) : raw.y >> (8 * (i - 4))) & 0xffu) ? s : 0.f;
}

// forward.  RES 0: out = relu(u * ms [* gate[n,c]]);  RES 2: out = relu(u * ms [* gate[n,c]] + res)   (block tail with
// the drop-path gate, resnet.py:172-173,243-244)
template <typename T, bool GATE, int RES>
__global__ void bn_act_drop_kernel(const T* __restrict__ y, const float* __restrict__ scale, const float* __restrict__ shift,
                                   const unsigned char* __restrict__ mask, const unsigned long long* __restrict__ kept,
                                   long long numel, const float* __restrict__ gate, const T* __restrict__ res,
                                   T* __restrict__ out, long long hw, int rows_per_block) {
    const int V = blockDim.x, C = V * 8;
    const int c0 = threadIdx.x * 8;
    float sc[8], sh[8], gt[8];
    ldg_f8(scale + c0, sc);
    ldg_f8(shift + c0, sh);
    ldg_f8(GATE ? gate + (size_t)blockIdx.y * C + c0 : nullptr, gt, 1.f);
    const float s = drop_block_scale(kept, numel);
    const long long r0 = (long long)blockIdx.x * rows_per_block;
    long long r1 = r0 + rows_per_block;
    if (r1 > hw) r1 = hw;
    const size_t img = (size_t)blockIdx.y * hw * C + c0;
    constexpr int U = RES ? 2 : 4;
    for (long long r = r0 + threadIdx.y; r < r1; r += (long long)U * blockDim.y) {
        uint4 raw[U], rraw[U];
        uint2 mraw[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
            const long long rr = r + (long long)u * blockDim.y;
            if (rr < r1) {
                raw[u] = ldg16(y + img + (size_t)rr * C);
                mraw[u] = __ldg(reinterpret_cast<const uint2*>(mask + img + (size_t)rr * C));
                if (RES) rraw[u] = ldg16(res + img + (size_t)rr * C);
            }
        }
#pragma unroll
        for (int u = 0; u < U; u++) {
            const long long rr = r + (long long)u * blockDim.y;
            if (rr >= r1) break;
            float f[8], ms[8];
            unpack8<T>(raw[u], f);
            unpack_mask8(mraw[u], s, ms);
#pragma unroll
            for (int i = 0; i < 8; i++) {
                f[i] = fmaf(f[i], sc[i], sh[i]) * ms[i];
                if (GATE) f[i] *= gt[i];
            }
            if (RES) {
                float g[8];
                unpack8<T>(rraw[u], g);
#pragma unroll
                for (int i = 0; i < 8; i++) f[i] += g[i];
            }
#pragma unroll
            for (int i = 0; i < 8; i++) f[i] = fmaxf(f[i], 0.f);
            stg16(out + img + (size_t)rr * C, pack8<T>(f));
        }
    }
}

// backward through a dropped BN + ReLU site: gu = round16(da * ms) * (u > 0), stored and reduced for the BN backward
// (s1 += sum gu, s2 += sum gu * xhat), as act_bwd_kernel reduces the stored value
template <typename T>
__global__ void act_bwd_drop_kernel(const T* __restrict__ da, const T* __restrict__ y, const float* __restrict__ scale,
                                    const float* __restrict__ shift, const float* __restrict__ mean,
                                    const float* __restrict__ rstd, const unsigned char* __restrict__ mask,
                                    const unsigned long long* __restrict__ kept, long long numel, T* __restrict__ gu,
                                    long long hw, int rows_per_block, double* __restrict__ s1, double* __restrict__ s2) {
    extern __shared__ float sm[];
    const int V = blockDim.x, C = V * 8;
    const int c0 = threadIdx.x * 8;
    float sc[8], sh[8], mu[8], rs[8], a1[8], a2[8];
    ldg_f8(scale + c0, sc);
    ldg_f8(shift + c0, sh);
    ldg_f8(mean + c0, mu);
    ldg_f8(rstd + c0, rs);
#pragma unroll
    for (int i = 0; i < 8; i++) { a1[i] = 0.f; a2[i] = 0.f; mu[i] = -mu[i] * rs[i]; }
    const float s = drop_block_scale(kept, numel);
    const long long r0 = (long long)blockIdx.x * rows_per_block;
    long long r1 = r0 + rows_per_block;
    if (r1 > hw) r1 = hw;
    const size_t img = (size_t)blockIdx.y * hw * C + c0;
    constexpr int U = 2;
    for (long long r = r0 + threadIdx.y; r < r1; r += (long long)U * blockDim.y) {
        uint4 draw_[U], yraw[U];
        uint2 mraw[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
            const long long rr = r + (long long)u * blockDim.y;
            if (rr < r1) {
                const size_t off = img + (size_t)rr * C;
                draw_[u] = ldg16(da + off);
                yraw[u] = ldg16(y + off);
                mraw[u] = __ldg(reinterpret_cast<const uint2*>(mask + off));
            }
        }
#pragma unroll
        for (int u = 0; u < U; u++) {
            const long long rr = r + (long long)u * blockDim.y;
            if (rr >= r1) break;
            float d[8], f[8], ms[8];
            unpack8<T>(draw_[u], d);
            unpack8<T>(yraw[u], f);
            unpack_mask8(mraw[u], s, ms);
#pragma unroll
            for (int i = 0; i < 8; i++) {
                const float uu = fmaf(f[i], sc[i], sh[i]);
                const float o = uu > 0.f ? round_t<T>(d[i] * ms[i]) : 0.f;
                d[i] = o;
                a1[i] += o;
                a2[i] = fmaf(o, fmaf(f[i], rs[i], mu[i]), a2[i]);      // xhat = (y - mean) * rstd
            }
            stg16(gu + img + (size_t)rr * C, pack8<T>(d));
        }
    }
    double* p1 = stat_slot(s1, C);
    double* p2 = stat_slot(s2, C);
    reduce_rows_and_emit(sm, a1, [&](int c, float v) { atomicAdd(p1 + c, (double)v); });
    reduce_rows_and_emit(sm, a2, [&](int c, float v) { atomicAdd(p2 + c, (double)v); });
}

// block tail backward with DropBlock and / or drop path: gm = round16(g + g2) * (out > 0) is stored unmasked (the identity /
// downsample path's gradient); the main branch's last BN sees gd = round16(gm * ms * gate[n,c]), stored and reduced
template <typename T, bool MASK, bool GATE>
__global__ void relu_bn_bwd_reduce_drop_kernel(const T* __restrict__ g, const T* __restrict__ g2, const T* __restrict__ y,
                                               const T* __restrict__ out, T* __restrict__ gm_out,
                                               const unsigned char* __restrict__ mask,
                                               const unsigned long long* __restrict__ kept, long long numel,
                                               const float* __restrict__ gate, T* __restrict__ gd_out,
                                               const float* __restrict__ mean, const float* __restrict__ rstd, long long hw,
                                               int rows_per_block, double* __restrict__ s1, double* __restrict__ s2) {
    extern __shared__ float sm[];
    const int V = blockDim.x, C = V * 8;
    const int c0 = threadIdx.x * 8;
    float mu[8], rs[8], gt[8], a1[8], a2[8];
#pragma unroll
    for (int i = 0; i < 8; i++) { a1[i] = 0.f; a2[i] = 0.f; }
    ldg_f8(mean + c0, mu);
    ldg_f8(rstd + c0, rs);
    ldg_f8(GATE ? gate + (size_t)blockIdx.y * C + c0 : nullptr, gt, 1.f);
    const float s = MASK ? drop_block_scale(kept, numel) : 1.f;
    const long long r0 = (long long)blockIdx.x * rows_per_block;
    long long r1 = r0 + rows_per_block;
    if (r1 > hw) r1 = hw;
    const size_t img = (size_t)blockIdx.y * hw * C + c0;
    constexpr int U = 2;
    for (long long r = r0 + threadIdx.y; r < r1; r += (long long)U * blockDim.y) {
        uint4 graw[U], yraw[U], oraw[U], g2raw[U];
        uint2 mraw[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
            const long long rr = r + (long long)u * blockDim.y;
            if (rr < r1) {
                const size_t off = img + (size_t)rr * C;
                graw[u] = ldg16(g + off);
                yraw[u] = ldg16(y + off);
                oraw[u] = ldg16(out + off);
                if (g2) g2raw[u] = ldg16(g2 + off);
                if (MASK) mraw[u] = __ldg(reinterpret_cast<const uint2*>(mask + off));
            }
        }
#pragma unroll
        for (int u = 0; u < U; u++) {
            const long long rr = r + (long long)u * blockDim.y;
            if (rr >= r1) break;
            const size_t off = img + (size_t)rr * C;
            float gg[8], yy[8], oo[8], ms[8];
            unpack8<T>(graw[u], gg);
            unpack8<T>(yraw[u], yy);
            unpack8<T>(oraw[u], oo);
            if (g2) {
                float hh[8];
                unpack8<T>(g2raw[u], hh);
#pragma unroll
                for (int i = 0; i < 8; i++) gg[i] = round_t<T>(gg[i] + hh[i]);
            }
#pragma unroll
            for (int i = 0; i < 8; i++) gg[i] = oo[i] > 0.f ? gg[i] : 0.f;
            stg16(gm_out + off, pack8<T>(gg));
            if (MASK) unpack_mask8(mraw[u], s, ms);
#pragma unroll
            for (int i = 0; i < 8; i++) {
                float o = gg[i];
                if (MASK) o *= ms[i];
                if (GATE) o *= gt[i];
                o = round_t<T>(o);
                gg[i] = o;
                a1[i] += o;
                a2[i] = fmaf(o, (yy[i] - mu[i]) * rs[i], a2[i]);
            }
            stg16(gd_out + off, pack8<T>(gg));
        }
    }
    double* p1 = stat_slot(s1, C);
    double* p2 = stat_slot(s2, C);
    reduce_rows_and_emit(sm, a1, [&](int c, float v) { atomicAdd(p1 + c, (double)v); });
    reduce_rows_and_emit(sm, a2, [&](int c, float v) { atomicAdd(p2 + c, (double)v); });
}

static size_t reduce_smem(const RowGeom& g) { return (size_t)g.block.x * 8 * g.block.y * sizeof(float); }

// ---------------------------------------------------------------------------------------------
// 2x2 / stride-2 average pool of the ResNet-D shortcut: nn.AvgPool2d(2, 2, ceil_mode=True, count_include_pad=False)
// (resnet.py:263-277). Ho = ceil(H/2), Wo = ceil(W/2); a window clipped by an odd extent averages its 2 or 1 in-image
// values. The count is 4, 2 or 1, so dividing by it is exact in fp32 and each output is rounded once.
// Row geometry: a row is one output pixel (forward) or one input pixel (backward).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float avgpool2_inv_count(int oy, int ox, int H, int W) {
    const int ch = 2 * oy + 1 < H ? 2 : 1, cw = 2 * ox + 1 < W ? 2 : 1;
    return 1.0f / (float)(ch * cw);
}

// y = round16(((x00 + x01) + x10) + x11) * (1 / count)), the terms in row-major order, out-of-image ones left out
template <typename T>
__global__ void avgpool2_fwd_kernel(const T* __restrict__ x, T* __restrict__ y, int H, int W, int Wo, long long hwo,
                                   int rows_per_block) {
    const int V = blockDim.x, C = V * 8;
    const int c0 = threadIdx.x * 8;
    const long long r0 = (long long)blockIdx.x * rows_per_block;
    long long r1 = r0 + rows_per_block;
    if (r1 > hwo) r1 = hwo;
    const T* img = x + (size_t)blockIdx.y * H * W * C + c0;
    T* out = y + (size_t)blockIdx.y * hwo * C + c0;
    for (long long r = r0 + threadIdx.y; r < r1; r += blockDim.y) {
        const int oy = (int)(r / Wo), ox = (int)(r - (long long)oy * Wo);
        const int iy = 2 * oy, ix = 2 * ox;
        const bool right = ix + 1 < W, below = iy + 1 < H;
        uint4 raw[4];
        raw[0] = ldg16(img + ((size_t)iy * W + ix) * C);
        if (right) raw[1] = ldg16(img + ((size_t)iy * W + ix + 1) * C);
        if (below) raw[2] = ldg16(img + ((size_t)(iy + 1) * W + ix) * C);
        if (right && below) raw[3] = ldg16(img + ((size_t)(iy + 1) * W + ix + 1) * C);
        float s[8], f[8];
        unpack8<T>(raw[0], s);
        if (right) {
            unpack8<T>(raw[1], f);
#pragma unroll
            for (int i = 0; i < 8; i++) s[i] += f[i];
        }
        if (below) {
            unpack8<T>(raw[2], f);
#pragma unroll
            for (int i = 0; i < 8; i++) s[i] += f[i];
        }
        if (right && below) {
            unpack8<T>(raw[3], f);
#pragma unroll
            for (int i = 0; i < 8; i++) s[i] += f[i];
        }
        const float inv = avgpool2_inv_count(oy, ox, H, W);
#pragma unroll
        for (int i = 0; i < 8; i++) s[i] *= inv;
        stg16(out + (size_t)r * C, pack8<T>(s));
    }
}

// dx = round16(add + dy[y/2, x/2] * (1 / count)); add == NULL reads as zero. Every dx element is written by one thread
// that reads add at the same address first, so add may be dx itself.
template <typename T>
__global__ void avgpool2_bwd_add_kernel(const T* __restrict__ dy, const T* add, T* dx, int H, int W, int Ho, int Wo,
                                        int rows_per_block) {
    const int V = blockDim.x, C = V * 8;
    const int c0 = threadIdx.x * 8;
    const long long hw = (long long)H * W;
    const long long r0 = (long long)blockIdx.x * rows_per_block;
    long long r1 = r0 + rows_per_block;
    if (r1 > hw) r1 = hw;
    const T* g = dy + (size_t)blockIdx.y * Ho * Wo * C + c0;
    const size_t img = (size_t)blockIdx.y * hw * C + c0;
    for (long long r = r0 + threadIdx.y; r < r1; r += blockDim.y) {
        const int iy = (int)(r / W), ix = (int)(r - (long long)iy * W);
        const int oy = iy >> 1, ox = ix >> 1;
        float f[8];
        unpack8<T>(ldg16(g + ((size_t)oy * Wo + ox) * C), f);
        const float inv = avgpool2_inv_count(oy, ox, H, W);
        if (add) {
            float a[8];
            unpack8<T>(*reinterpret_cast<const uint4*>(add + img + (size_t)r * C), a);
#pragma unroll
            for (int i = 0; i < 8; i++) f[i] = fmaf(f[i], inv, a[i]);
        } else {
#pragma unroll
            for (int i = 0; i < 8; i++) f[i] *= inv;
        }
        stg16(dx + img + (size_t)r * C, pack8<T>(f));
    }
}

// Tail of a strided Xception block (xception.py:110-124): out = maxpool3x3s2p1(scale*y + shift) + (scale_s*ys + shift_s), the
// pooled BatchNorm output never stored and the sum rounded to 16 bit once. Windows are padded with -inf (the BN output can be
// negative); the arg-max is the first maximum in row-major window order (as dfd_maxpool_fwd and ATen), one byte per output,
// and is not written when idx == NULL (eval mode). Rows are output pixels.
template <typename T>
__global__ void bn_maxpool_add_kernel(const T* __restrict__ y, const float* __restrict__ scale, const float* __restrict__ shift,
                                      const T* __restrict__ ys, const float* __restrict__ scale_s,
                                      const float* __restrict__ shift_s, T* __restrict__ out, unsigned char* __restrict__ idx,
                                      int H, int W, int Wo, long long hwo, int rows_per_block) {
    const int V = blockDim.x, C = V * 8;
    const int c0 = threadIdx.x * 8;
    float sc[8], sh[8], ss[8], hs[8];
    ldg_f8(scale + c0, sc);
    ldg_f8(shift + c0, sh);
    ldg_f8(scale_s + c0, ss);
    ldg_f8(shift_s + c0, hs);
    const long long r0 = (long long)blockIdx.x * rows_per_block;
    long long r1 = r0 + rows_per_block;
    if (r1 > hwo) r1 = hwo;
    const T* x = y + (size_t)blockIdx.y * H * W * C + c0;
    const size_t img = (size_t)blockIdx.y * hwo * C + c0;
    for (long long r = r0 + threadIdx.y; r < r1; r += blockDim.y) {
        const int oy = (int)(r / Wo), ox = (int)(r - (long long)oy * Wo);
        float best[8], f[8];
        unsigned char bi[8];
#pragma unroll
        for (int j = 0; j < 8; j++) { best[j] = -INFINITY; bi[j] = 0; }
        for (int kh = 0; kh < 3; kh++) {
            const int iy = oy * 2 - 1 + kh;
            if (iy < 0 || iy >= H) continue;
            for (int kw = 0; kw < 3; kw++) {
                const int ix = ox * 2 - 1 + kw;
                if (ix < 0 || ix >= W) continue;
                unpack8<T>(ldg16(x + ((size_t)iy * W + ix) * C), f);
#pragma unroll
                for (int j = 0; j < 8; j++) {
                    const float u = fmaf(f[j], sc[j], sh[j]);
                    if (u > best[j]) { best[j] = u; bi[j] = (unsigned char)(kh * 3 + kw); }
                }
            }
        }
        unpack8<T>(ldg16(ys + img + (size_t)r * C), f);
#pragma unroll
        for (int j = 0; j < 8; j++) best[j] += fmaf(f[j], ss[j], hs[j]);
        stg16(out + img + (size_t)r * C, pack8<T>(best));
        if (idx) {
            uint2 pk;
            pk.x = bi[0] | (bi[1] << 8) | (bi[2] << 16) | (bi[3] << 24);
            pk.y = bi[4] | (bi[5] << 8) | (bi[6] << 16) | (bi[7] << 24);
            *reinterpret_cast<uint2*>(idx + img + (size_t)r * C) = pk;
        }
    }
}

// Backward of the pooled BatchNorm of bn_maxpool_add_kernel: gx[iy, ix] = round16(sum of gy over the (at most 2 x 2) windows
// whose arg-max is (iy, ix)) - a gather, no atomics - and in the same pass the BN-backward sums s1 += gx, s2 += gx * xhat,
// xhat = (y - mean) * rstd, of the rounded gx. Rows are input pixels.
template <typename T>
__global__ void maxpool_bn_bwd_reduce_kernel(const T* __restrict__ gy, const unsigned char* __restrict__ idx,
                                             const T* __restrict__ y, const float* __restrict__ mean,
                                             const float* __restrict__ rstd, T* __restrict__ gx, int H, int W, int Ho,
                                             int Wo, int rows_per_block, double* __restrict__ s1, double* __restrict__ s2) {
    extern __shared__ float sm[];
    const int V = blockDim.x, C = V * 8;
    const int c0 = threadIdx.x * 8;
    float mu[8], rs[8], a1[8], a2[8];
#pragma unroll
    for (int i = 0; i < 8; i++) { a1[i] = 0.f; a2[i] = 0.f; }
    ldg_f8(mean + c0, mu);
    ldg_f8(rstd + c0, rs);
    const long long hw = (long long)H * W;
    const long long r0 = (long long)blockIdx.x * rows_per_block;
    long long r1 = r0 + rows_per_block;
    if (r1 > hw) r1 = hw;
    const size_t oimg = (size_t)blockIdx.y * Ho * Wo * C + c0;
    const size_t img = (size_t)blockIdx.y * hw * C + c0;
    for (long long r = r0 + threadIdx.y; r < r1; r += blockDim.y) {
        const int iy = (int)(r / W), ix = (int)(r - (long long)iy * W);
        float acc[8], f[8];
#pragma unroll
        for (int j = 0; j < 8; j++) acc[j] = 0.f;
        for (int kh = 0; kh < 3; kh++) {        // window (oy, ox) holds the pixel at tap (iy + 1 - 2*oy, ix + 1 - 2*ox)
            const int ay = iy + 1 - kh;
            if (ay < 0 || (ay & 1) || (ay >> 1) >= Ho) continue;
            for (int kw = 0; kw < 3; kw++) {
                const int ax = ix + 1 - kw;
                if (ax < 0 || (ax & 1) || (ax >> 1) >= Wo) continue;
                const size_t o = oimg + ((size_t)(ay >> 1) * Wo + (ax >> 1)) * C;
                const uint2 pk = *reinterpret_cast<const uint2*>(idx + o);
                unpack8<T>(ldg16(gy + o), f);
                const unsigned char want = (unsigned char)(kh * 3 + kw);
#pragma unroll
                for (int j = 0; j < 8; j++) {
                    const unsigned char b = (unsigned char)(((j < 4 ? pk.x : pk.y) >> (8 * (j & 3))) & 0xff);
                    if (b == want) acc[j] += f[j];
                }
            }
        }
        const uint4 pk = pack8<T>(acc);
        stg16(gx + img + (size_t)r * C, pk);
        unpack8<T>(pk, acc);
        unpack8<T>(ldg16(y + img + (size_t)r * C), f);
#pragma unroll
        for (int i = 0; i < 8; i++) {
            a1[i] += acc[i];
            a2[i] = fmaf(acc[i], (f[i] - mu[i]) * rs[i], a2[i]);
        }
    }
    double* p1 = stat_slot(s1, C);
    double* p2 = stat_slot(s2, C);
    reduce_rows_and_emit(sm, a1, [&](int c, float v) { atomicAdd(p1 + c, (double)v); });
    reduce_rows_and_emit(sm, a2, [&](int c, float v) { atomicAdd(p2 + c, (double)v); });
}

}  // namespace

// =============================================================================================
// C ABI
// =============================================================================================
#define DISPATCH_T(dt, ...)                                              \
    if ((dt) == DFD_DT_BF16) { typedef bf16 T; __VA_ARGS__; }            \
    else if ((dt) == DFD_DT_FP16) { typedef __half T; __VA_ARGS__; }     \
    else return dfd_set_error(DFD_ERR_ARG, "bad dtype");

extern "C" {

int dfd_colstats(const void* y, int n, long long hw, int C, int dt, double* dsum, double* dsq, void* stream) {
    if (C % 8 || C <= 0 || hw <= 0 || n <= 0) return dfd_set_error(DFD_ERR_ARG, "dfd_colstats: C%8, sizes");
    RowGeom g = make_geom(C, hw, n);
    cudaStream_t st = (cudaStream_t)stream;
    DISPATCH_T(dt, (colstats_kernel<T><<<g.grid, g.block, reduce_smem(g), st>>>((const T*)y, hw, g.rows_per_block, dsum, dsq)));
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

int dfd_bn_finalize(const double* dsum, const double* dsq, double count, const float* gamma, const float* beta,
                    float* running_mean, float* running_var, long long* nbt, float momentum, float eps,
                    int training, int C, float* scale, float* shift, float* mean, float* rstd, void* stream) {
    if (C <= 0) return dfd_set_error(DFD_ERR_ARG, "dfd_bn_finalize: C");
    bn_finalize_kernel<<<cdiv(C, 128), 128, 0, (cudaStream_t)stream>>>(dsum, dsq, 1.0 / count, count > 1 ? count / (count - 1) : 1.0, gamma, beta, running_mean,
                                                                         running_var, nbt, momentum, eps, training, C,
                                                                         scale, shift, mean, rstd);
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

int dfd_bn_act(const void* y, const float* scale, const float* shift, const float* gate, const void* res, void* out,
               int n, long long hw, int C, int act, int res_mode, int dt, void* stream) {
    if (C % 8 || C <= 0 || hw <= 0 || n <= 0) return dfd_set_error(DFD_ERR_ARG, "dfd_bn_act: C%8, sizes");
    if ((res_mode != 0) != (res != nullptr)) return dfd_set_error(DFD_ERR_ARG, "dfd_bn_act: res/res_mode");
    RowGeom g = make_geom(C, hw, n, DFD_SMS * 6, row_maxt(hw, false));
    cudaStream_t st = (cudaStream_t)stream;
#define LAUNCH(ACT, GATE, RES)                                                                                    \
    bn_act_kernel<T, ACT, GATE, RES><<<g.grid, g.block, 0, st>>>((const T*)y, scale, shift, gate, (const T*)res, \
                                                                   (T*)out, hw, g.rows_per_block)
    int key = act * 100 + (gate ? 10 : 0) + res_mode;
    DISPATCH_T(dt, {
        switch (key) {
            case 0: LAUNCH(0, false, 0); break;
            case 1: LAUNCH(0, false, 1); break;
            case 2: LAUNCH(0, false, 2); break;
            case 10: LAUNCH(0, true, 0); break;        // drop-path scaling of a gradient (unit affine, per-sample gate)
            case 11: LAUNCH(0, true, 1); break;        // block tail with drop path: (scale*y + shift) * gate[n] + residual
            case 12: LAUNCH(0, true, 2); break;        // ResNet block tail with drop path: relu((scale*y + shift) * gate[n] + residual)
            case 212: LAUNCH(2, true, 2); break;       // SE-ResNet basic block tail: relu(relu(scale*y + shift) * gate[n,c] + residual)
            case 100: LAUNCH(1, false, 0); break;
            case 110: LAUNCH(1, true, 0); break;
            case 200: LAUNCH(2, false, 0); break;
            default: return dfd_set_error(DFD_ERR_UNSUPPORTED, "dfd_bn_act: (act, gate, res) combination");
        }
    });
#undef LAUNCH
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

// geometry of the per-image pools: one CTA per image while the batch fills the GPU; otherwise up to max_chunks row chunks per
// image (fixed-slot partials in the library scratch, combined in chunk order by the last chunk of the image to arrive)
static RowGeom pool_geom(int C, long long hw, int n, int max_chunks) {
    const bool chunked = max_chunks > 1 && n < 296 && n <= ROWRED_TICKETS;
    RowGeom g = make_geom(C, hw, n, chunked ? 592 : 1, row_maxt(hw, true));
    if (!chunked) { g.grid = dim3(1, n, 1); g.rows_per_block = (int)hw; }
    if ((int)g.grid.x > max_chunks && g.grid.x > 1) {
        long long rpb = (hw + max_chunks - 1) / max_chunks;
        rpb = ((rpb + g.block.y - 1) / g.block.y) * g.block.y;
        g.rows_per_block = (int)rpb;
        g.grid.x = (unsigned)((hw + rpb - 1) / rpb);
    }
    if ((long long)g.grid.x * n * C > ROWRED_WS_FLOATS) { g.grid = dim3(1, n, 1); g.rows_per_block = (int)hw; }
    return g;
}

static int launch_pool(const void* y, const float* scale, const float* shift, float* pooled, int n, long long hw, int C,
                       int act, int dt, int max_chunks, const SeFwdArgs& se, void* stream, int se_act = DFD_ACT_SWISH) {
    if (C % 8 || C <= 0 || hw <= 0 || n <= 0) return dfd_set_error(DFD_ERR_ARG, "dfd_pool: C%8, sizes");
    const RowGeom g = pool_geom(C, hw, n, max_chunks);
    cudaStream_t st = (cudaStream_t)stream;
    const long long rpb = g.rows_per_block;
    const size_t smem = reduce_smem(g) + (size_t)(C + se.Cse) * sizeof(float);
    if (smem > 48 * 1024) return dfd_set_error(DFD_ERR_UNSUPPORTED, "dfd_pool: channel count exceeds shared memory");
    DISPATCH_T(dt, {
        if (se_act == DFD_ACT_RELU && act == DFD_ACT_RELU) pool_kernel<T, 2, DFD_ACT_RELU><<<g.grid, g.block, smem, st>>>((const T*)y, scale, shift, pooled, hw, rpb, se);
        else if (se_act == DFD_ACT_RELU) pool_kernel<T, 0, DFD_ACT_RELU><<<g.grid, g.block, smem, st>>>((const T*)y, scale, shift, pooled, hw, rpb, se);
        else if (act == DFD_ACT_SWISH) pool_kernel<T, 1><<<g.grid, g.block, smem, st>>>((const T*)y, scale, shift, pooled, hw, rpb, se);
        else if (act == DFD_ACT_RELU) pool_kernel<T, 2><<<g.grid, g.block, smem, st>>>((const T*)y, scale, shift, pooled, hw, rpb, se);
        else pool_kernel<T, 0><<<g.grid, g.block, smem, st>>>((const T*)y, scale, shift, pooled, hw, rpb, se);
    });
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

int dfd_pool(const void* y, const float* scale, const float* shift, float* pooled, int n, long long hw, int C,
             int act, int dt, float* partial, int max_chunks, void* stream) {
    (void)partial;       // kept in the signature: the chunk partials now live in the library's own scratch
    SeFwdArgs se = {nullptr, nullptr, nullptr, nullptr, nullptr, 0};
    return launch_pool(y, scale, shift, pooled, n, hw, C, act, dt, max_chunks, se, stream);
}

int dfd_global_pool(const void* y, const float* scale, const float* shift, float* pooled, int* argmax, int n, long long hw,
                    int C, int act, int pool_type, int dt, int max_chunks, void* stream) {
    if (C % 8 || C <= 0 || hw <= 0 || n <= 0 || hw > INT_MAX) return dfd_set_error(DFD_ERR_ARG, "dfd_global_pool: C%8, sizes");
    if (pool_type < DFD_POOL_AVG || pool_type > DFD_POOL_CATAVGMAX) return dfd_set_error(DFD_ERR_ARG, "dfd_global_pool: pool_type");
    if (act != DFD_ACT_NONE && act != DFD_ACT_SWISH && act != DFD_ACT_RELU) return dfd_set_error(DFD_ERR_ARG, "dfd_global_pool: act");
    // dfd_pool's geometry, so the mean is summed in dfd_pool's order (the max scratch is as large as the sums')
    const RowGeom g = pool_geom(C, hw, n, max_chunks);
    cudaStream_t st = (cudaStream_t)stream;
    const long long rpb = g.rows_per_block;
    const size_t smem = 3 * reduce_smem(g);       // sums, maxima, argmax per row of the CTA
    if (smem > 48 * 1024) return dfd_set_error(DFD_ERR_UNSUPPORTED, "dfd_global_pool: channel count exceeds shared memory");
#define GP_LAUNCH(ACT, PT) gpool_kernel<T, ACT, PT><<<g.grid, g.block, smem, st>>>((const T*)y, scale, shift, pooled, argmax, hw, rpb)
#define GP_ACT(PT)                                            \
    if (act == DFD_ACT_SWISH) GP_LAUNCH(DFD_ACT_SWISH, PT);    \
    else if (act == DFD_ACT_RELU) GP_LAUNCH(DFD_ACT_RELU, PT); \
    else GP_LAUNCH(DFD_ACT_NONE, PT)
    DISPATCH_T(dt, {
        switch (pool_type) {
            case DFD_POOL_AVG: GP_ACT(DFD_POOL_AVG); break;
            case DFD_POOL_MAX: GP_ACT(DFD_POOL_MAX); break;
            case DFD_POOL_AVGMAX: GP_ACT(DFD_POOL_AVGMAX); break;
            default: GP_ACT(DFD_POOL_CATAVGMAX); break;
        }
    });
#undef GP_ACT
#undef GP_LAUNCH
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

// global pooling + the whole squeeze-excite gate in ONE launch: pooled[n,c] = mean_hw act(scale*y + shift), then
// gate[n,:] = sigmoid(We * swish(Wr * pooled[n,:] + br) + be) computed by the CTA that completed image n
int dfd_pool_se(const void* y, const float* scale, const float* shift, float* pooled, const float* Wr, const float* br,
                const float* We, const float* be, float* gate, int n, long long hw, int C, int Cse, int act, int dt,
                int max_chunks, void* stream) {
    if (!Wr || !br || !We || !be || !gate || Cse <= 0) return dfd_set_error(DFD_ERR_ARG, "dfd_pool_se: operands");
    SeFwdArgs se = {Wr, br, We, be, gate, Cse};
    return launch_pool(y, scale, shift, pooled, n, hw, C, act, dt, max_chunks, se, stream);
}

// SENet's SEModule (senet.py:67-86) on a BatchNorm output: pooled[n,c] = mean_hw act(scale*y + shift) (act NONE or RELU), then
// gate[n,:] = sigmoid(We * relu(Wr * pooled[n,:] + br) + be) by the CTA that completed image n
int dfd_pool_se_relu(const void* y, const float* scale, const float* shift, float* pooled, const float* Wr, const float* br,
                     const float* We, const float* be, float* gate, int n, long long hw, int C, int Cse, int act, int dt,
                     int max_chunks, void* stream) {
    if (!scale || !shift || !Wr || !br || !We || !be || !gate || Cse <= 0)
        return dfd_set_error(DFD_ERR_ARG, "dfd_pool_se_relu: operands");
    if (act != DFD_ACT_NONE && act != DFD_ACT_RELU) return dfd_set_error(DFD_ERR_ARG, "dfd_pool_se_relu: act");
    SeFwdArgs se = {Wr, br, We, be, gate, Cse};
    return launch_pool(y, scale, shift, pooled, n, hw, C, act, dt, max_chunks, se, stream, DFD_ACT_RELU);
}

int dfd_bn_bwd_reduce(const void* g_, const void* y, const void* out, const float* mean, const float* rstd, int n,
                      long long hw, int C, int dt, double* s1, double* s2, const void* fin, void* stream) {
    if (C % 8 || C <= 0 || hw <= 0 || n <= 0) return dfd_set_error(DFD_ERR_ARG, "dfd_bn_bwd_reduce: C%8, sizes");
    RowGeom g = make_geom(C, hw, n, DFD_SMS * 6, row_maxt(hw, false));
    cudaStream_t st = (cudaStream_t)stream;
    DISPATCH_T(dt, {
        if (out) bn_bwd_reduce_kernel<T, true><<<g.grid, g.block, reduce_smem(g), st>>>((const T*)g_, (const T*)y, (const T*)out, mean, rstd, hw, g.rows_per_block, s1, s2, (const BnBwdFinDesc*)fin);
        else bn_bwd_reduce_kernel<T, false><<<g.grid, g.block, reduce_smem(g), st>>>((const T*)g_, (const T*)y, nullptr, mean, rstd, hw, g.rows_per_block, s1, s2, (const BnBwdFinDesc*)fin);
    });
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

int dfd_bn_bwd_finalize(const double* s1, const double* s2, double count, const float* gamma, const float* mean,
                        const float* rstd, float* dgamma, float* dbeta, float* cA, float* cB, float* cC, int C,
                        void* stream) {
    if (C <= 0) return dfd_set_error(DFD_ERR_ARG, "dfd_bn_bwd_finalize: C");
    bn_bwd_finalize_kernel<<<cdiv(C, 128), 128, 0, (cudaStream_t)stream>>>(s1, s2, 1.0 / count, gamma, mean, rstd, dgamma,
                                                                             dbeta, cA, cB, cC, C);
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

// ReLU backward + BN backward reduction in one pass (ResNet block tail, resnet.py:172-173,243-244): gm = (g + g2) * (out > 0)
// is stored AND reduced (s1 += sum gm, s2 += sum gm * xhat); replaces [dfd_add_inplace,] dfd_relu_bwd, dfd_bn_bwd_reduce.
// g2 (optional): second gradient source - the residual add of the block above (main path + identity path), rounded to the
// 16-bit type before the mask exactly as the materialised sum was
int dfd_relu_bn_bwd_reduce(const void* g_, const void* g2, const void* y, const void* out, void* gm, const float* mean,
                           const float* rstd, int n, long long hw, int C, int dt, double* s1, double* s2, void* stream) {
    if (C % 8 || C <= 0 || hw <= 0 || n <= 0) return dfd_set_error(DFD_ERR_ARG, "dfd_relu_bn_bwd_reduce: C%8, sizes");
    if (!out || !gm) return dfd_set_error(DFD_ERR_ARG, "dfd_relu_bn_bwd_reduce: operands");
    RowGeom g = make_geom(C, hw, n, DFD_SMS * 6, row_maxt(hw, false));
    cudaStream_t st = (cudaStream_t)stream;
    DISPATCH_T(dt, (bn_bwd_reduce_kernel<T, true><<<g.grid, g.block, reduce_smem(g), st>>>((const T*)g_, (const T*)y, (const T*)out, mean, rstd,
                                                                                           hw, g.rows_per_block, s1, s2, nullptr, (T*)gm, (const T*)g2)));
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

int dfd_bn_bwd_apply(const void* g_, const void* y, const void* out, const float* cA, const float* cB,
                     const float* cC, void* dy, int n, long long hw, int C, int dt, void* stream) {
    if (C % 8 || C <= 0 || hw <= 0 || n <= 0) return dfd_set_error(DFD_ERR_ARG, "dfd_bn_bwd_apply: C%8, sizes");
    RowGeom g = make_geom(C, hw, n);
    cudaStream_t st = (cudaStream_t)stream;
    DISPATCH_T(dt, {
        if (out) bn_bwd_apply_kernel<T, true><<<g.grid, g.block, 0, st>>>((const T*)g_, (const T*)y, (const T*)out, cA, cB, cC, (T*)dy, hw, g.rows_per_block);
        else bn_bwd_apply_kernel<T, false><<<g.grid, g.block, 0, st>>>((const T*)g_, (const T*)y, nullptr, cA, cB, cC, (T*)dy, hw, g.rows_per_block);
    });
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

static int launch_se_bwd_reduce(const void* da, const void* y, const float* scale, const float* shift, float* draw, int n,
                                long long hw, int C, int dt, const SeBwdArgs& se, void* stream) {
    if (C % 8 || C <= 0 || hw <= 0 || n <= 0) return dfd_set_error(DFD_ERR_ARG, "dfd_se_bwd_reduce: C%8, sizes");
    // one CTA per image while the batch fills the GPU (>= 2 CTAs per SM); otherwise several row chunks per image
    RowGeom g = make_geom(C, hw, n, n >= 296 ? 1 : 592, row_maxt(hw, true));
    if ((long long)g.grid.x * n * C > ROWRED_WS_FLOATS || n > ROWRED_TICKETS) g = make_geom(C, hw, n, 1, row_maxt(hw, true));   // one chunk per image
    cudaStream_t st = (cudaStream_t)stream;
    const int nw = (int)(g.block.x * g.block.y) / 32;
    const size_t smem = reduce_smem(g) + (size_t)(2 * C + (3 + nw) * se.Cse) * sizeof(float);
    if (smem > 48 * 1024) {
        static bool attr[2] = {false, false};
        const int ti = dt == DFD_DT_FP16 ? 1 : 0;
        if (!attr[ti]) {
            cudaError_t e = dt == DFD_DT_FP16
                ? cudaFuncSetAttribute(se_bwd_reduce_kernel<__half, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024)
                : cudaFuncSetAttribute(se_bwd_reduce_kernel<bf16, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024);
            if (e != cudaSuccess) return dfd_set_cuda_error(e, __FILE__, __LINE__);
            attr[ti] = true;
        }
        if (smem > 160 * 1024) return dfd_set_error(DFD_ERR_UNSUPPORTED, "dfd_se_bwd: channel count exceeds shared memory");
    }
    DISPATCH_T(dt, (se_bwd_reduce_kernel<T, 1><<<g.grid, g.block, smem, st>>>((const T*)da, (const T*)y, scale, shift, draw, hw,
                                                                               (long long)g.rows_per_block, se)));
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

int dfd_se_bwd_reduce(const void* da, const void* y, const float* scale, const float* shift, float* draw, int n,
                      long long hw, int C, int dt, void* stream) {
    SeBwdArgs se = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, 0};
    return launch_se_bwd_reduce(da, y, scale, shift, draw, n, hw, C, dt, se, stream);
}

// dfd_se_bwd_reduce + the per-image backward FC chain of dfd_se_fc_bwd in ONE launch (the CTA that completes dL/dgate of
// image n runs the chain); the SE parameter gradients still take dfd_se_fc_wgrad afterwards
int dfd_se_bwd_chain(const void* da, const void* y, const float* scale, const float* shift, float* draw, const float* pooled,
                     const float* Wr, const float* br, const float* We, const float* be, float* d_e, float* r, float* d_rpre,
                     float* dpool, int n, long long hw, int C, int Cse, int dt, void* stream) {
    if (!pooled || !Wr || !br || !We || !be || !d_e || !r || !d_rpre || !dpool || Cse <= 0)
        return dfd_set_error(DFD_ERR_ARG, "dfd_se_bwd_chain: operands");
    SeBwdArgs se = {pooled, Wr, br, We, be, d_e, r, d_rpre, dpool, Cse};
    return launch_se_bwd_reduce(da, y, scale, shift, draw, n, hw, C, dt, se, stream);
}

// SE-ResNet block tail backward in one pass over the block output (relu_se_bwd_reduce_kernel), its SE chain with the ReLU
// inner activation in the CTA that completes each image; geometry and chunk order as dfd_se_bwd_chain
int dfd_relu_se_bwd_reduce(const void* g_, const void* g2, const void* y, const void* out, const float* scale, const float* shift,
                           void* gm, float* draw, const float* pooled, const float* Wr, const float* br, const float* We,
                           const float* be, float* d_e, float* r, float* d_rpre, float* dpool, int n, long long hw, int C,
                           int Cse, int act, int dt, void* stream) {
    if (C % 8 || C <= 0 || hw <= 0 || n <= 0 || Cse <= 0) return dfd_set_error(DFD_ERR_ARG, "dfd_relu_se_bwd_reduce: C%8, sizes");
    if (act != DFD_ACT_NONE && act != DFD_ACT_RELU) return dfd_set_error(DFD_ERR_ARG, "dfd_relu_se_bwd_reduce: act");
    if (!g_ || !y || !out || !scale || !shift || !gm || !draw || !pooled || !Wr || !br || !We || !be || !d_e || !r || !d_rpre ||
        !dpool)
        return dfd_set_error(DFD_ERR_ARG, "dfd_relu_se_bwd_reduce: operands");
    RowGeom g = make_geom(C, hw, n, n >= 296 ? 1 : 592, row_maxt(hw, true));
    if ((long long)g.grid.x * n * C > ROWRED_WS_FLOATS || n > ROWRED_TICKETS) g = make_geom(C, hw, n, 1, row_maxt(hw, true));
    const int nw = (int)(g.block.x * g.block.y) / 32;
    const size_t smem = reduce_smem(g) + (size_t)(2 * C + (3 + nw) * Cse) * sizeof(float);
    if (smem > 48 * 1024) return dfd_set_error(DFD_ERR_UNSUPPORTED, "dfd_relu_se_bwd_reduce: channel count exceeds shared memory");
    SeBwdArgs se = {pooled, Wr, br, We, be, d_e, r, d_rpre, dpool, Cse};
    cudaStream_t st = (cudaStream_t)stream;
#define RSE_ARGS (const T*)g_, (const T*)g2, (const T*)y, (const T*)out, scale, shift, (T*)gm, draw, hw, (long long)g.rows_per_block, se
    DISPATCH_T(dt, {
        if (act == DFD_ACT_RELU) relu_se_bwd_reduce_kernel<T, DFD_ACT_RELU><<<g.grid, g.block, smem, st>>>(RSE_ARGS);
        else relu_se_bwd_reduce_kernel<T, DFD_ACT_NONE><<<g.grid, g.block, smem, st>>>(RSE_ARGS);
    });
#undef RSE_ARGS
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

int dfd_act_bwd(const void* da, const void* y, const float* scale, const float* shift, const float* mean,
                const float* rstd, const float* gate, const float* dpool, void* gu, int n, long long hw, int C,
                int act, int dt, double* s1, double* s2, const void* fin, void* stream) {
    if (C % 8 || C <= 0 || hw <= 0 || n <= 0) return dfd_set_error(DFD_ERR_ARG, "dfd_act_bwd: C%8, sizes");
    if (!da && !dpool) return dfd_set_error(DFD_ERR_ARG, "dfd_act_bwd: need da or dpool");
    RowGeom g = make_geom(C, hw, n);
    cudaStream_t st = (cudaStream_t)stream;
    float inv_hw = 1.f / (float)hw;
    const size_t smem_ab = reduce_smem(g) + (size_t)12 * g.block.x * sizeof(float4);     // + the per-channel operands
    if (smem_ab > 200 * 1024) return dfd_set_error(DFD_ERR_UNSUPPORTED, "dfd_act_bwd: channel count exceeds shared memory");
    static bool smem_attr[2][3][2][3] = {};
    static int occ3 = -1;
    if (occ3 < 0) { const char* e = getenv("DFD_ACTBWD_OCC3"); occ3 = e ? atoi(e) : 0; }
    // variant: 0 = 256 threads x 2 CTAs per SM with 6 loads in flight per thread (default), 1 = 256 x 3 with 4 loads in flight
    // (DFD_ACTBWD_OCC3, diagnostic: slower on the large layers and barely faster at 7x7 on the GPU this code was first tuned on (not re-measured on the H100)),
    // 2 = more than 2048 channels (one row of C / 8 threads)
    const int var = g.block.x * g.block.y > 256 ? 2 : (occ3 ? 1 : 0);
#define ABARGS (const T*)da, (const T*)y, scale, shift, mean, rstd, gate, dpool, inv_hw, (T*)gu, hw, g.rows_per_block, s1, s2, (const BnBwdFinDesc*)fin
#define LAUNCH(ACT, HAS) do {                                                                                       \
    if (smem_ab > 48 * 1024 && !smem_attr[(dt) == DFD_DT_FP16][ACT][HAS][var]) {                                     \
        cudaError_t e_ = var == 2 ? cudaFuncSetAttribute(act_bwd_kernel<T, ACT, HAS, 512, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024) \
                       : var == 1 ? cudaFuncSetAttribute(act_bwd_kernel<T, ACT, HAS, 256, 3>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024) \
                                  : cudaFuncSetAttribute(act_bwd_kernel<T, ACT, HAS, 256, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024); \
        if (e_ != cudaSuccess) return dfd_set_cuda_error(e_, __FILE__, __LINE__);                                    \
        smem_attr[(dt) == DFD_DT_FP16][ACT][HAS][var] = true;                                                        \
    }                                                                                                                \
    if (var == 2) act_bwd_kernel<T, ACT, HAS, 512, 1><<<g.grid, g.block, smem_ab, st>>>(ABARGS);                     \
    else if (var == 1) act_bwd_kernel<T, ACT, HAS, 256, 3><<<g.grid, g.block, smem_ab, st>>>(ABARGS);                \
    else act_bwd_kernel<T, ACT, HAS, 256, 2><<<g.grid, g.block, smem_ab, st>>>(ABARGS);                              \
    } while (0)
    DISPATCH_T(dt, {
        if (act == DFD_ACT_SWISH) { if (da) LAUNCH(1, true); else LAUNCH(1, false); }
        else if (act == DFD_ACT_RELU) { if (da) LAUNCH(2, true); else LAUNCH(2, false); }
        else { if (da) LAUNCH(0, true); else LAUNCH(0, false); }
    });
#undef LAUNCH
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

int dfd_act_bwd_gpool(const void* y, const float* scale, const float* shift, const float* mean, const float* rstd,
                      const float* dpooled, const int* argmax, void* gu, int n, long long hw, int C, int act, int pool_type,
                      int dt, double* s1, double* s2, const void* fin, void* stream) {
    if (C % 8 || C <= 0 || hw <= 0 || n <= 0 || hw > INT_MAX) return dfd_set_error(DFD_ERR_ARG, "dfd_act_bwd_gpool: C%8, sizes");
    if (!dpooled || !argmax) return dfd_set_error(DFD_ERR_ARG, "dfd_act_bwd_gpool: operands");
    if (pool_type != DFD_POOL_MAX && pool_type != DFD_POOL_AVGMAX && pool_type != DFD_POOL_CATAVGMAX)
        return dfd_set_error(DFD_ERR_ARG, "dfd_act_bwd_gpool: pool_type (avg: dfd_act_bwd)");
    if (act != DFD_ACT_SWISH && act != DFD_ACT_RELU)
        return dfd_set_error(DFD_ERR_UNSUPPORTED, "dfd_act_bwd_gpool: activation (Swish or ReLU)");
    RowGeom g = make_geom(C, hw, n);
    cudaStream_t st = (cudaStream_t)stream;
    const float inv_hw = 1.f / (float)hw;
    const size_t smem_ab = reduce_smem(g) + (size_t)14 * g.block.x * sizeof(float4);     // + g_max, g_avg / hw, argmax
    if (smem_ab > 200 * 1024) return dfd_set_error(DFD_ERR_UNSUPPORTED, "dfd_act_bwd_gpool: channel count exceeds shared memory");
    static bool smem_attr[2][2][2] = {};
    const int var = g.block.x * g.block.y > 256 ? 1 : 0;      // 1: more than 2048 channels (one row of C / 8 threads)
    const int relu = act == DFD_ACT_RELU;
#define GARGS nullptr, (const T*)y, scale, shift, mean, rstd, nullptr, dpooled, inv_hw, (T*)gu, hw, g.rows_per_block, s1, s2, \
              (const BnBwdFinDesc*)fin, argmax, pool_type
#define GLAUNCH(ACT_) do {                                                                                                      \
        if (smem_ab > 48 * 1024 && !smem_attr[dt == DFD_DT_FP16][relu][var]) {                                               \
            cudaError_t e_ = var ? cudaFuncSetAttribute(act_bwd_kernel<T, ACT_, false, 512, 1, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024) \
                                 : cudaFuncSetAttribute(act_bwd_kernel<T, ACT_, false, 256, 2, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024); \
            if (e_ != cudaSuccess) return dfd_set_cuda_error(e_, __FILE__, __LINE__);                                         \
            smem_attr[dt == DFD_DT_FP16][relu][var] = true;                                                                   \
        }                                                                                                                     \
        if (var) act_bwd_kernel<T, ACT_, false, 512, 1, true><<<g.grid, g.block, smem_ab, st>>>(GARGS);                       \
        else act_bwd_kernel<T, ACT_, false, 256, 2, true><<<g.grid, g.block, smem_ab, st>>>(GARGS);                           \
    } while (0)
    DISPATCH_T(dt, {
        if (relu) GLAUNCH(DFD_ACT_RELU);
        else GLAUNCH(DFD_ACT_SWISH);
    });
#undef GLAUNCH
#undef GARGS
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

int dfd_bn_act_drop(const void* y, const float* scale, const float* shift, const unsigned char* mask,
                    const unsigned long long* kept, long long numel, const float* gate, const void* res, void* out, int n,
                    long long hw, int C, int res_mode, int dt, void* stream) {
    if (C % 8 || C <= 0 || hw <= 0 || n <= 0) return dfd_set_error(DFD_ERR_ARG, "dfd_bn_act_drop: C%8, sizes");
    if (res_mode != 0 && res_mode != 2) return dfd_set_error(DFD_ERR_ARG, "dfd_bn_act_drop: res_mode");
    if ((res_mode != 0) != (res != nullptr)) return dfd_set_error(DFD_ERR_ARG, "dfd_bn_act_drop: res/res_mode");
    if (!scale || !shift) return dfd_set_error(DFD_ERR_ARG, "dfd_bn_act_drop: operands");
    // no mask (eval mode): the plain BN + ReLU or block tail, exactly as the undropped plan computes it
    if (!mask) return dfd_bn_act(y, scale, shift, gate, res, out, n, hw, C, res_mode ? DFD_ACT_NONE : DFD_ACT_RELU, res_mode, dt, stream);
    if (!kept || numel <= 0) return dfd_set_error(DFD_ERR_ARG, "dfd_bn_act_drop: kept count");
    RowGeom g = make_geom(C, hw, n, DFD_SMS * 6, row_maxt(hw, false));
    cudaStream_t st = (cudaStream_t)stream;
#define LAUNCH(GATE, RES)                                                                                            \
    bn_act_drop_kernel<T, GATE, RES><<<g.grid, g.block, 0, st>>>((const T*)y, scale, shift, mask, kept, numel, gate, \
                                                                  (const T*)res, (T*)out, hw, g.rows_per_block)
    DISPATCH_T(dt, {
        if (res_mode == 0) { if (gate) LAUNCH(true, 0); else LAUNCH(false, 0); }
        else { if (gate) LAUNCH(true, 2); else LAUNCH(false, 2); }
    });
#undef LAUNCH
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

int dfd_act_bwd_drop(const void* da, const void* y, const float* scale, const float* shift, const float* mean,
                     const float* rstd, const unsigned char* mask, const unsigned long long* kept, long long numel, void* gu,
                     int n, long long hw, int C, int dt, double* s1, double* s2, void* stream) {
    if (C % 8 || C <= 0 || hw <= 0 || n <= 0) return dfd_set_error(DFD_ERR_ARG, "dfd_act_bwd_drop: C%8, sizes");
    if (!da || !mask || !kept || numel <= 0) return dfd_set_error(DFD_ERR_ARG, "dfd_act_bwd_drop: operands");
    RowGeom g = make_geom(C, hw, n, DFD_SMS * 6, row_maxt(hw, false));
    cudaStream_t st = (cudaStream_t)stream;
    DISPATCH_T(dt, (act_bwd_drop_kernel<T><<<g.grid, g.block, reduce_smem(g), st>>>((const T*)da, (const T*)y, scale, shift, mean, rstd,
                                                                                    mask, kept, numel, (T*)gu, hw, g.rows_per_block, s1, s2)));
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

int dfd_relu_bn_bwd_reduce_drop(const void* g_, const void* g2, const void* y, const void* out, void* gm,
                                const unsigned char* mask, const unsigned long long* kept, long long numel, const float* gate,
                                void* gd, const float* mean, const float* rstd, int n, long long hw, int C, int dt, double* s1,
                                double* s2, void* stream) {
    if (C % 8 || C <= 0 || hw <= 0 || n <= 0) return dfd_set_error(DFD_ERR_ARG, "dfd_relu_bn_bwd_reduce_drop: C%8, sizes");
    if (!out || !gm || !gd || (!mask && !gate)) return dfd_set_error(DFD_ERR_ARG, "dfd_relu_bn_bwd_reduce_drop: operands");
    if (mask && (!kept || numel <= 0)) return dfd_set_error(DFD_ERR_ARG, "dfd_relu_bn_bwd_reduce_drop: kept count");
    RowGeom g = make_geom(C, hw, n, DFD_SMS * 6, row_maxt(hw, false));
    cudaStream_t st = (cudaStream_t)stream;
#define LAUNCH(MASK, GATE)                                                                                                      \
    relu_bn_bwd_reduce_drop_kernel<T, MASK, GATE><<<g.grid, g.block, reduce_smem(g), st>>>(                                      \
        (const T*)g_, (const T*)g2, (const T*)y, (const T*)out, (T*)gm, mask, kept, numel, gate, (T*)gd, mean, rstd, hw,        \
        g.rows_per_block, s1, s2)
    DISPATCH_T(dt, {
        if (mask) { if (gate) LAUNCH(true, true); else LAUNCH(true, false); }
        else LAUNCH(false, true);
    });
#undef LAUNCH
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

int dfd_add_inplace(void* a, const void* b, long long numel, int dt, void* stream) {
    if (numel % 8) return dfd_set_error(DFD_ERR_ARG, "dfd_add_inplace: numel%8");
    size_t nvec = (size_t)(numel / 8);
    int blocks = (int)((nvec + 255) / 256);
    if (blocks > DFD_SMS * 16) blocks = DFD_SMS * 16;
    cudaStream_t st = (cudaStream_t)stream;
    DISPATCH_T(dt, (add_inplace_kernel<T><<<blocks, 256, 0, st>>>((T*)a, (const T*)b, nvec)));
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

int dfd_avgpool2_fwd(const void* x, void* y, int N, int H, int W, int C, int dt, void* stream) {
    if (C % 8 || C <= 0 || C > 8192 || N <= 0 || H <= 0 || W <= 0)
        return dfd_set_error(DFD_ERR_ARG, "dfd_avgpool2_fwd: C%8, C <= 8192, sizes");
    const int Ho = (H + 1) / 2, Wo = (W + 1) / 2;
    RowGeom g = make_geom(C, (long long)Ho * Wo, N);
    DISPATCH_T(dt, (avgpool2_fwd_kernel<T><<<g.grid, g.block, 0, (cudaStream_t)stream>>>((const T*)x, (T*)y, H, W, Wo,
                                                                                        (long long)Ho * Wo, g.rows_per_block)));
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

int dfd_avgpool2_bwd_add(const void* dy, const void* add, void* dx, int N, int H, int W, int C, int dt, void* stream) {
    if (C % 8 || C <= 0 || C > 8192 || N <= 0 || H <= 0 || W <= 0)
        return dfd_set_error(DFD_ERR_ARG, "dfd_avgpool2_bwd_add: C%8, C <= 8192, sizes");
    const int Ho = (H + 1) / 2, Wo = (W + 1) / 2;
    RowGeom g = make_geom(C, (long long)H * W, N);
    DISPATCH_T(dt, (avgpool2_bwd_add_kernel<T><<<g.grid, g.block, 0, (cudaStream_t)stream>>>((const T*)dy, (const T*)add, (T*)dx,
                                                                                            H, W, Ho, Wo, g.rows_per_block)));
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

// out [N, Ho, Wo, C] = maxpool3x3s2p1(scale*y + shift) + scale_s*ys + shift_s, Ho = (H - 1) / 2 + 1 (Xception's strided block
// tail); idx (optional): the arg-max byte per output that dfd_maxpool_bn_bwd_reduce routes the gradient by
int dfd_bn_maxpool_add(const void* y, const float* scale, const float* shift, const void* ys, const float* scale_s,
                       const float* shift_s, void* out, void* idx, int N, int H, int W, int C, int dt, void* stream) {
    if (C % 8 || C <= 0 || C > 8192 || N <= 0 || H <= 0 || W <= 0)
        return dfd_set_error(DFD_ERR_ARG, "dfd_bn_maxpool_add: C%8, C <= 8192, sizes");
    if (!scale || !shift || !ys || !scale_s || !shift_s) return dfd_set_error(DFD_ERR_ARG, "dfd_bn_maxpool_add: operands");
    const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
    RowGeom g = make_geom(C, (long long)Ho * Wo, N);
    DISPATCH_T(dt, (bn_maxpool_add_kernel<T><<<g.grid, g.block, 0, (cudaStream_t)stream>>>((const T*)y, scale, shift, (const T*)ys,
        scale_s, shift_s, (T*)out, (unsigned char*)idx, H, W, Wo, (long long)Ho * Wo, g.rows_per_block)));
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

// gx [N, H, W, C]: the gradient of dfd_bn_maxpool_add's pooled BatchNorm output (gy routed by idx), and the BN-backward sums
// s1 += gx, s2 += gx * (y - mean) * rstd for dfd_bn_bwd_finalize
int dfd_maxpool_bn_bwd_reduce(const void* gy, const void* idx, const void* y, const float* mean, const float* rstd, void* gx,
                              int N, int H, int W, int C, int dt, double* s1, double* s2, void* stream) {
    if (C % 8 || C <= 0 || C > 8192 || N <= 0 || H <= 0 || W <= 0)
        return dfd_set_error(DFD_ERR_ARG, "dfd_maxpool_bn_bwd_reduce: C%8, C <= 8192, sizes");
    if (!gy || !idx || !y || !mean || !rstd || !gx || !s1 || !s2) return dfd_set_error(DFD_ERR_ARG, "dfd_maxpool_bn_bwd_reduce: operands");
    const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
    RowGeom g = make_geom(C, (long long)H * W, N);
    DISPATCH_T(dt, (maxpool_bn_bwd_reduce_kernel<T><<<g.grid, g.block, reduce_smem(g), (cudaStream_t)stream>>>((const T*)gy,
        (const unsigned char*)idx, (const T*)y, mean, rstd, (T*)gx, H, W, Ho, Wo, g.rows_per_block, s1, s2)));
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

}  // extern "C"
