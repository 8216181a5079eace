// Shared device helpers for the sm_90a kernels of the dfd train/validate hot path.
// Activations are NHWC in a 16-bit type T (bf16 or fp16); all arithmetic is fp32; per-channel
// statistics are accumulated in fp64 in HBM (one atomic per channel per CTA).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/dfd_b200.h"   // the C ABI: every definition is checked against its declaration

#define DFD_OK 0
#define DFD_ERR_ARG (-1)
#define DFD_ERR_CUDA (-2)
#define DFD_ERR_UNSUPPORTED (-3)

#define DFD_DT_BF16 0
#define DFD_DT_FP16 1

#define DFD_ACT_NONE 0
#define DFD_ACT_SWISH 1
#define DFD_ACT_RELU 2

typedef __nv_bfloat16 bf16;

#define DFD_LAUNCH_CHECK()                                   \
    do {                                                     \
        cudaError_t e__ = cudaGetLastError();                \
        if (e__ != cudaSuccess) return dfd_set_cuda_error(e__, __FILE__, __LINE__); \
    } while (0)

int dfd_set_cuda_error(cudaError_t e, const char* file, int line);
int dfd_set_error(int code, const char* msg);

// ------------------------------------------------------------------------------------------
// 16-bit <-> fp32 conversion of 8-element vectors (one 16-byte load/store per thread)
// ------------------------------------------------------------------------------------------
template <typename T> struct Vec2;
template <> struct Vec2<bf16> { typedef __nv_bfloat162 type; };
template <> struct Vec2<__half> { typedef __half2 type; };

template <typename T> __device__ __forceinline__ float2 unpack2(uint32_t u);
template <> __device__ __forceinline__ float2 unpack2<bf16>(uint32_t u) {
    // bf16 -> fp32 is a 16-bit shift
    float2 r;
    r.x = __uint_as_float(u << 16);
    r.y = __uint_as_float(u & 0xffff0000u);
    return r;
}
template <> __device__ __forceinline__ float2 unpack2<__half>(uint32_t u) {
    __half2 h = *reinterpret_cast<__half2*>(&u);
    return __half22float2(h);
}
template <typename T> __device__ __forceinline__ uint32_t pack2(float a, float b);
template <> __device__ __forceinline__ uint32_t pack2<bf16>(float a, float b) {
    __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
}
template <> __device__ __forceinline__ uint32_t pack2<__half>(float a, float b) {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
}

template <typename T> __device__ __forceinline__ void unpack8(const uint4& v, float* f) {
    float2 a = unpack2<T>(v.x), b = unpack2<T>(v.y), c = unpack2<T>(v.z), d = unpack2<T>(v.w);
    f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
}
template <typename T> __device__ __forceinline__ uint4 pack8(const float* f) {
    uint4 v;
    v.x = pack2<T>(f[0], f[1]); v.y = pack2<T>(f[2], f[3]);
    v.z = pack2<T>(f[4], f[5]); v.w = pack2<T>(f[6], f[7]);
    return v;
}
template <typename T> __device__ __forceinline__ float to_f(T x);
template <> __device__ __forceinline__ float to_f<bf16>(bf16 x) { return __bfloat162float(x); }
template <> __device__ __forceinline__ float to_f<__half>(__half x) { return __half2float(x); }
template <typename T> __device__ __forceinline__ T from_f(float x);
template <> __device__ __forceinline__ bf16 from_f<bf16>(float x) { return __float2bfloat16_rn(x); }
template <> __device__ __forceinline__ __half from_f<__half>(float x) { return __float2half_rn(x); }

// round a float through T and back (what a store + reload would do)
template <typename T> __device__ __forceinline__ float round_t(float x) { return to_f<T>(from_f<T>(x)); }

// streaming 16-byte global accesses
__device__ __forceinline__ uint4 ldg16(const void* p) { return __ldg(reinterpret_cast<const uint4*>(p)); }
__device__ __forceinline__ void stg16(void* p, const uint4& v) { *reinterpret_cast<uint4*>(p) = v; }

// ------------------------------------------------------------------------------------------
// activations. sigmoid via one MUFU op: sigma(x) = 0.5 * tanh(0.5 x) + 0.5
// (an SM has 16 MUFU lanes per clock; exp+rcp would make every swish pass MUFU-bound before HBM-bound)
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ float fast_tanh(float x) {
    float y;
    asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float sigmoid_fast(float x) { return fmaf(fast_tanh(0.5f * x), 0.5f, 0.5f); }
// precise variant for the tiny per-image vectors (SE gates, loss)
__device__ __forceinline__ float sigmoid_precise(float x) { return 1.0f / (1.0f + __expf(-x)); }

template <int ACT> __device__ __forceinline__ float act_fwd(float u) {
    if (ACT == DFD_ACT_SWISH) return u * sigmoid_fast(u);
    if (ACT == DFD_ACT_RELU) return fmaxf(u, 0.0f);
    return u;
}
// d act(u) / du  (reference: layers/activations.py:30-33 recomputes sigmoid from the pre-activation)
template <int ACT> __device__ __forceinline__ float act_bwd(float u) {
    if (ACT == DFD_ACT_SWISH) {
        float s = sigmoid_fast(u);
        return fmaf(s, fmaf(-u, s, u), s);      // s * (1 + u * (1 - s)) in two FMAs
    }
    if (ACT == DFD_ACT_RELU) return u > 0.0f ? 1.0f : 0.0f;
    return 1.0f;
}

// ------------------------------------------------------------------------------------------
// reductions
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Per-channel statistics are accumulated with fp64 atomics into DFD_STAT_SLOTS interleaved copies
// ([slot][C]) so that thousands of CTAs do not serialise on C addresses; the finalise kernels sum the slots.
#define DFD_STAT_SLOTS 8
__device__ __forceinline__ double* stat_slot(double* base, int C) {
    unsigned b = blockIdx.x + blockIdx.y * 7u + blockIdx.z * 13u;
    return base + (size_t)(b % DFD_STAT_SLOTS) * C;
}
__device__ __forceinline__ double stat_total(const double* base, int C, int c) {
    double s = 0.0;
#pragma unroll
    for (int i = 0; i < DFD_STAT_SLOTS; i++) s += base[(size_t)i * C + c];
    return s;
}

static inline int cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

// SM count of the target GPU (H100 SXM). Grid shapes are sized with it; it also fixes the split counts of the
// order-deterministic weight-gradient reductions, so those results do not depend on the device the library runs on.
#define DFD_SMS 132
