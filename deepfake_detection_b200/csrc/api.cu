// Error reporting, version and small runtime helpers of the C-ABI library.
#include <stdio.h>
#include <string.h>

#include "common.cuh"

static thread_local char g_err[512] = "";

int dfd_set_error(int code, const char* msg) {
    snprintf(g_err, sizeof(g_err), "%s", msg ? msg : "");
    return code;
}
int dfd_set_cuda_error(cudaError_t e, const char* file, int line) {
    snprintf(g_err, sizeof(g_err), "CUDA error %d (%s) at %s:%d", (int)e, cudaGetErrorString(e), file, line);
    return DFD_ERR_CUDA;
}

extern "C" {

const char* dfd_last_error(void) { return g_err; }

int dfd_abi_version(void) { return 1; }

int dfd_stat_slots(void) { return DFD_STAT_SLOTS; }

int dfd_memset_async(void* p, int value, long long bytes, void* stream) {
    cudaError_t e = cudaMemsetAsync(p, value, (size_t)bytes, (cudaStream_t)stream);
    if (e != cudaSuccess) return dfd_set_cuda_error(e, __FILE__, __LINE__);
    return DFD_OK;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------------------------------
// Order-deterministic reduction of split partial sums (the second half of the wgmma weight gradient and of the fused
// depthwise backward in workspace mode): for every table entry  dst[i] += sum_{p = 0 .. parts-1} src[p * stride + i],  i < n,
// the partials added in index order - whatever order the producing CTAs finished in.  One launch serves every entry
// (blockIdx.y); entries with many parts spread them over 32 part-lanes whose sums meet in a fixed order too.
// ---------------------------------------------------------------------------------------------------------------------
namespace {
struct RedDesc {
    const float* src;
    float* dst;
    long long n;          // floats per partial (multiple of 4; src / dst / stride 16-byte aligned)
    long long stride;     // floats between consecutive partials
    int parts;
    int _pad;
};

__global__ void __launch_bounds__(256) ordered_reduce_kernel(const RedDesc* __restrict__ table) {
    const RedDesc d = table[blockIdx.y];
    const long long n4 = d.n >> 2;
    const float4* src = reinterpret_cast<const float4*>(d.src);
    float4* dst = reinterpret_cast<float4*>(d.dst);
    const long long s4 = d.stride >> 2;
    if (d.parts <= 64) {
        for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n4; i += (long long)gridDim.x * 256) {
            float4 acc = dst[i];
#pragma unroll 8
            for (int p = 0; p < d.parts; p++) {
                const float4 a = __ldcg(src + p * s4 + i);
                acc.x += a.x; acc.y += a.y; acc.z += a.z; acc.w += a.w;
            }
            dst[i] = acc;
        }
        return;
    }
    __shared__ float4 sm[256];
    const int lane_p = threadIdx.x >> 3, e = threadIdx.x & 7;      // 32 part-lanes x 8 consecutive float4 per block trip
    const long long trips = (n4 + (long long)gridDim.x * 8 - 1) / ((long long)gridDim.x * 8);
    for (long long t = 0; t < trips; t++) {
        const long long i = (t * gridDim.x + blockIdx.x) * 8 + e;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        if (i < n4) {
#pragma unroll 4
            for (int p = lane_p; p < d.parts; p += 32) {
                const float4 a = __ldcg(src + p * s4 + i);
                acc.x += a.x; acc.y += a.y; acc.z += a.z; acc.w += a.w;
            }
        }
        sm[threadIdx.x] = acc;
        __syncthreads();
        if (lane_p == 0 && i < n4) {
            float4 tot = dst[i];
#pragma unroll 8
            for (int l = 0; l < 32; l++) {
                const float4 a = sm[l * 8 + e];
                tot.x += a.x; tot.y += a.y; tot.z += a.z; tot.w += a.w;
            }
            dst[i] = tot;
        }
        __syncthreads();
    }
}
}  // namespace

extern "C" int dfd_ordered_reduce(const void* table, int count, const float* first_dst, int blocks_x, void* stream) {
    (void)first_dst;       // lowest gradient address this launch writes: lets a host-side planner place it (no device use)
    if (count <= 0) return DFD_OK;
    if (!table || blocks_x <= 0) return dfd_set_error(DFD_ERR_ARG, "dfd_ordered_reduce: operands");
    // blocks_x: CTAs per entry. A CTA covers 256 float4 per trip of an entry with <= 64 parts and 8 float4 per trip of an
    // entry with more (32 part-lanes each); the caller sizes it for its largest entry (any value is correct)
    if (blocks_x > 2048) blocks_x = 2048;
    ordered_reduce_kernel<<<dim3((unsigned)blocks_x, (unsigned)count), 256, 0, (cudaStream_t)stream>>>((const RedDesc*)table);
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

