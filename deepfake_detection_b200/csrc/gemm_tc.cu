// Pointwise (1x1) convolution GEMM on the Hopper tensor-core path: TMA -> shared memory (128B swizzle) ->
// wgmma.mma_async (kind f16 / bf16, fp32 accumulators in registers) -> swizzled smem -> TMA store, with the per-channel
// BatchNorm statistics of the stored tile reduced in the same epilogue.
//
//   C[M,N] = A[M,K] * B[N,K]^T          A: NHWC activations / output gradients (K-contiguous rows)
//                                        B: conv weight [Cout,Cin] (forward) or its transpose [Cin,Cout] (dgrad)
//
// Replaces nn.Conv2d 1x1 (cuDNN/cuBLAS in the reference: dfd/timm/models/efficientnet_blocks.py:165,277,299,
// efficientnet.py:292, resnet.py:192,199) and its input-gradient (autograd, train.py:634-636).
//
// Shape regime (SURVEY.md 8a H1a): M = N*H*W is 12.5k .. 3.2M, K and N are 16 .. 1280 -> every instance is
// HBM-bound, so the design goal is to stream A and C at HBM rate, not MMA peak:
//   * persistent CTAs (one per SM), tiles 128 x BLOCK_N, BLOCK_N = whole N when N <= 128 (A is read once);
//   * K/N/M tails need no padding copies: TMA zero-fills out-of-bounds loads and clips stores;
//   * warp roles: w0 TMA producer (runs up to `stages` k-blocks ahead, so the loads of tile i+1 stream during the
//     epilogue of tile i); warpgroups 1 and 2 issue the MMAs of rows 0-63 / 64-127 of a tile and drain them.
#include <cuda.h>
#include <stdio.h>
#include <stdlib.h>

#include <type_traits>

#include "common.cuh"
#include "bn_finalize.cuh"

namespace {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;          // 64 x 2 B = one 128-byte swizzle row
constexpr int MMA_K = 16;
constexpr int SLAB = 64;             // epilogue / TMA-store column slab
constexpr int NUM_THREADS = 384;     // producer warpgroup (one active thread) + two MMA / epilogue warpgroups
constexpr int EPI_THREADS = 256;
constexpr int MAX_BLOCK_N = 128;
constexpr int SMEM_BUDGET = 224 * 1024;   // one CTA per SM (H100: up to 227 KB of shared memory per block)

__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarrier -------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_addr(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t addr = smem_addr(bar);
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra WAIT_DONE;\n"
        "bra WAIT_LOOP;\n"
        "WAIT_DONE:\n"
        "}\n" ::"r"(addr), "r"(parity) : "memory");
}

// ---- TMA ------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_addr(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_addr(bar)), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, const void* smem_src, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
                 ::"l"(reinterpret_cast<uint64_t>(map)), "r"(smem_addr(smem_src)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(smem_addr(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_addr(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* map, const void* smem_src, int c0, int c1, int c2, int c3) {
    asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
                 ::"l"(reinterpret_cast<uint64_t>(map)), "r"(smem_addr(smem_src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
// TMA reduction store: global (16-bit) += shared tile, element-wise add performed in L2 (round to nearest in the tensor's type)
__device__ __forceinline__ void tma_reduce_add_4d(const CUtensorMap* map, const void* smem_src, int c0, int c1, int c2, int c3) {
    asm volatile("cp.reduce.async.bulk.tensor.4d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
                 ::"l"(reinterpret_cast<uint64_t>(map)), "r"(smem_addr(smem_src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void tma_store_wait_read() {
    asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}

// ---- wgmma ----------------------------------------------------------------------------------
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { wgmma_wait<0>(); }
// keeps the compiler from touching the accumulators while an asynchronous MMA owns them
template <int R> __device__ __forceinline__ void fence_acc(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; i++) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x 64] (+)= A[64 x 16] * B[16 x 64], both operands from shared-memory descriptors; TA / TB = 1: that operand
// is MN-major. accumulate == 0 overwrites D.
template <typename T, int TA, int TB>
__device__ __forceinline__ void wgmma_n64(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    if constexpr (std::is_same<T, bf16>::value) {
        asm volatile(
            "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
            "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {"
            "%0,%1,%2,%3,%4,%5,%6,%7,"
            "%8,%9,%10,%11,%12,%13,%14,%15,"
            "%16,%17,%18,%19,%20,%21,%22,%23,"
            "%24,%25,%26,%27,%28,%29,%30,%31"
            "}, %32, %33, p, 1, 1, %35, %36;\n}\n"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
              "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
              "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
            : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(TA), "n"(TB));
    }
    else {
        asm volatile(
            "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
            "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {"
            "%0,%1,%2,%3,%4,%5,%6,%7,"
            "%8,%9,%10,%11,%12,%13,%14,%15,"
            "%16,%17,%18,%19,%20,%21,%22,%23,"
            "%24,%25,%26,%27,%28,%29,%30,%31"
            "}, %32, %33, p, 1, 1, %35, %36;\n}\n"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
              "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
              "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
            : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(TA), "n"(TB));
    }
}
// D[64 x 128] (+)= A[64 x 16] * B[16 x 128], both operands from shared-memory descriptors; TA / TB = 1: that operand
// is MN-major. accumulate == 0 overwrites D.
template <typename T, int TA, int TB>
__device__ __forceinline__ void wgmma_n128(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    if constexpr (std::is_same<T, bf16>::value) {
        asm volatile(
            "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
            "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {"
            "%0,%1,%2,%3,%4,%5,%6,%7,"
            "%8,%9,%10,%11,%12,%13,%14,%15,"
            "%16,%17,%18,%19,%20,%21,%22,%23,"
            "%24,%25,%26,%27,%28,%29,%30,%31,"
            "%32,%33,%34,%35,%36,%37,%38,%39,"
            "%40,%41,%42,%43,%44,%45,%46,%47,"
            "%48,%49,%50,%51,%52,%53,%54,%55,"
            "%56,%57,%58,%59,%60,%61,%62,%63"
            "}, %64, %65, p, 1, 1, %67, %68;\n}\n"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
              "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
              "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
              "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
              "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
              "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
              "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
            : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(TA), "n"(TB));
    }
    else {
        asm volatile(
            "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
            "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {"
            "%0,%1,%2,%3,%4,%5,%6,%7,"
            "%8,%9,%10,%11,%12,%13,%14,%15,"
            "%16,%17,%18,%19,%20,%21,%22,%23,"
            "%24,%25,%26,%27,%28,%29,%30,%31,"
            "%32,%33,%34,%35,%36,%37,%38,%39,"
            "%40,%41,%42,%43,%44,%45,%46,%47,"
            "%48,%49,%50,%51,%52,%53,%54,%55,"
            "%56,%57,%58,%59,%60,%61,%62,%63"
            "}, %64, %65, p, 1, 1, %67, %68;\n}\n"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
              "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
              "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
              "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
              "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
              "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
              "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
            : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(TA), "n"(TB));
    }
}

// D[64 x 32] (+)= A[64 x 16] * B[16 x 32]: the narrow tiles of the DenseNet 3x3 convolutions (growth 32 / 48)
template <typename T, int TA, int TB>
__device__ __forceinline__ void wgmma_n32(float (&d)[16], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    if constexpr (std::is_same<T, bf16>::value) {
        asm volatile(
            "{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
            "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {"
            "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15"
            "}, %16, %17, p, 1, 1, %19, %20;\n}\n"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
            : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(TA), "n"(TB));
    }
    else {
        asm volatile(
            "{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
            "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {"
            "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15"
            "}, %16, %17, p, 1, 1, %19, %20;\n}\n"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
            : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(TA), "n"(TB));
    }
}
// D[64 x 48] (+)= A[64 x 16] * B[16 x 48]: the narrow tiles of the DenseNet 3x3 convolutions (growth 32 / 48)
template <typename T, int TA, int TB>
__device__ __forceinline__ void wgmma_n48(float (&d)[24], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    if constexpr (std::is_same<T, bf16>::value) {
        asm volatile(
            "{\n.reg .pred p;\nsetp.ne.b32 p, %26, 0;\n"
            "wgmma.mma_async.sync.aligned.m64n48k16.f32.bf16.bf16 {"
            "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23"
            "}, %24, %25, p, 1, 1, %27, %28;\n}\n"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
            : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(TA), "n"(TB));
    }
    else {
        asm volatile(
            "{\n.reg .pred p;\nsetp.ne.b32 p, %26, 0;\n"
            "wgmma.mma_async.sync.aligned.m64n48k16.f32.f16.f16 {"
            "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23"
            "}, %24, %25, p, 1, 1, %27, %28;\n}\n"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
            : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(TA), "n"(TB));
    }
}

template <typename T, int BN, int TA, int TB>
__device__ __forceinline__ void wgmma_tile(float (&d)[BN / 2], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    if constexpr (BN == 32) wgmma_n32<T, TA, TB>(d, adesc, bdesc, accumulate);
    else if constexpr (BN == 48) wgmma_n48<T, TA, TB>(d, adesc, bdesc, accumulate);
    else if constexpr (BN == 64) wgmma_n64<T, TA, TB>(d, adesc, bdesc, accumulate);
    else wgmma_n128<T, TA, TB>(d, adesc, bdesc, accumulate);
}

// Shared-memory matrix descriptor (sm_90 GMMA): start>>4 [0,14), LBO>>4 [16,30), SBO>>4 [32,46), layout [62,64) (1 = 128B
// swizzle). K-major operand: rows of 128 B, 8-row groups 1024 B apart (SBO), LBO unused. MN-major operand: 64 contiguous
// MN elements per K row, 8-row groups along K 1024 B apart (SBO), 64-element MN blocks `lbo_bytes` apart (LBO).
__device__ __forceinline__ uint64_t make_sw128_desc(uint32_t saddr, uint32_t lbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr & 0x3FFFF) >> 4);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
    d |= (uint64_t)(1024 >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}

__device__ __forceinline__ void epi_barrier() { asm volatile("bar.sync 1, %0;" ::"n"(EPI_THREADS) : "memory"); }

struct BlockDiagDesc {
    const void* src;
    void* dst;
    int N, K, pack, _pad;
};

struct TcParams {
    int M, N, K;
    int block_n;          // multiple of 16, <= MAX_BLOCK_N
    int num_m_tiles, num_n_tiles, num_k_blocks;
    int stages;
    int is_bf16;
    double* dsum;         // optional [DFD_STAT_SLOTS][N]
    double* dsq;
    int stat_n;           // statistics channel of output column c is c % stat_n (== N unless rows are packed)
    const BnFinDesc* fin; // optional: the last CTA finalises the BatchNorm behind this convolution (bn_finalize.cuh)
    // ---- implicit-GEMM convolution mode (conv != 0): k x k, stride 1, "same" padding, NHWC ------------------------------
    // The A operand is never materialised: an M tile is a (TW x TH x TN) patch of output pixels, and for every tap (kh, kw) and
    // 64-channel block the producer issues ONE 4-D TMA load of the input box shifted by the tap - rows outside the image
    // arrive as zeros (TMA out-of-bounds fill), which IS the padding. K runs over (tap, channel block); B is the packed weight
    // [Cout][kh][kw][Cin]. The C tile goes back through a 4-D map over the output tensor (the store clips at the borders).
    int conv;
    int cv_TW, cv_TH, cv_TN;          // output patch of one M tile (cv_rows = TW * TH * TN <= 128 rows are real)
    int cv_rows;
    int cv_tiles_x, cv_tiles_y;       // patches per image row / column; M tile index = (n_tile * tiles_y + ty) * tiles_x + tx
    int cv_W, cv_H, cv_N;             // output (= input) extent
    int cv_k, cv_pad, cv_cpb;         // kernel size, padding, 64-channel blocks per tap
    int cv_S;                         // convolution stride (1 or 2): the A box starts at S * patch origin + tap - pad
    // explicit tap list (cv_ntaps > 0; the parity classes of a strided input gradient): tap t reads the A box at patch origin +
    // (cv_tox[t], cv_toy[t]) against weight k-blocks (cv_tk[t] * cv_cpb + cb)
    int cv_ntaps;
    int cv_tox[9], cv_toy[9], cv_tk[9];
    int cv_accum;                     // conv mode: the output tile is ADDED to the destination (TMA reduction store)
    int dbg;              // debug switches (DFD_DBG env): 1 = skip TMA store, 2 = skip stats pass, 8 = A from L2
};

// BN = the MMA's N (32, 48, 64 or 128): the B tile holds block_n <= BN real rows; the MMA also reads the rows above them,
// whose products land in accumulator columns that are never stored.
// KTAP (convolution mode only; 0 = 64-channel k-blocks): a k-block is ONE tap of a KTAP-channel input (32 or 48). The A box
// is still 64 channels wide - TMA fills the channels past KTAP with zeros - but only KTAP / 16 MMAs are issued per k-block,
// and the B box starts at column tap * KTAP of the [rows][taps * KTAP] packed weight (its columns past KTAP are not read).
template <typename T, int BN, int KTAP = 0>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
               const __grid_constant__ CUtensorMap tmap_c, const TcParams p) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    // SWIZZLE_128B tiles must sit on 1024-byte boundaries of the shared address space
    uint8_t* smem = smem_raw + ((1024u - (smem_addr(smem_raw) & 1023u)) & 1023u);
    // carve-up (all tile bases 1024-byte aligned): [A stages][B stages][2 C slabs][barriers][statistics scratch]
    constexpr uint32_t a_bytes = BLOCK_M * BLOCK_K * 2;
    constexpr uint32_t b_stride = BN * BLOCK_K * 2;
    const uint32_t b_bytes = (uint32_t)p.block_n * BLOCK_K * 2;      // bytes TMA delivers per B tile
    uint8_t* smem_a = smem;
    uint8_t* smem_b = smem_a + (size_t)p.stages * a_bytes;
    uint8_t* smem_c = smem_b + (size_t)p.stages * b_stride;
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem_c + 2 * BLOCK_M * SLAB * 2);
    uint64_t* full_bar = bars;
    uint64_t* empty_bar = bars + 8;
    float* red = reinterpret_cast<float*>(bars + 16);    // [sum / sq][4 row quarters][64 columns]

    const int lane = threadIdx.x & 31;
    // warpgroup index made visibly warp-uniform: the compiler can then keep the wgmma sequences of the MMA warpgroups unserialised
    const int wgi = __shfl_sync(0xffffffffu, (int)threadIdx.x / 128, 0);
    const int num_tiles = p.num_m_tiles * p.num_n_tiles;

    if (threadIdx.x == 0) {
        prefetch_tmap(&tmap_a);
        prefetch_tmap(&tmap_b);
        prefetch_tmap(&tmap_c);
        for (int i = 0; i < p.stages; i++) { mbar_init(full_bar + i, 1); mbar_init(empty_bar + i, 2); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (wgi == 0) {
        // ================= TMA producer =================
        if (threadIdx.x == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
                const int m_idx = tile / p.num_n_tiles, n_idx = tile - m_idx * p.num_n_tiles;
                int cx0 = 0, cy0 = 0, cn0 = 0;
                if (p.conv) {
                    const int txi = m_idx % p.cv_tiles_x, r = m_idx / p.cv_tiles_x;
                    cx0 = txi * p.cv_TW; cy0 = (r % p.cv_tiles_y) * p.cv_TH; cn0 = (r / p.cv_tiles_y) * p.cv_TN;
                }
                for (int kb = 0; kb < p.num_k_blocks; kb++) {
                    mbar_wait(empty_bar + stage, phase ^ 1);
                    int bk = kb * BLOCK_K;
                    if (p.conv) {
                        const int tap = kb / p.cv_cpb, cb = kb - tap * p.cv_cpb;
                        if constexpr (KTAP != 0) bk = tap * KTAP;
                        int ax, ay;
                        if (p.cv_ntaps) {
                            ax = cx0 + p.cv_tox[tap]; ay = cy0 + p.cv_toy[tap];
                            bk = (p.cv_tk[tap] * p.cv_cpb + cb) * BLOCK_K;
                        } else {
                            const int kh = tap / p.cv_k, kw = tap - kh * p.cv_k;
                            ax = cx0 * p.cv_S + kw - p.cv_pad; ay = cy0 * p.cv_S + kh - p.cv_pad;
                        }
                        mbar_arrive_expect_tx(full_bar + stage, (uint32_t)p.cv_rows * 128u + b_bytes);
                        tma_load_4d(smem_a + (size_t)stage * a_bytes, &tmap_a, full_bar + stage, cb * BLOCK_K, ax, ay, cn0);
                    } else {
                        mbar_arrive_expect_tx(full_bar + stage, a_bytes + b_bytes);
                        tma_load_2d(smem_a + (size_t)stage * a_bytes, &tmap_a, full_bar + stage, kb * BLOCK_K, (p.dbg & 8) ? 0 : m_idx * BLOCK_M);
                    }
                    tma_load_2d(smem_b + (size_t)stage * b_stride, &tmap_b, full_bar + stage, bk, n_idx * p.block_n);
                    if (++stage == p.stages) { stage = 0; phase ^= 1; }
                }
            }
        }
    } else {
        // ================= MMA + epilogue: warpgroup wg owns rows 64 * wg .. 64 * wg + 63 of every tile =================
        const int et = threadIdx.x - (NUM_THREADS - EPI_THREADS);      // 0..255
        const int wg = wgi - 1;
        const int r0 = wg * 64 + ((et >> 5) & 3) * 16 + (lane >> 2);    // this thread's accumulator rows: r0 and r0 + 8
        const int cq = (lane & 3) * 2;                                  // and columns 8 j + cq, 8 j + cq + 1
        const bool leader = et == 0;
        int stage = 0;
        uint32_t phase = 0;
        uint32_t slab_count = 0;
        const int nslabs = (p.block_n + SLAB - 1) / SLAB;
        const bool keep = p.num_n_tiles == 1;          // column identity is fixed -> keep sums in registers
        float ks[2] = {0.f, 0.f}, kq[2] = {0.f, 0.f};
        float acc[BN / 2];
#pragma unroll
        for (int i = 0; i < BN / 2; i++) acc[i] = 0.f;
        for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
            const int m_idx = tile / p.num_n_tiles, n_idx = tile - m_idx * p.num_n_tiles;
            // convolution mode: row r of the tile is output pixel (n0 + tn, y0 + ty, x0 + tx) of the patch; rows beyond the patch
            // or the image hold garbage accumulators and are zeroed (they would otherwise enter the BatchNorm statistics)
            int cx0 = 0, cy0 = 0, cn0 = 0;
            bool ok0 = true, ok1 = true;
            if (p.conv) {
                const int txi = m_idx % p.cv_tiles_x, r = m_idx / p.cv_tiles_x;
                cx0 = txi * p.cv_TW; cy0 = (r % p.cv_tiles_y) * p.cv_TH; cn0 = (r / p.cv_tiles_y) * p.cv_TN;
                auto row_ok = [&](int row) {
                    const int px = row % p.cv_TW, q2 = row / p.cv_TW;
                    const int py = q2 % p.cv_TH, pn = q2 / p.cv_TH;
                    return row < p.cv_rows && cx0 + px < p.cv_W && cy0 + py < p.cv_H && cn0 + pn < p.cv_N;
                };
                ok0 = row_ok(r0); ok1 = row_ok(r0 + 8);
            }
            // one k-block's MMAs stay in flight while the next block's are issued; a stage goes back to the producer once the
            // MMAs that read it have completed (the wait for all but the newest group)
            int prev_stage = -1;
            for (int kb = 0; kb < p.num_k_blocks; kb++) {
                mbar_wait(full_bar + stage, phase);
                const uint32_t a_addr = smem_addr(smem_a + (size_t)stage * a_bytes) + wg * 64 * 128;
                const uint32_t b_addr = smem_addr(smem_b + (size_t)stage * b_stride);
                const int krem = p.K - kb * BLOCK_K;
                const int nk = KTAP != 0 ? KTAP / MMA_K : krem >= BLOCK_K ? BLOCK_K / MMA_K : (krem + MMA_K - 1) / MMA_K;
                fence_acc(acc);
                wgmma_fence();
                for (int k = 0; k < nk; k++)
                    wgmma_tile<T, BN, 0, 0>(acc, make_sw128_desc(a_addr + k * MMA_K * 2, 16),
                                            make_sw128_desc(b_addr + k * MMA_K * 2, 16), (kb | k) != 0 ? 1u : 0u);
                wgmma_commit();
                wgmma_wait<1>();
                fence_acc(acc);
                if (prev_stage >= 0 && (et & 127) == 0) mbar_arrive(empty_bar + prev_stage);   // this warpgroup is done with it
                prev_stage = stage;
                if (++stage == p.stages) { stage = 0; phase ^= 1; }
            }
            wgmma_wait_all();
            fence_acc(acc);
            if ((et & 127) == 0) mbar_arrive(empty_bar + prev_stage);
#pragma unroll
            for (int s = 0; s < (BN + SLAB - 1) / SLAB; s++) {
                if (s >= nslabs) break;
                uint8_t* cbuf = smem_c + (size_t)(slab_count & 1) * (BLOCK_M * SLAB * 2);
                const int ncols = min(SLAB, p.block_n - s * SLAB);
                if (leader) tma_store_wait_read<1>();       // the store that last used this buffer has drained
                epi_barrier();
#pragma unroll
                for (int j = 0; j < SLAB / 8; j++) {
                    if (s * SLAB + j * 8 < BN && j * 8 < ncols) {
                        const int i = (s * (SLAB / 8) + j) * 4;
                        // logical 16-byte chunk j of a 128-byte row sits at chunk j ^ (row & 7) (r0 and r0 + 8 share row & 7)
                        const uint32_t off = ((j ^ (r0 & 7)) << 4) + cq * 2;
                        *reinterpret_cast<uint32_t*>(cbuf + r0 * 128 + off) = ok0 ? pack2<T>(acc[i], acc[i + 1]) : 0u;
                        *reinterpret_cast<uint32_t*>(cbuf + (r0 + 8) * 128 + off) = ok1 ? pack2<T>(acc[i + 2], acc[i + 3]) : 0u;
                    }
                }
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                epi_barrier();
                if (leader && !(p.dbg & 1)) {
                    if (p.conv && p.cv_accum) tma_reduce_add_4d(&tmap_c, cbuf, n_idx * p.block_n + s * SLAB, cx0, cy0, cn0);
                    else if (p.conv) tma_store_4d(&tmap_c, cbuf, n_idx * p.block_n + s * SLAB, cx0, cy0, cn0);
                    else tma_store_2d(&tmap_c, cbuf, n_idx * p.block_n + s * SLAB, m_idx * BLOCK_M);
                    tma_store_commit();
                }
                if (p.dsum && !(p.dbg & 2)) {
                    // column statistics of the stored (rounded) slab; rows past M are exact zeros
                    const int c = et & 63, qd = et >> 6;
                    float sum = 0.f, sq = 0.f;
                    if (c < ncols) {
                        const uint8_t* colp = cbuf + (c & 7) * 2;
                        const int jc = c >> 3;
                        float s1 = 0.f, q1 = 0.f;            // two chains: the adds are latency-, not throughput-bound
#pragma unroll 8
                        for (int r = qd * 32; r < qd * 32 + 32; r += 2) {
                            float x0 = to_f<T>(*reinterpret_cast<const T*>(colp + r * 128 + ((jc ^ (r & 7)) << 4)));
                            float x1 = to_f<T>(*reinterpret_cast<const T*>(colp + (r + 1) * 128 + ((jc ^ ((r + 1) & 7)) << 4)));
                            sum += x0; s1 += x1;
                            sq = fmaf(x0, x0, sq); q1 = fmaf(x1, x1, q1);
                        }
                        sum += s1; sq += q1;
                    }
                    red[qd * 64 + c] = sum;
                    red[256 + qd * 64 + c] = sq;
                    epi_barrier();
                    if (et < 64) {
                        float ts = (red[et] + red[64 + et]) + (red[128 + et] + red[192 + et]);
                        float tq = (red[256 + et] + red[320 + et]) + (red[384 + et] + red[448 + et]);
                        if (keep) { ks[s] += ts; kq[s] += tq; }
                        else {
                            int gc = n_idx * p.block_n + s * SLAB + et;
                            if (et < ncols && gc < p.N) {
                                atomicAdd(stat_slot(p.dsum, p.stat_n) + gc % p.stat_n, (double)ts);
                                atomicAdd(stat_slot(p.dsq, p.stat_n) + gc % p.stat_n, (double)tq);
                            }
                        }
                    }
                }
                slab_count++;
            }
        }
        if (p.dsum && keep && et < 64) {
#pragma unroll
            for (int s = 0; s < MAX_BLOCK_N / SLAB; s++) {
                int gc = s * SLAB + et;
                if (s < nslabs && gc < p.N && gc < p.block_n) {
                    atomicAdd(stat_slot(p.dsum, p.stat_n) + gc % p.stat_n, (double)ks[s]);
                    atomicAdd(stat_slot(p.dsq, p.stat_n) + gc % p.stat_n, (double)kq[s]);
                }
            }
        }
        if (leader) tma_store_wait_read<0>();
    }

    __syncthreads();
    bn_finalize_tail(p.fin, threadIdx.x, NUM_THREADS);
}

// =============================================================================================
// 1x1 conv weight gradient on wgmma: dW[Nw,Kw] (fp32, accumulated) += G[M,Nw]^T * X[M,Kw].
// The contraction runs over the NHWC rows, so BOTH operands are MN-major for the MMA: a TMA box of {64 channels, 64 rows}
// with 128-byte swizzle is already the canonical MN-major SW128 layout (64 contiguous MN elements per K row, 8-row
// groups 1024 B apart = SBO; 64-channel column blocks one box apart = LBO), so the tiles go from NHWC memory to the tensor
// core without any transpose. One CTA = one (128 x block_n) tile of dW and one contiguous range of 64-row blocks (split-K);
// warpgroup w accumulates rows 64 w .. 64 w + 63 of the tile in registers for the whole range and flushes them once.
// Thread 0 also issues the TMA loads, `stages` row blocks ahead of the MMAs.
// =============================================================================================
constexpr int WG_KP = 64;                      // rows (pixels) per pipeline stage
constexpr int WG_BOX_BYTES = WG_KP * 128;      // one {64 ch, 64 rows} box
constexpr int WG_THREADS = 256;

struct WgParams {
    long long M;
    int Nw, Kw;
    int block_n;            // dW columns per tile: multiple of 16, <= 128
    long long kblocks;      // ceil(M / 64)
    long long kb_per_split;
    int stages;
    int is_bf16;
    // order-deterministic mode (part != NULL): split z stores its fp32 partial tile at part[z][Nw][Kw] with plain stores and
    // dW is left alone; dfd_ordered_reduce adds the partials in split order later. part == NULL: red.global.add from every
    // split straight into dW (the order of the fp32 additions then varies run to run).
    float* part;
    int splits;
    // ---- implicit-GEMM convolution mode (conv != 0): G = dY [N,H,W,Cout] and X = the layer input [N,H,W,Cin] through 4-D
    // tensor maps; one pipeline stage = one patch of cv_rows <= 64 output pixels (TW x TH x TN); column block j of dW
    // (64 wide) = (tap = j / cpb, channel block = j % cpb): its X box is the patch shifted by the tap, padding and rows past
    // the image arrive as zeros. Rows cv_rows..63 of every box are never written by TMA and are zeroed once at kernel start.
    int conv;
    int cv_TW, cv_TH, cv_TN, cv_rows;
    int cv_tiles_x, cv_tiles_y;
    int cv_k, cv_pad, cv_cpb, cv_S;
};

// BN = the MMA's N (64 or 128) = 64 x the number of X boxes per stage
template <typename T, int BN>
__global__ void __launch_bounds__(WG_THREADS, 2)
wgrad_tc_kernel(const __grid_constant__ CUtensorMap tmap_g, const __grid_constant__ CUtensorMap tmap_x,
                float* __restrict__ dW, const WgParams p) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_addr(smem_raw) & 1023u)) & 1023u);
    constexpr int nbox_b = BN / 64;
    constexpr uint32_t a_bytes = 2 * WG_BOX_BYTES, b_bytes = nbox_b * WG_BOX_BYTES;
    uint8_t* smem_a = smem;
    uint8_t* smem_b = smem_a + (size_t)p.stages * a_bytes;
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem_b + (size_t)p.stages * b_bytes);
    uint64_t* full_bar = bars;
    uint64_t* empty_bar = bars + 8;

    const int lane = threadIdx.x & 31;
    const int m0 = blockIdx.x * 128, n0 = blockIdx.y * p.block_n;
    const long long kb0 = (long long)blockIdx.z * p.kb_per_split;
    long long kb1 = kb0 + p.kb_per_split;
    if (kb1 > p.kblocks) kb1 = p.kblocks;
    if (kb0 >= kb1) return;                                   // uniform per CTA
    const bool a_box1 = m0 + 64 < p.Nw;                       // second 64-channel block of the tile exists
    const bool b_box1 = nbox_b == 2 && n0 + 64 < p.Kw;

    if (p.conv && p.cv_rows < WG_KP) {
        uint4* z = reinterpret_cast<uint4*>(smem_a);
        const int n16 = (int)((size_t)p.stages * (a_bytes + b_bytes) / 16);
        for (int i = threadIdx.x; i < n16; i += blockDim.x) z[i] = make_uint4(0u, 0u, 0u, 0u);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    if (threadIdx.x == 0) {
        prefetch_tmap(&tmap_g);
        prefetch_tmap(&tmap_x);
        for (int i = 0; i < p.stages; i++) { mbar_init(full_bar + i, 1); mbar_init(empty_bar + i, 2); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    // loads of row block kb into `stage` (thread 0 only)
    auto issue = [&](long long kb, int stage) {
        const uint32_t box_bytes = p.conv ? (uint32_t)p.cv_rows * 128u : (uint32_t)WG_BOX_BYTES;
        mbar_arrive_expect_tx(full_bar + stage, ((a_box1 ? 2u : 1u) + (b_box1 ? 2u : 1u)) * box_bytes);
        uint8_t* a = smem_a + (size_t)stage * a_bytes;
        uint8_t* b = smem_b + (size_t)stage * b_bytes;
        if (p.conv) {
            const int pt = (int)kb, txi = pt % p.cv_tiles_x, r = pt / p.cv_tiles_x;
            const int cx0 = txi * p.cv_TW, cy0 = (r % p.cv_tiles_y) * p.cv_TH, cn0 = (r / p.cv_tiles_y) * p.cv_TN;
            tma_load_4d(a, &tmap_g, full_bar + stage, m0, cx0, cy0, cn0);
            if (a_box1) tma_load_4d(a + WG_BOX_BYTES, &tmap_g, full_bar + stage, m0 + 64, cx0, cy0, cn0);
            // (tap, channel block) of this tile's one or two 64-column blocks
            for (int i = 0; i < (b_box1 ? 2 : 1); i++) {
                const int jb = n0 / 64 + i, tap = jb / p.cv_cpb;
                tma_load_4d(b + i * WG_BOX_BYTES, &tmap_x, full_bar + stage, (jb - tap * p.cv_cpb) * 64,
                            cx0 * p.cv_S + tap % p.cv_k - p.cv_pad, cy0 * p.cv_S + tap / p.cv_k - p.cv_pad, cn0);
            }
            return;
        }
        const int row = (int)(kb * WG_KP);
        tma_load_2d(a, &tmap_g, full_bar + stage, m0, row);
        if (a_box1) tma_load_2d(a + WG_BOX_BYTES, &tmap_g, full_bar + stage, m0 + 64, row);
        tma_load_2d(b, &tmap_x, full_bar + stage, n0, row);
        if (b_box1) tma_load_2d(b + WG_BOX_BYTES, &tmap_x, full_bar + stage, n0 + 64, row);
    };

    const long long nkb = kb1 - kb0;
    if (threadIdx.x == 0)
        for (int s = 0; s < p.stages && s < nkb; s++) issue(kb0 + s, s);

    const int wg = threadIdx.x >> 7;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; i++) acc[i] = 0.f;
    int stage = 0;
    uint32_t phase = 0;
    for (long long i = 0; i < nkb; i++) {
        mbar_wait(full_bar + stage, phase);
        const uint32_t a_addr = smem_addr(smem_a + (size_t)stage * a_bytes + wg * WG_BOX_BYTES);
        const uint32_t b_addr = smem_addr(smem_b + (size_t)stage * b_bytes);
        fence_acc(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < WG_KP / MMA_K; k++)      // 16 rows of K = two 8-row groups = 2048 bytes further into every box
            wgmma_tile<T, BN, 1, 1>(acc, make_sw128_desc(a_addr + k * (MMA_K * 128), WG_BOX_BYTES),
                                    make_sw128_desc(b_addr + k * (MMA_K * 128), WG_BOX_BYTES), (i > 0 || k > 0) ? 1u : 0u);
        wgmma_commit();
        wgmma_wait_all();
        fence_acc(acc);
        if ((threadIdx.x & 127) == 0) mbar_arrive(empty_bar + stage);
        if (threadIdx.x == 0 && i + p.stages < nkb) {
            mbar_wait(empty_bar + stage, phase);            // both warpgroups have read the stage: refill it
            issue(kb0 + i + p.stages, stage);
        }
        __syncwarp();
        if (++stage == p.stages) { stage = 0; phase ^= 1; }
    }

    // Accumulator (row r, columns 8 j + 2 q, +1) and (row r + 8, same columns), q = lane & 3. Neighbouring lanes swap one pair
    // so that each holds four consecutive columns of one row: 16-byte stores / reductions (the small-M layers are bound by
    // the NUMBER of L2 reduction ops, not by their bytes). Kw % 8 == 0 keeps every group of 4 columns aligned and all-or-nothing.
    const int q = lane & 3;
    const bool odd = q & 1;
    const int row = m0 + wg * 64 + ((threadIdx.x >> 5) & 3) * 16 + (lane >> 2) + (odd ? 8 : 0);
    const int cb = 2 * (q & 2);
    float* base = p.part ? p.part + (size_t)blockIdx.z * p.Nw * p.Kw : dW;
#pragma unroll
    for (int j = 0; j < BN / 8; j++) {
        const float s0 = odd ? acc[4 * j] : acc[4 * j + 2], s1 = odd ? acc[4 * j + 1] : acc[4 * j + 3];
        const float o0 = __shfl_xor_sync(0xffffffffu, s0, 1), o1 = __shfl_xor_sync(0xffffffffu, s1, 1);
        const float4 v = odd ? make_float4(o0, o1, acc[4 * j + 2], acc[4 * j + 3]) : make_float4(acc[4 * j], acc[4 * j + 1], o0, o1);
        const int col = n0 + 8 * j + cb;
        if (8 * j < p.block_n && row < p.Nw && col < p.Kw) {
            float* dst = base + (size_t)row * p.Kw + col;
            if (p.part) *reinterpret_cast<float4*>(dst) = v;     // deterministic path: summed later in split order
            else
                asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
                             : "memory");
        }
    }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
    }
    return fn;
}

// 2-D row-major [rows, cols] 16-bit tensor, box = [box_rows, 64 cols], 128-byte swizzle, OOB -> zeros / clipped
static int make_map(CUtensorMap* m, const void* base, long long rows, int cols, int box_rows, int is_bf16) {
    EncodeTiledFn fn = get_encode_fn();
    if (!fn) return dfd_set_error(DFD_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
    cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)cols * 2};
    cuuint32_t box[2] = {(cuuint32_t)BLOCK_K, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(m, is_bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2,
                    const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        char buf[160];
        snprintf(buf, sizeof(buf), "cuTensorMapEncodeTiled failed (%d) rows=%lld cols=%d box_rows=%d", (int)r, rows, cols, box_rows);
        return dfd_set_error(DFD_ERR_CUDA, buf);
    }
    return DFD_OK;
}


// 4-D NHWC tensor [N, H, W, C] (16-bit) seen as dims {C, W, H, N}; box = {64 channels, bw, bh, bn}, 128-byte swizzle, OOB -> zeros
struct PixelView { long long sW, sH, sN; };      // byte strides between pixels / rows / images (a parity class of a tensor)
static int make_map_nhwc(CUtensorMap* m, const void* base, int N, int H, int W, int C, int bw, int bh, int bn, int is_bf16,
                         int es = 1, const PixelView* pv = nullptr) {
    EncodeTiledFn fn = get_encode_fn();
    if (!fn) return dfd_set_error(DFD_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
    cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
    cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
    if (pv) { strides[0] = (cuuint64_t)pv->sW; strides[1] = (cuuint64_t)pv->sH; strides[2] = (cuuint64_t)pv->sN; }
    // es = traversal stride in W and H (strided convolution): a box of (b - 1) * es + 1 tensor elements delivers b of them
    cuuint32_t box[4] = {(cuuint32_t)BLOCK_K, (cuuint32_t)((bw - 1) * es + 1), (cuuint32_t)((bh - 1) * es + 1), (cuuint32_t)bn};
    cuuint32_t estr[4] = {1, (cuuint32_t)es, (cuuint32_t)es, 1};
    CUresult r = fn(m, is_bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4,
                    const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        char buf[200];
        snprintf(buf, sizeof(buf), "cuTensorMapEncodeTiled (4-D) failed (%d) N=%d H=%d W=%d C=%d box=%dx%dx%d", (int)r, N, H, W, C, bw, bh, bn);
        return dfd_set_error(DFD_ERR_CUDA, buf);
    }
    return DFD_OK;
}

template <typename T, int BN, int KTAP = 0>
static void launch_tc_kernel(int grid, size_t smem, cudaStream_t st, const CUtensorMap& ma, const CUtensorMap& mb,
                             const CUtensorMap& mc, const TcParams& p) {
    static bool attr = false;
    if (!attr) { cudaFuncSetAttribute(gemm_tc_kernel<T, BN, KTAP>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BUDGET); attr = true; }
    gemm_tc_kernel<T, BN, KTAP><<<grid, NUM_THREADS, smem, st>>>(ma, mb, mc, p);
}

template <typename T, int BN>
static void launch_wgrad_kernel(dim3 grid, size_t smem, cudaStream_t st, const CUtensorMap& mg, const CUtensorMap& mx, float* dW,
                                const WgParams& p) {
    static bool attr = false;
    if (!attr) { cudaFuncSetAttribute(wgrad_tc_kernel<T, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024); attr = true; }
    wgrad_tc_kernel<T, BN><<<grid, WG_THREADS, smem, st>>>(mg, mx, dW, p);
}

// pipeline depth, shared memory and grid of gemm_tc_kernel for the tile shape in p, then the launch. narrow = the MMA N
// follows block_n down to 32 / 48 (the DenseNet entry points; the others keep 64-wide MMAs at block_n <= 64); ktap: see
// gemm_tc_kernel
static int run_tc(TcParams& p, const CUtensorMap& ma, const CUtensorMap& mb, const CUtensorMap& mc, void* stream, const char* what,
                  bool narrow = false, int ktap = 0) {
    const int bn = narrow && p.block_n <= 32 ? 32 : narrow && p.block_n <= 48 ? 48 : p.block_n <= 64 ? 64 : 128;
    p.dbg = 0;
    { const char* e = getenv("DFD_DBG"); if (e) p.dbg = atoi(e); }
    const int stage_bytes = BLOCK_M * BLOCK_K * 2 + bn * BLOCK_K * 2;
    const int fixed = 2 * BLOCK_M * SLAB * 2 + 16 * 8 + 2 * 4 * 64 * 4 + 1024 /* alignment slack */;
    int stages = (SMEM_BUDGET - fixed) / stage_bytes;
    if (stages > 6) stages = 6;
    if (stages < 2) return dfd_set_error(DFD_ERR_UNSUPPORTED, what);
    p.stages = stages;
    const size_t smem = (size_t)stages * stage_bytes + fixed;
    int device = 0, sms = DFD_SMS;
    cudaGetDevice(&device);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
    int grid = p.num_m_tiles * p.num_n_tiles;
    if (grid > sms) grid = sms;
    cudaStream_t st = (cudaStream_t)stream;
    if (ktap == 32 && bn == 128) {
        if (p.is_bf16) launch_tc_kernel<bf16, 128, 32>(grid, smem, st, ma, mb, mc, p);
        else launch_tc_kernel<__half, 128, 32>(grid, smem, st, ma, mb, mc, p);
    } else if (ktap == 48 && bn == 128) {
        if (p.is_bf16) launch_tc_kernel<bf16, 128, 48>(grid, smem, st, ma, mb, mc, p);
        else launch_tc_kernel<__half, 128, 48>(grid, smem, st, ma, mb, mc, p);
    } else if (ktap) {
        return dfd_set_error(DFD_ERR_UNSUPPORTED, what);
    } else if (p.is_bf16) {
        if (bn == 32) launch_tc_kernel<bf16, 32>(grid, smem, st, ma, mb, mc, p);
        else if (bn == 48) launch_tc_kernel<bf16, 48>(grid, smem, st, ma, mb, mc, p);
        else if (bn == 64) launch_tc_kernel<bf16, 64>(grid, smem, st, ma, mb, mc, p);
        else launch_tc_kernel<bf16, 128>(grid, smem, st, ma, mb, mc, p);
    } else {
        if (bn == 32) launch_tc_kernel<__half, 32>(grid, smem, st, ma, mb, mc, p);
        else if (bn == 48) launch_tc_kernel<__half, 48>(grid, smem, st, ma, mb, mc, p);
        else if (bn == 64) launch_tc_kernel<__half, 64>(grid, smem, st, ma, mb, mc, p);
        else launch_tc_kernel<__half, 128>(grid, smem, st, ma, mb, mc, p);
    }
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

// Implicit-GEMM convolution on the kernel above (conv mode): y[N,H,W,Cout] = conv_{k x k, stride 1, pad (k-1)/2}(x[N,H,W,Cin]),
// wpk = packed weight [Cout][kh][kw][Cin] (K-major rows of k*k*Cin). Cin % 64 == 0 keeps every 64-channel K block inside one tap.
struct ConvTaps { int n, ox[9], oy[9], kidx[9]; };
static int launch_conv_tc(const void* x, const void* wpk, void* y, int N, int Hin, int Win, int Cin, int Cout, int k, int S,
                          int dt, double* dsum, double* dsq, const void* fin, void* stream, const ConvTaps* taps = nullptr,
                          int outH = 0, int outW = 0, const PixelView* out_view = nullptr, int wcols = 0, int accum = 0,
                          int ktap = 0, int ldy = 0, int stat_ld = 0) {
    TcParams p;
    p.fin = (const BnFinDesc*)fin;
    p.conv = 1;
    p.cv_S = S;
    p.cv_accum = accum;
    p.cv_ntaps = taps ? taps->n : 0;
    if (taps) for (int t = 0; t < taps->n; t++) { p.cv_tox[t] = taps->ox[t]; p.cv_toy[t] = taps->oy[t]; p.cv_tk[t] = taps->kidx[t]; }
    // output extents (explicit tap list: the caller's output grid, e.g. one parity class of the input-gradient tensor)
    const int H = taps ? outH : (Hin + 2 * ((k - 1) / 2) - k) / S + 1, W = taps ? outW : (Win + 2 * ((k - 1) / 2) - k) / S + 1;
    // output patch of an M tile: whole rows when they fit (W <= 128), as many rows as 128 / W allows, split evenly over the
    // image height; images stacked when a whole image is smaller than half a tile (7 x 7 -> two images per tile)
    int TW = W <= 128 ? W : 128;
    int maxTH = 128 / TW; if (maxTH < 1) maxTH = 1;
    int ty = (H + maxTH - 1) / maxTH;
    int TH = (H + ty - 1) / ty;
    int TN = TH == H && TW == W ? 128 / (TW * TH) : 1;
    if (TN < 1) TN = 1;
    if (TN > N) TN = N;
    p.cv_TW = TW; p.cv_TH = TH; p.cv_TN = TN; p.cv_rows = TW * TH * TN;
    p.cv_tiles_x = (W + TW - 1) / TW; p.cv_tiles_y = (H + TH - 1) / TH;
    p.cv_W = W; p.cv_H = H; p.cv_N = N;
    p.cv_k = k; p.cv_pad = (k - 1) / 2; p.cv_cpb = ktap ? 1 : Cin / BLOCK_K;
    const int K = taps ? wcols : k * k * Cin;          // columns of the packed weight matrix
    p.M = N * H * W; p.N = Cout; p.K = K;
    p.stat_n = stat_ld ? stat_ld : Cout;
    p.is_bf16 = dt == DFD_DT_BF16;
    p.block_n = Cout <= MAX_BLOCK_N ? ((Cout + 15) / 16) * 16 : MAX_BLOCK_N;
    p.num_m_tiles = p.cv_tiles_x * p.cv_tiles_y * ((N + TN - 1) / TN);
    p.num_n_tiles = cdiv(Cout, p.block_n);
    p.num_k_blocks = (taps ? taps->n : k * k) * p.cv_cpb;
    p.dsum = dsum; p.dsq = dsq;
    CUtensorMap ma, mb, mc;
    int rc;
    if ((rc = make_map_nhwc(&ma, x, N, Hin, Win, Cin, TW, TH, TN, p.is_bf16, S))) return rc;
    if ((rc = make_map(&mb, wpk, Cout, K, p.block_n, p.is_bf16))) return rc;
    // ldy: the output is the channel slice [0, Cout) of a tensor with ldy channels per pixel (the store clips at Cout)
    PixelView slice = {(long long)ldy * 2, (long long)W * ldy * 2, (long long)H * W * ldy * 2};
    if ((rc = make_map_nhwc(&mc, y, N, H, W, Cout, TW, TH, TN, p.is_bf16, 1, ldy ? &slice : out_view))) return rc;
    return run_tc(p, ma, mb, mc, stream, "dfd_conv_tc: smem", ldy != 0 || ktap != 0, ktap);
}

// C[M,N] = A[M,K] * B[N,K]^T; statistics of output column c go to channel c % stat_n
static int launch_gemm_tc(const void* A, const void* B, void* C, long long M, int N, int K, int dt, double* dsum,
                          double* dsq, int stat_n, const void* fin, void* stream) {
    TcParams p;
    p.fin = (const BnFinDesc*)fin;
    p.conv = 0;
    p.M = (int)M; p.N = N; p.K = K;
    p.stat_n = stat_n;
    p.is_bf16 = dt == DFD_DT_BF16;
    p.block_n = N <= MAX_BLOCK_N ? ((N + 15) / 16) * 16 : MAX_BLOCK_N;
    p.num_m_tiles = cdiv(M, BLOCK_M);
    p.num_n_tiles = cdiv(N, p.block_n);
    p.num_k_blocks = cdiv(K, BLOCK_K);
    p.dsum = dsum; p.dsq = dsq;
    CUtensorMap ma, mb, mc;
    int rc;
    if ((rc = make_map(&ma, A, M, K, BLOCK_M, p.is_bf16))) return rc;
    if ((rc = make_map(&mb, B, N, K, p.block_n, p.is_bf16))) return rc;
    if ((rc = make_map(&mc, C, M, N, BLOCK_M, p.is_bf16))) return rc;
    return run_tc(p, ma, mb, mc, stream, "dfd_gemm_tn: smem");
}

#define DISPATCH_16(dt, ...)                                          \
    if ((dt) == DFD_DT_FP16) { typedef __half T16; __VA_ARGS__; }     \
    else { typedef bf16 T16; __VA_ARGS__; }

template <typename T>
__global__ void blockdiag_kernel(const BlockDiagDesc* __restrict__ table) {
    const BlockDiagDesc d = table[blockIdx.y];
    const T* src = (const T*)d.src;
    T* dst = (T*)d.dst;
    const int Kp = d.K * d.pack;
    const long long total = (long long)d.N * d.pack * Kp;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int col = (int)(i % Kp), row = (int)(i / Kp);
        const int j = row / d.N, n = row - j * d.N, jj = col / d.K, k = col - jj * d.K;
        dst[i] = j == jj ? src[(size_t)n * d.K + k] : from_f<T>(0.f);
    }
}

}  // namespace

extern "C" {

// C[M,N] = A[M,K] * B[N,K]^T on wgmma; optional fp64 column statistics of the stored C ([8][N] slots).
// All pointers must be 16-byte aligned, K % 8 == 0 and N % 8 == 0 (TMA global strides are multiples of 16 B).
int dfd_gemm_tn(const void* A, const void* B, void* C, long long M, int N, int K, int dt, double* dsum, double* dsq,
                const void* fin, void* stream) {
    if (M <= 0 || N <= 0 || K <= 0 || (N % 8) || (K % 8)) return dfd_set_error(DFD_ERR_ARG, "dfd_gemm_tn: N%8, K%8");
    if (dt != DFD_DT_BF16 && dt != DFD_DT_FP16) return dfd_set_error(DFD_ERR_ARG, "dfd_gemm_tn: dtype");
    return launch_gemm_tc(A, B, C, M, N, K, dt, dsum, dsq, N, fin, stream);
}

// The same product for SMALL K (a pointwise conv with 16 / 24 / 32 input channels): `pack` consecutive rows of A are
// read as ONE row of pack*K values and multiplied by the block-diagonal weight Bd[pack*N, pack*K] (dfd_blockdiag_weights),
// which yields `pack` consecutive rows of C side by side - byte for byte the row-major C[M,N]. TMA fetches a tile row
// per request, so 32-byte rows (K = 16) leave the load path request-bound at a quarter of the HBM rate; the packed view
// issues 128-byte rows. The extra MMA work multiplies zeros and is free at these K.
int dfd_gemm_tn_rowpack(const void* A, const void* Bd, void* C, long long M, int N, int K, int pack, int dt,
                        double* dsum, double* dsq, const void* fin, void* stream) {
    if (M <= 0 || N <= 0 || K <= 0 || (N % 8) || (K % 8)) return dfd_set_error(DFD_ERR_ARG, "dfd_gemm_tn_rowpack: N%8, K%8");
    if (dt != DFD_DT_BF16 && dt != DFD_DT_FP16) return dfd_set_error(DFD_ERR_ARG, "dfd_gemm_tn_rowpack: dtype");
    if (pack < 1 || pack > 8 || (M % pack)) return dfd_set_error(DFD_ERR_ARG, "dfd_gemm_tn_rowpack: M % pack");
    return launch_gemm_tc(A, Bd, C, M / pack, N * pack, K * pack, dt, dsum, dsq, N, fin, stream);
}

// Dense k x k convolution (stride 1, padding (k-1)/2) as an IMPLICIT GEMM on wgmma: no im2col matrix exists in memory - the
// TMA producer fetches, per tap and 64-channel block, the input box shifted by the tap through a 4-D tensor map over the NHWC
// tensor (out-of-bounds rows arrive as zeros = the padding) straight into the swizzled MMA operand buffer.
//   forward : x = input,  wpk = [Cout][kh][kw][Cin]                      (resnet.py:129-136,195-197: nn.Conv2d 3x3)
//   dgrad   : x = dY,     wpk = [Cin][kh'][kw'][Cout] with flipped taps   (autograd input gradient of the same conv)
int dfd_conv_tc(const void* x, const void* wpk, void* y, int N, int H, int W, int Cin, int Cout, int k, int stride, int dt,
                double* dsum, double* dsq, const void* fin, void* stream) {
    if (N <= 0 || H <= 0 || W <= 0 || Cin <= 0 || Cout <= 0 || (Cin % 64) || (Cout % 64) || (k != 1 && k != 3 && k != 5 && k != 7) ||
        (stride != 1 && stride != 2))
        return dfd_set_error(DFD_ERR_ARG, "dfd_conv_tc: Cin % 64, Cout % 64, k in {1,3,5,7}, stride in {1,2}");
    if (dt != DFD_DT_BF16 && dt != DFD_DT_FP16) return dfd_set_error(DFD_ERR_ARG, "dfd_conv_tc: dtype");
    return launch_conv_tc(x, wpk, y, N, H, W, Cin, Cout, k, stride, dt, dsum, dsq, fin, stream);
}

// DenseNet's 3x3 convolution (densenet.py:44-45: bn_size * k -> k channels, stride 1, padding 1) for growth k = Cout in
// {32, 48}: the implicit GEMM above with 32- / 48-wide MMAs, whose output is the channel slice at y of a tensor with ldy
// channels per pixel (the dense block's concatenated buffer). The store goes through a tensor map over that slice alone,
// so no channel outside it is ever written. dsum / dsq: [DFD_STAT_SLOTS][stat_ld] statistics, offset to the slice's first
// channel (NULL: none).
int dfd_conv3x3_narrow_tc(const void* x, const void* wpk, void* y, int N, int H, int W, int Cin, int Cout, int ldy, int dt,
                          double* dsum, double* dsq, int stat_ld, void* stream) {
    if (N <= 0 || H <= 0 || W <= 0 || Cin <= 0 || (Cin % 64) || (Cout != 32 && Cout != 48) || ldy < Cout || (ldy % 8) ||
        ((uintptr_t)y & 15) || (dsum && stat_ld < Cout))
        return dfd_set_error(DFD_ERR_ARG, "dfd_conv3x3_narrow_tc: Cin % 64, Cout in {32, 48}, ldy % 8 >= Cout, y 16-byte aligned");
    if (dt != DFD_DT_BF16 && dt != DFD_DT_FP16) return dfd_set_error(DFD_ERR_ARG, "dfd_conv3x3_narrow_tc: dtype");
    return launch_conv_tc(x, wpk, y, N, H, W, Cin, Cout, 3, 1, dt, dsum, dsq, nullptr, stream, nullptr, 0, 0, nullptr, 0, 0, 0,
                          ldy, stat_ld ? stat_ld : Cout);
}

// Input gradient of dfd_conv3x3_narrow_tc: dx[N,H,W,Cin] = conv3x3(dy[N,H,W,Cout], tap-flipped wpkD [Cin][kh'][kw'][Cout]),
// dy contiguous with Cout in {32, 48} channels. Each k-block is one tap of Cout channels (KTAP): no padding of K, so no MMA
// multiplies a padded zero.
int dfd_conv3x3_narrow_dgrad_tc(const void* dy, const void* wpkD, void* dx, int N, int H, int W, int Cin, int Cout, int dt,
                                void* stream) {
    if (N <= 0 || H <= 0 || W <= 0 || Cin < 128 || (Cin % 64) || (Cout != 32 && Cout != 48))
        return dfd_set_error(DFD_ERR_ARG, "dfd_conv3x3_narrow_dgrad_tc: Cin % 64 >= 128, Cout in {32, 48}");
    if (dt != DFD_DT_BF16 && dt != DFD_DT_FP16) return dfd_set_error(DFD_ERR_ARG, "dfd_conv3x3_narrow_dgrad_tc: dtype");
    return launch_conv_tc(dy, wpkD, dx, N, H, W, Cout, Cin, 3, 1, dt, nullptr, nullptr, nullptr, stream, nullptr, 0, 0, nullptr, 0,
                          0, Cout);
}

// Input gradient of a 3x3, stride-2, padding-1 convolution as FOUR implicit GEMMs, one per parity class (py, px) of the input
// pixels: dx[2a+py][2b+px] = sum over the taps whose parity matches of dY[a + oy][b + ox] * W[kh][kw] - 1, 2, 2 and 4 taps.
// Each class is a stride-1 implicit GEMM over dY (out-of-range rows / columns arrive as TMA zeros) whose output tensor map is
// a strided VIEW of dx (every other pixel of every other row, offset by the parity): every dx element is written exactly once,
// no 9 x Cin column matrix and no col2im scatter. wpkD = the tap-flipped [Cin][kh'][kw'][Cout] layout of dfd_repack_weights.
int dfd_conv_dgrad_s2_tc(const void* dy, const void* wpkD, void* dx, int N, int H, int W, int Cin, int Cout, int dt, void* stream) {
    if (N <= 0 || H <= 0 || W <= 0 || Cin <= 0 || Cout <= 0 || (Cin % 64) || (Cout % 64))
        return dfd_set_error(DFD_ERR_ARG, "dfd_conv_dgrad_s2_tc: Cin % 64, Cout % 64");
    if (dt != DFD_DT_BF16 && dt != DFD_DT_FP16) return dfd_set_error(DFD_ERR_ARG, "dfd_conv_dgrad_s2_tc: dtype");
    const int Ho = (H + 2 - 3) / 2 + 1, Wo = (W + 2 - 3) / 2 + 1;
    for (int py = 0; py < 2; py++) {
        for (int px = 0; px < 2; px++) {
            const int Ha = (H - py + 1) / 2, Wb = (W - px + 1) / 2;
            if (Ha <= 0 || Wb <= 0) continue;
            ConvTaps t;
            t.n = 0;
            for (int kh = 0; kh < 3; kh++) {
                if (((py + 1 - kh) & 1) != 0) continue;                 // iy + 1 - kh must be even
                for (int kw = 0; kw < 3; kw++) {
                    if (((px + 1 - kw) & 1) != 0) continue;
                    t.oy[t.n] = (py + 1 - kh) / 2;                      // dY row = a + (py + 1 - kh) / 2
                    t.ox[t.n] = (px + 1 - kw) / 2;
                    t.kidx[t.n] = 8 - (kh * 3 + kw);                    // position of tap (kh, kw) in the flipped layout
                    t.n++;
                }
            }
            PixelView pv = {2LL * Cin * 2, 2LL * W * Cin * 2, (long long)H * W * Cin * 2};
            void* base = (char*)dx + ((size_t)py * W + px) * Cin * 2;
            // GEMM: M = N * Ha * Wb pixels of the class, K = taps x Cout (A = dY), N = Cin
            int rc = launch_conv_tc(dy, wpkD, base, N, Ho, Wo, Cout, Cin, 3, 1, dt, nullptr, nullptr, nullptr, stream, &t, Ha, Wb, &pv,
                                    9 * Cout);
            if (rc) return rc;
        }
    }
    return DFD_OK;
}

// Input gradient of a 1x1 convolution with stride s (the downsample branch, resnet.py:249-260) ADDED into dx, which already
// holds the main-path gradient of the block input: dx[n, s*a, s*b, :] += dY[n, a, b, :] * W. One implicit GEMM (k = 1) whose
// output map is the stride-s pixel view of dx and whose epilogue is a TMA reduction store (bf16 / fp16 add in L2) - replaces
// GEMM -> scratch, then col2im scatter + add (stride 2) or add_inplace (stride 1). wT = the transposed [Cin][Cout] weight.
int dfd_conv1x1_dgrad_add(const void* dy, const void* wT, void* dx, int N, int H, int W, int Cin, int Cout, int stride, int dt,
                          void* stream) {
    if (N <= 0 || H <= 0 || W <= 0 || Cin <= 0 || Cout <= 0 || (Cin % 64) || (Cout % 64) || (stride != 1 && stride != 2))
        return dfd_set_error(DFD_ERR_ARG, "dfd_conv1x1_dgrad_add: Cin % 64, Cout % 64, stride in {1,2}");
    if (dt != DFD_DT_BF16 && dt != DFD_DT_FP16) return dfd_set_error(DFD_ERR_ARG, "dfd_conv1x1_dgrad_add: dtype");
    const int Ho = (H - 1) / stride + 1, Wo = (W - 1) / stride + 1;
    ConvTaps t;
    t.n = 1; t.ox[0] = 0; t.oy[0] = 0; t.kidx[0] = 0;
    PixelView pv = {(long long)stride * Cin * 2, (long long)stride * W * Cin * 2, (long long)H * W * Cin * 2};
    return launch_conv_tc(dy, wT, dx, N, Ho, Wo, Cout, Cin, 1, 1, dt, nullptr, nullptr, nullptr, stream, &t, Ho, Wo, &pv, Cout, 1);
}

// table: device array of {src [N,K], dst [pack*N, pack*K], N, K, pack}; dst(j*N+n, j'*K+k) = (j == j') ? src(n,k) : 0
int dfd_blockdiag_weights(const void* table, int count, int dt, void* stream) {
    if (count <= 0) return DFD_OK;
    dim3 grid(16, count);
    DISPATCH_16(dt, (blockdiag_kernel<T16><<<grid, 256, 0, (cudaStream_t)stream>>>((const BlockDiagDesc*)table)));
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

// dW[Nw,Kw] (fp32, accumulated) += G[M,Nw]^T * X[M,Kw] on wgmma (MN-major operands straight from NHWC, split over M)
// split count of the workspace (order-deterministic) mode: as many row ranges as fill the GPU once, but no more than keep
// the partial-sum traffic (one write + one read of splits x Nw x Kw floats) under half of the operand traffic
static long long wgrad_ws_splits(long long M, int Nw, int Kw, int sms, long long kblocks = 0) {
    const int block_n = Kw >= 128 ? 128 : ((Kw + 15) / 16) * 16;
    if (!kblocks) kblocks = (M + WG_KP - 1) / WG_KP;
    const int tm = cdiv(Nw, 128), tn = cdiv(Kw, block_n);
    long long splits = (2LL * sms + tm * tn - 1) / (tm * tn);
    const long long max_splits = (kblocks + 3) / 4;
    if (splits > max_splits) splits = max_splits;
    const long long cap = (2 * M * ((long long)Nw + Kw)) / (2LL * 2 * 4 * Nw * Kw);
    if (splits > cap) splits = cap;
    if (splits < 1) splits = 1;
    const long long kb_per = (kblocks + splits - 1) / splits;
    return (kblocks + kb_per - 1) / kb_per;
}

// number of partial matrices [Nw, Kw] dfd_gemm_wgrad writes into its workspace for this shape (workspace bytes = that x Nw x Kw x 4)
int dfd_gemm_wgrad_splits(long long M, int Nw, int Kw) {
    if (M <= 0 || Nw <= 0 || Kw <= 0) return 0;
    return (int)wgrad_ws_splits(M, Nw, Kw, DFD_SMS);
}

// patch (TW x TH x TN <= 64 output pixels) of one pipeline stage of the implicit-GEMM weight gradient: the shape that covers
// the N x H x W pixels with the fewest patches (ties: the widest, longest contiguous runs for TMA)
struct WgPatch { int TW, TH, TN; long long patches; };
static WgPatch wg_patch(int N, int H, int W) {
    WgPatch best = {1, 1, 1, -1};
    for (int tw = 1; tw <= W && tw <= WG_KP; tw++) {
        for (int th = 1; th <= H && tw * th <= WG_KP; th++) {
            int tn = (tw == W && th == H) ? WG_KP / (tw * th) : 1;
            if (tn > N) tn = N;
            long long n = (long long)cdiv(W, tw) * cdiv(H, th) * cdiv(N, tn);
            if (best.patches < 0 || n < best.patches || (n == best.patches && tw > best.TW)) best = {tw, th, tn, n};
        }
    }
    return best;
}

static int launch_wgrad_tc(const void* G, const void* X, float* dW, long long M, int Nw, int Kw, int dt, void* ws,
                           long long ws_bytes, void* stream, int cvN, int cvH, int cvW, int cvCin, int cvk, int cvS = 1);

int dfd_gemm_wgrad(const void* G, const void* X, float* dW, long long M, int Nw, int Kw, int dt, void* ws, long long ws_bytes,
                   void* stream) {
    if (M <= 0 || Nw <= 0 || Kw <= 0 || (Nw % 8) || (Kw % 8)) return dfd_set_error(DFD_ERR_ARG, "dfd_gemm_wgrad: Nw%8, Kw%8");
    if (dt != DFD_DT_BF16 && dt != DFD_DT_FP16) return dfd_set_error(DFD_ERR_ARG, "dfd_gemm_wgrad: dtype");
    return launch_wgrad_tc(G, X, dW, M, Nw, Kw, dt, ws, ws_bytes, stream, 0, 0, 0, 0, 0);
}

// Weight gradient of a dense k x k convolution (stride 1, padding (k-1)/2) as an IMPLICIT GEMM: dW[Cout][kh][kw][Cin] (fp32,
// the packed order of dfd_repack_weights; accumulated, or written as split partials into `ws` like dfd_gemm_wgrad) =
// sum over output pixels of dY[pixel, co] * x[pixel shifted by the tap, ci]; no im2col matrix in memory.
static inline int conv_out_extent(int h, int k, int s) { return (h + 2 * ((k - 1) / 2) - k) / s + 1; }
int dfd_conv_wgrad_splits(int N, int H, int W, int Cin, int Cout, int k, int stride) {
    if (N <= 0 || H <= 0 || W <= 0 || Cin <= 0 || Cout <= 0 || stride <= 0) return 0;
    const int Ho = conv_out_extent(H, k, stride), Wo = conv_out_extent(W, k, stride);
    WgPatch pt = wg_patch(N, Ho, Wo);
    return (int)wgrad_ws_splits((long long)N * Ho * Wo, Cout, k * k * Cin, DFD_SMS, pt.patches);
}

int dfd_conv_wgrad_tc(const void* dy, const void* x, float* dW, int N, int H, int W, int Cin, int Cout, int k, int stride, int dt,
                      void* ws, long long ws_bytes, void* stream) {
    if (N <= 0 || H <= 0 || W <= 0 || Cin <= 0 || Cout <= 0 || (Cin % 64) || (Cout % 8) || (k != 1 && k != 3 && k != 5 && k != 7) ||
        (stride != 1 && stride != 2))
        return dfd_set_error(DFD_ERR_ARG, "dfd_conv_wgrad_tc: Cin % 64, Cout % 8, k in {1,3,5,7}, stride in {1,2}");
    if (dt != DFD_DT_BF16 && dt != DFD_DT_FP16) return dfd_set_error(DFD_ERR_ARG, "dfd_conv_wgrad_tc: dtype");
    const int Ho = conv_out_extent(H, k, stride), Wo = conv_out_extent(W, k, stride);
    return launch_wgrad_tc(dy, x, dW, (long long)N * Ho * Wo, Cout, k * k * Cin, dt, ws, ws_bytes, stream, N, H, W, Cin, k, stride);
}

static int launch_wgrad_tc(const void* G, const void* X, float* dW, long long M, int Nw, int Kw, int dt, void* ws,
                           long long ws_bytes, void* stream, int cvN, int cvH, int cvW, int cvCin, int cvk, int cvS) {
    WgParams p;
    // cvH / cvW: INPUT extents of the convolution; the patches tile the OUTPUT pixels
    const int cvHo = cvN > 0 ? conv_out_extent(cvH, cvk, cvS) : 0, cvWo = cvN > 0 ? conv_out_extent(cvW, cvk, cvS) : 0;
    p.M = M; p.Nw = Nw; p.Kw = Kw;
    p.is_bf16 = dt == DFD_DT_BF16;
    p.block_n = Kw >= 128 ? 128 : ((Kw + 15) / 16) * 16;
    p.kblocks = (M + WG_KP - 1) / WG_KP;
    p.conv = cvN > 0;
    if (p.conv) {
        WgPatch pt = wg_patch(cvN, cvHo, cvWo);
        p.cv_TW = pt.TW; p.cv_TH = pt.TH; p.cv_TN = pt.TN; p.cv_rows = pt.TW * pt.TH * pt.TN;
        p.cv_tiles_x = cdiv(cvWo, pt.TW); p.cv_tiles_y = cdiv(cvHo, pt.TH);
        p.cv_k = cvk; p.cv_pad = (cvk - 1) / 2; p.cv_cpb = cvCin / 64; p.cv_S = cvS;
        p.kblocks = pt.patches;
    }
    const int tm = cdiv(Nw, 128), tn = cdiv(Kw, p.block_n);
    int device = 0, sms = DFD_SMS;
    cudaGetDevice(&device);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
    long long splits = (2LL * sms + tm * tn - 1) / (tm * tn);
    long long max_splits = (p.kblocks + 3) / 4;              // at least 4 row blocks per CTA
    if (splits > max_splits) splits = max_splits;
    if (splits < 1) splits = 1;
    if (splits > 65535) splits = 65535;
    p.part = nullptr;
    if (ws) {
        splits = wgrad_ws_splits(M, Nw, Kw, DFD_SMS, p.conv ? p.kblocks : 0);
        if (splits * (long long)Nw * Kw * 4 > ws_bytes)
            return dfd_set_error(DFD_ERR_ARG, "dfd_gemm_wgrad: workspace too small (dfd_gemm_wgrad_splits x Nw x Kw floats)");
        p.part = (float*)ws;
    }
    p.kb_per_split = (p.kblocks + splits - 1) / splits;
    splits = (p.kblocks + p.kb_per_split - 1) / p.kb_per_split;
    const int nbox_b = p.block_n > 64 ? 2 : 1;
    const int stage_bytes = (2 + nbox_b) * WG_BOX_BYTES;
    const int fixed = 16 * 8 + 1024;
    // ~100 KB per CTA: two CTAs share an SM, so 2 x SMs splits run as one wave
    int stages = (100 * 1024 - fixed) / stage_bytes;
    if (stages > 6) stages = 6;
    if (stages < 2) stages = 2;
    p.stages = stages;
    size_t smem = (size_t)stages * stage_bytes + fixed;
    CUtensorMap mg, mx;
    int rc;
    if (p.conv) {
        if ((rc = make_map_nhwc(&mg, G, cvN, cvHo, cvWo, Nw, p.cv_TW, p.cv_TH, p.cv_TN, p.is_bf16))) return rc;
        if ((rc = make_map_nhwc(&mx, X, cvN, cvH, cvW, cvCin, p.cv_TW, p.cv_TH, p.cv_TN, p.is_bf16, cvS))) return rc;
    } else {
        if ((rc = make_map(&mg, G, M, Nw, WG_KP, p.is_bf16))) return rc;
        if ((rc = make_map(&mx, X, M, Kw, WG_KP, p.is_bf16))) return rc;
    }
    dim3 grid(tm, tn, (unsigned)splits);
    cudaStream_t st = (cudaStream_t)stream;
    if (p.is_bf16) {
        if (nbox_b == 1) launch_wgrad_kernel<bf16, 64>(grid, smem, st, mg, mx, dW, p);
        else launch_wgrad_kernel<bf16, 128>(grid, smem, st, mg, mx, dW, p);
    } else {
        if (nbox_b == 1) launch_wgrad_kernel<__half, 64>(grid, smem, st, mg, mx, dW, p);
        else launch_wgrad_kernel<__half, 128>(grid, smem, st, mg, mx, dW, p);
    }
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

}  // extern "C"
