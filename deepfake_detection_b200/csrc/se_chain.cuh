// The per-image squeeze-excite FC chains as device functions, so that the CTA which completes an image's pooling (forward)
// or its gate-gradient reduction (backward) carries straight on with the FCs instead of a separate one-CTA-per-image launch:
// the chains are latency-bound (a few thousand dependent cycles on a few hundred KB of L2-resident weights) and hide in the
// tail of the streaming kernel that feeds them.   Reference: SqueezeExcite.forward, efficientnet_blocks.py:104-110.
// All threads of the CTA must call these (they contain __syncthreads); `tid` / `nt` are the linear thread id / CTA size.
#pragma once
#include "common.cuh"

__device__ __forceinline__ float se_swish_precise(float x) { return x * sigmoid_precise(x); }

// inner activation of the chain: DFD_ACT_SWISH (EfficientNet's SqueezeExcite) or DFD_ACT_RELU (SENet's SEModule,
// senet.py:67-86); its derivative in terms of the pre-activation x
template <int INNER> __device__ __forceinline__ float se_inner(float x) {
    return INNER == DFD_ACT_RELU ? fmaxf(x, 0.f) : se_swish_precise(x);
}
template <int INNER> __device__ __forceinline__ float se_inner_grad(float x) {
    if (INNER == DFD_ACT_RELU) return x > 0.f ? 1.f : 0.f;
    const float sg = sigmoid_precise(x);
    return sg * (1.f + x * (1.f - sg));
}

// p: [C] pooled activations of this image in SHARED memory; r: [Cse] shared scratch.
// gate[c] = sigmoid(be[c] + sum_j We[c,j] * inner(br[j] + sum_c' Wr[j,c'] p[c'])), inner = swish or ReLU
template <int INNER = DFD_ACT_SWISH>
__device__ __forceinline__ void se_fwd_chain(const float* p, float* r, const float* __restrict__ Wr,
                                             const float* __restrict__ br, const float* __restrict__ We,
                                             const float* __restrict__ be, float* __restrict__ gate_out, int C, int Cse,
                                             int tid, int nt) {
    const int warp = tid >> 5, lane = tid & 31, nw = nt >> 5;       // nw FULL warps cooperate (a ragged last warp sits out)
    if (warp < nw)
        for (int j = warp; j < Cse; j += nw) {
            const float* w = Wr + (size_t)j * C;
            float s = 0.f;
            for (int c = lane; c < C; c += 32) s = fmaf(w[c], p[c], s);
            s = warp_sum(s);
            if (lane == 0) r[j] = se_inner<INNER>(s + br[j]);
        }
    __syncthreads();
    // one thread per output row: a row is Cse consecutive floats, so the warp's 32 rows stay L1-resident across the j loop
    for (int c = tid; c < C; c += nt) {
        const float* w = We + (size_t)c * Cse;
        float s = be[c];
        for (int j = 0; j < Cse; j++) s = fmaf(w[j], r[j], s);
        gate_out[c] = sigmoid_precise(s);
    }
}

// shared scratch `sm`: p [C] (in), de [C], rpre / r / drp [Cse] each, r_part [nw][Cse]   = 2C + (3 + nw) Cse floats.
// draw: dL/dgate of this image in SHARED or global memory (read once per channel).
// Emits d_e [C], r [Cse], d_rpre [Cse] (operands of the SE parameter gradients) and dpool [C] to global memory.
template <int INNER = DFD_ACT_SWISH>
__device__ __forceinline__ void se_bwd_chain(float* sm, const float* draw, const float* __restrict__ Wr,
                                             const float* __restrict__ br, const float* __restrict__ We,
                                             const float* __restrict__ be, float* __restrict__ d_e_out,
                                             float* __restrict__ r_out, float* __restrict__ d_rpre_out,
                                             float* __restrict__ dpool_out, int C, int Cse, int tid, int nt) {
    float* p = sm;
    float* de = sm + C;
    float* rpre = sm + 2 * C;
    float* r = rpre + Cse;
    float* drp = r + Cse;
    float* r_part = drp + Cse;
    const int warp = tid >> 5, lane = tid & 31, nw = nt >> 5;       // nw FULL warps cooperate (a ragged last warp sits out)
    if (warp < nw)
        for (int j = warp; j < Cse; j += nw) {
            const float* w = Wr + (size_t)j * C;
            float s = 0.f;
            for (int c = lane; c < C; c += 32) s = fmaf(w[c], p[c], s);
            s = warp_sum(s);
            if (lane == 0) { rpre[j] = s + br[j]; r[j] = se_inner<INNER>(s + br[j]); }
        }
    __syncthreads();
    for (int c = tid; c < C; c += nt) {
        const float* w = We + (size_t)c * Cse;
        float s = be[c];
        for (int j = 0; j < Cse; j++) s = fmaf(w[j], r[j], s);
        const float g = sigmoid_precise(s);
        const float v = draw[c] * g * (1.f - g);
        de[c] = v;
        d_e_out[c] = v;
    }
    __syncthreads();
    // d_r[j] = sum_c We[c,j] * de[c]: lanes walk j (contiguous in We's rows), warps split c; per-warp partials are summed in
    // warp order (no shared-memory atomics: the result does not depend on warp scheduling)
    if (warp < nw)
        for (int j0 = 0; j0 < Cse; j0 += 32) {
            const int j = j0 + lane;
            float s = 0.f;
            if (j < Cse) {
                for (int c = warp; c < C; c += nw) s = fmaf(We[(size_t)c * Cse + j], de[c], s);
                r_part[warp * Cse + j] = s;
            }
        }
    __syncthreads();
    for (int j = tid; j < Cse; j += nt) {
        float s = 0.f;
        for (int w = 0; w < nw; w++) s += r_part[w * Cse + j];
        const float v = s * se_inner_grad<INNER>(rpre[j]);
        drp[j] = v;
        d_rpre_out[j] = v;
        r_out[j] = r[j];
    }
    __syncthreads();
    for (int c = tid; c < C; c += nt) {
        float s = 0.f;
        for (int j = 0; j < Cse; j++) s = fmaf(Wr[(size_t)j * C + c], drp[j], s);
        dpool_out[c] = s;
    }
}
