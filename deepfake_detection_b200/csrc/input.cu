// The step's inputs that are not activations: the prefetcher's image normalisation and the stochastic-regularisation
// masks.
//
// Reference semantics restated here:
//   PrefetchLoader.__iter__       dfd/timm/data/loader.py:243-256  (uint8 NCHW batch -> float, (x - mean*255) / (std*255),
//                                 mean / std repeated per frame: img_num x RGB, dfd/params.py:24-27)
//   drop_path                     dfd/timm/models/layers/drop.py:84-100 (per-sample mask floor(keep + U[0,1)), x / keep * mask),
//                                 applied before the residual add, efficientnet_blocks.py:343-346
//   classifier dropout            F.dropout(x, p=drop_rate, training), dfd/timm/models/efficientnet.py:346-347
//
// The masks come from a counter-based generator: value(seed, step, stream, index) is a pure function, the (seed, step) pair
// lives in device memory and `dfd_rng_tick` advances the step inside the captured CUDA graph, so every replay draws fresh
// masks without any host involvement.  torch's Philox stream cannot be reproduced bit for bit (it depends on torch's
// launch geometry); parity tests therefore read the masks back and hand the SAME masks to the oracle (exact comparison)
// and check the keep rate statistically.
#include "common.cuh"

namespace {

// ---------------------------------------------------------------------------------------------
// uint8 NCHW -> 16-bit NCHW, out = (x - mean255[c]) / std255[c]  (fp32 arithmetic, IEEE division, one rounding to T)
// grid: (chunks of a plane, N*C planes); a thread converts 16 consecutive pixels (one 16-byte load, two 16-byte stores)
// ---------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256)
input_normalize_kernel(const unsigned char* __restrict__ x, const float* __restrict__ mean255,
                       const float* __restrict__ std255, T* __restrict__ out, int C, long long plane) {
    const long long pl = blockIdx.y;
    const int c = (int)(pl % C);
    const float m = mean255[c], s = std255[c];
    const unsigned char* src = x + pl * plane;
    T* dst = out + pl * plane;
    const bool vec_ok = (plane & 15) == 0 && ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(out)) & 15) == 0;
    if (vec_ok) {
        const long long nvec = plane >> 4;
        for (long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x; v < nvec; v += (long long)gridDim.x * blockDim.x) {
            const uint4 raw = __ldg(reinterpret_cast<const uint4*>(src) + v);
            const uint32_t w[4] = {raw.x, raw.y, raw.z, raw.w};
            float f[16];
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
                for (int j = 0; j < 4; j++) f[i * 4 + j] = ((float)((w[i] >> (8 * j)) & 0xffu) - m) / s;
            stg16(dst + v * 16, pack8<T>(f));
            stg16(dst + v * 16 + 8, pack8<T>(f + 8));
        }
    } else {
        for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < plane; i += (long long)gridDim.x * blockDim.x)
            dst[i] = from_f<T>(((float)src[i] - m) / s);
    }
}

// ---------------------------------------------------------------------------------------------
// counter-based uniform generator (splitmix64 finaliser over a 64-bit counter built from step / stream / index)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned long long mix64(unsigned long long z) {
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
__device__ __forceinline__ float uniform01(unsigned long long seed, unsigned long long step, unsigned stream, unsigned long long idx) {
    unsigned long long h = mix64(seed + 0x9E3779B97F4A7C15ull * (step + 1));
    h = mix64(h ^ (0xD1B54A32D192ED03ull * (stream + 1)));
    h = mix64(h ^ (idx * 0x8CB92BA72F3D8DD7ull + 0x2545F4914F6CDD1Dull));
    return (float)(h >> 40) * (1.0f / 16777216.0f);          // 24 random bits -> [0, 1)
}

struct MaskDesc {
    float* out;          // [rows, width]
    long long rows;
    int width;           // values per random draw (drop path: the channel count, one draw per sample; dropout: 1)
    float keep_prob;
    int stream;          // generator stream id (one per mask tensor)
    int _pad;
};

// out[r, :] = floor(keep + u(r)) / keep      (drop.py:95-99: random_tensor.floor_(); x.div(keep_prob) * random_tensor)
__global__ void rng_masks_kernel(const MaskDesc* __restrict__ table, const long long* __restrict__ state) {
    const MaskDesc d = table[blockIdx.y];
    const unsigned long long seed = (unsigned long long)state[0], step = (unsigned long long)state[1];
    const long long total = d.rows * d.width;
    const float inv = 1.0f / d.keep_prob;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long r = i / d.width;
        const float u = uniform01(seed, step, (unsigned)d.stream, (unsigned long long)r);
        d.out[i] = floorf(d.keep_prob + u) * inv;
    }
}

// ---------------------------------------------------------------------------------------------
// DropBlock block masks (drop_block_2d, dfd/timm/models/layers/drop.py:24-63), one site per grid row
// ---------------------------------------------------------------------------------------------
struct DropBlockDesc {
    unsigned char* mask;        // [N, H, W, C] block mask: 1 kept, 0 dropped
    float* noise;               // optional [N, H, W, C]: the uniform draws
    unsigned long long* kept;   // number of ones in mask (zeroed before the launch)
    double gamma;               // seed drop rate, as the reference computes it in double
    int N, H, W, C;
    int cb;                     // clipped block size (odd, <= DB_MAX_CB)
    int stream;                 // generator stream id of the site
    int _pad[2];
};

constexpr int DB_TILE = 16;     // output pixels per tile side
constexpr int DB_CG = 32;       // channels per tile (consecutive bytes of an NHWC pixel)
constexpr int DB_MAX_CB = 7;
constexpr int DB_HALO = DB_TILE + DB_MAX_CB - 1;

// One CTA walks tiles of [DB_TILE x DB_TILE pixels x DB_CG channels] of one image. It stages the seeds of the tile and its
// halo in shared memory (each uniform is drawn once per tile), takes the min over the cb columns, then over the cb rows
// (min of 0/1 = AND; pixels outside the map are ignored, as max_pool2d's implicit -inf padding is), and counts the ones.
// seed = (2 - gamma - valid + u) >= 1 in the reference's fp32 order; valid follows the reference's [W, H] meshgrid reshaped
// to [H, W]: pixel (h, w) reads entry f = h*W + w of the [W, H] grid, i.e. (i, j) = (f / H, f % H).
__global__ void __launch_bounds__(256) drop_block_kernel(const DropBlockDesc* __restrict__ table,
                                                         const long long* __restrict__ state) {
    __shared__ unsigned char seeds[DB_HALO][DB_HALO][DB_CG];
    __shared__ unsigned char rowmin[DB_HALO][DB_TILE][DB_CG];
    __shared__ unsigned long long warp_cnt[8];
    const DropBlockDesc d = table[blockIdx.y];
    const unsigned long long seed = (unsigned long long)state[0], step = (unsigned long long)state[1];
    const int H = d.H, W = d.W, C = d.C, cb = d.cb, r = cb / 2;
    const float a = (float)(2.0 - d.gamma);
    const int lo = cb / 2, hi_w = W - (cb - 1) / 2, hi_h = H - (cb - 1) / 2;
    const int th_n = (H + DB_TILE - 1) / DB_TILE, tw_n = (W + DB_TILE - 1) / DB_TILE, cg_n = (C + DB_CG - 1) / DB_CG;
    const long long ntiles = (long long)d.N * th_n * tw_n * cg_n;
    const int c_l = threadIdx.x % DB_CG, p_l = threadIdx.x / DB_CG, p_step = blockDim.x / DB_CG;
    unsigned long long cnt = 0;
    for (long long t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const int cg = (int)(t % cg_n);
        long long q = t / cg_n;
        const int tw = (int)(q % tw_n); q /= tw_n;
        const int th = (int)(q % th_n);
        const int n = (int)(q / th_n);
        const int h0 = th * DB_TILE, w0 = tw * DB_TILE, c = cg * DB_CG + c_l;
        const int oh_n = min(DB_TILE, H - h0), ow_n = min(DB_TILE, W - w0);
        const int hh_n = oh_n + cb - 1, ww_n = ow_n + cb - 1;
        for (int p = p_l; p < hh_n * ww_n; p += p_step) {
            const int hh = p / ww_n, ww = p - hh * ww_n;
            const int h = h0 - r + hh, w = w0 - r + ww;
            unsigned char s = 1;
            if (h >= 0 && h < H && w >= 0 && w < W && c < C) {
                const int f = h * W + w, i = f / H, j = f - (f / H) * H;
                const bool valid = i >= lo && i < hi_w && j >= lo && j < hi_h;
                // outside `valid` the seed is (a + u >= 1) with u >= 0: always kept when a >= 1, so no draw is needed there
                // (the draws do not depend on which elements are drawn: with the noise output every element is drawn)
                if (valid || a < 1.f || d.noise) {
                    const unsigned long long idx = (((unsigned long long)n * H + h) * W + w) * C + c;
                    const float u = uniform01(seed, step, (unsigned)d.stream, idx);
                    const float v = __fadd_rn(__fsub_rn(a, valid ? 1.f : 0.f), u);
                    s = v >= 1.f ? 1 : 0;
                    if (d.noise && hh >= r && hh < r + oh_n && ww >= r && ww < r + ow_n) d.noise[idx] = u;
                }
            }
            seeds[hh][ww][c_l] = s;
        }
        __syncthreads();
        for (int p = p_l; p < hh_n * ow_n; p += p_step) {
            const int hh = p / ow_n, ow = p - hh * ow_n;
            unsigned char m = 1;
            for (int k = 0; k < cb; k++) m &= seeds[hh][ow + k][c_l];
            rowmin[hh][ow][c_l] = m;
        }
        __syncthreads();
        if (c < C) {
            for (int p = p_l; p < oh_n * ow_n; p += p_step) {
                const int oh = p / ow_n, ow = p - oh * ow_n;
                unsigned char m = 1;
                for (int k = 0; k < cb; k++) m &= rowmin[oh + k][ow][c_l];
                d.mask[(((size_t)n * H + h0 + oh) * W + w0 + ow) * C + c] = m;
                cnt += m;
            }
        }
        __syncthreads();
    }
    // exact count: integer sums do not depend on the order of the CTAs
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    if ((threadIdx.x & 31) == 0) warp_cnt[threadIdx.x >> 5] = cnt;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long s = 0;
        for (int i = 0; i < (int)(blockDim.x >> 5); i++) s += warp_cnt[i];
        if (s) atomicAdd(d.kept, s);
    }
}

__global__ void rng_tick_kernel(long long* __restrict__ state) { state[1] += 1; }

__global__ void mul_f32_kernel(float* __restrict__ a, const float* __restrict__ b, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (size_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) a[i] *= b[i];
}

}  // namespace

extern "C" {

int dfd_input_normalize(const void* x_u8, const float* mean255, const float* std255, void* out, int N, int C, int H, int W,
                        int dt, void* stream) {
    if (N <= 0 || C <= 0 || H <= 0 || W <= 0 || !mean255 || !std255) return dfd_set_error(DFD_ERR_ARG, "dfd_input_normalize: sizes");
    const long long plane = (long long)H * W;
    const long long planes = (long long)N * C;
    if (planes > 65535LL * 32768) return dfd_set_error(DFD_ERR_ARG, "dfd_input_normalize: too many planes");
    int bx = (int)((plane / 16 + 255) / 256);
    if (bx < 1) bx = 1;
    if (bx > 64) bx = 64;
    // planes go on grid.y (<= 65535): fold larger batches into several launches
    for (long long p0 = 0; p0 < planes; p0 += 65535) {
        const int py = (int)((planes - p0 < 65535) ? planes - p0 : 65535);
        if (p0 % C) return dfd_set_error(DFD_ERR_UNSUPPORTED, "dfd_input_normalize: plane split");
        dim3 grid(bx, py);
        const unsigned char* src = (const unsigned char*)x_u8 + p0 * plane;
        if (dt == DFD_DT_BF16)
            input_normalize_kernel<bf16><<<grid, 256, 0, (cudaStream_t)stream>>>(src, mean255, std255, (bf16*)out + p0 * plane, C, plane);
        else if (dt == DFD_DT_FP16)
            input_normalize_kernel<__half><<<grid, 256, 0, (cudaStream_t)stream>>>(src, mean255, std255, (__half*)out + p0 * plane, C, plane);
        else
            return dfd_set_error(DFD_ERR_ARG, "dfd_input_normalize: dtype");
    }
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

// table: device array of { float* out; long long rows; int width; float keep_prob; int stream; int _pad; }
// state: device int64 [seed, step]
int dfd_rng_masks(const void* table, int count, const long long* state, void* stream) {
    if (count <= 0) return DFD_OK;
    if (!table || !state) return dfd_set_error(DFD_ERR_ARG, "dfd_rng_masks: operands");
    rng_masks_kernel<<<dim3(8, count), 256, 0, (cudaStream_t)stream>>>((const MaskDesc*)table, state);
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

// table: device array of DropBlockDesc (64 bytes each, see include/dfd_b200.h); every `kept` slot must be zero on entry
int dfd_drop_block_masks(const void* table, int count, const long long* state, void* stream) {
    if (count <= 0) return DFD_OK;
    if (!table || !state || count > 65535) return dfd_set_error(DFD_ERR_ARG, "dfd_drop_block_masks: operands");
    drop_block_kernel<<<dim3(4 * DFD_SMS, count), 256, 0, (cudaStream_t)stream>>>((const DropBlockDesc*)table, state);
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

int dfd_rng_tick(long long* state, void* stream) {
    rng_tick_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(state);
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

int dfd_mul_f32(float* a, const float* b, long long n, void* stream) {
    if (n <= 0) return DFD_OK;
    long long blocks = (n + 255) / 256;
    if (blocks > 1184) blocks = 1184;
    mul_f32_kernel<<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(a, b, (size_t)n);
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

}  // extern "C"
