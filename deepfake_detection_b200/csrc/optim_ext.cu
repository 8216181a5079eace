// The flat-arena optimizers beyond sgd / adam / adamw / rmsproptf that dfd/timm/optim/optim_factory.py:26-100 offers:
//
//   RAdam        dfd/timm/optim/radam.py:10-82          (factory :57-59; weight decay divided by the initial lr, :29-33)
//   Adadelta     torch.optim.Adadelta(rho 0.9)          (factory :63-65; _single_tensor_adadelta)
//   RMSprop      torch.optim.RMSprop(alpha 0.9)         (factory :66-69; _single_tensor_rmsprop, not centered)
//   NovoGrad     dfd/timm/optim/novograd.py:12-77       (factory :73-74; layer-wise)
//   NvNovoGrad   dfd/timm/optim/nvnovograd.py:13-117    (factory :75-76; layer-wise)
//
// Conventions are those of the optimizers in se_head_optim.cu: the gradient the update sees is g * grad_scale *
// (*gscale_dev), a non-zero *skip (fp16 overflow) makes every kernel return before it writes anything, the learning rate
// is read from lr_dev when given, the step count from step_dev (advanced by dfd_opt_tick before these launches), and p16
// receives the 16-bit copy of the updated weights.
//
// The two NovoGrads need the squared L2 norm of each parameter tensor's gradient. dfd_tensor_sumsq computes it from a
// host-built table of fixed-size chunks that never straddle a tensor: one CTA per chunk writes its partial to the chunk's
// slot, then one warp per tensor adds the slots of its chunks in a fixed order. No floating-point atomics, so two runs give
// identical bits. The squares of fp32 values are exact in fp64 and the partials are summed in fp64: the only rounding that
// reaches the fp32 result is its final conversion, so the sum is as accurate as the reference's fp32 norm can be compared
// to, and fp64 adds cost nothing here (the kernel streams 4 bytes per element).
#include "common.cuh"

namespace {

// one chunk of the layer-wise table: elements [off, off + len) of the arena, all of tensor `tensor`
struct LwChunk {
    long long off;
    int len;
    int tensor;
};
constexpr int LW_THREADS = 256;

__device__ __forceinline__ float eff_scale(float grad_scale, const float* gscale_dev) {
    return gscale_dev ? grad_scale * *gscale_dev : grad_scale;
}

template <typename T16>
__device__ __forceinline__ void put16(void* p16, size_t i, float v) {
    if (p16) reinterpret_cast<T16*>(p16)[i] = from_f<T16>(v);
}

// radam.py:47-80. N_sma and the step size depend only on the step and on the lr of the group that computes them first
// (the reference caches them per step in self.buffer, shared across groups: group 0 wins); the decoupled decay uses the
// range's own lr. The scalars are computed in double, as the reference does in Python floats.
template <typename T16>
__global__ void radam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                             float* __restrict__ v, size_t n, float lr, double b1, double b2, float eps, float wd,
                             float grad_scale, const float* __restrict__ gscale_dev, const int* __restrict__ skip,
                             void* __restrict__ p16, const float* __restrict__ lr_dev, const float* __restrict__ lr0_dev,
                             const int* __restrict__ step_dev) {
    if (skip && *skip) return;
    const float s = eff_scale(grad_scale, gscale_dev);
    if (lr_dev) lr = *lr_dev;
    const double lr0 = lr0_dev ? (double)*lr0_dev : (double)lr;
    const double t = (double)*step_dev;
    const double b2t = pow(b2, t);
    const double nmax = 2.0 / (1.0 - b2) - 1.0;
    const double nsma = nmax - 2.0 * t * b2t / (1.0 - b2t);
    const bool rect = nsma >= 5.0;
    const double ss = rect ? lr0 * sqrt((1.0 - b2t) * (nsma - 4.0) / (nmax - 4.0) * (nsma - 2.0) / nsma * nmax / (nmax - 2.0)) /
                                 (1.0 - pow(b1, t))
                           : lr0 / (1.0 - pow(b1, t));
    const float step_size = (float)ss, dec = (float)(-(double)wd * (double)lr);
    const float fb1 = (float)b1, fb2 = (float)b2, ob1 = (float)(1.0 - b1), ob2 = (float)(1.0 - b2);
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (size_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        const float gg = g[i] * s;
        const float vv = fmaf(fb2, v[i], ob2 * gg * gg);     // :51
        const float mm = fmaf(fb1, m[i], ob1 * gg);          // :52
        v[i] = vv;
        m[i] = mm;
        float w = p[i];
        if (wd != 0.f) w = fmaf(dec, w, w);                          // :73-74
        w = rect ? w - step_size * (mm / (sqrtf(vv) + eps)) : fmaf(-step_size, mm, w);   // :77-80
        p[i] = w;
        put16<T16>(p16, i, w);
    }
}

// torch.optim.Adadelta, single-tensor form: L2 decay into the gradient, std = sqrt(sq + eps),
// delta = sqrt(acc + eps) / std * g, acc updated with delta, p -= lr * delta
template <typename T16>
__global__ void adadelta_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ sq,
                                float* __restrict__ acc, size_t n, float lr, float rho, float eps, float wd, float grad_scale,
                                const float* __restrict__ gscale_dev, const int* __restrict__ skip, void* __restrict__ p16,
                                const float* __restrict__ lr_dev) {
    if (skip && *skip) return;
    const float s = eff_scale(grad_scale, gscale_dev);
    if (lr_dev) lr = *lr_dev;
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (size_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        float w = p[i];
        const float gg = fmaf(wd, w, g[i] * s);
        const float sa = fmaf(rho, sq[i], (1.f - rho) * gg * gg);
        sq[i] = sa;
        const float a = acc[i];
        const float delta = sqrtf(a + eps) / sqrtf(sa + eps) * gg;
        acc[i] = fmaf(rho, a, (1.f - rho) * delta * delta);
        w = fmaf(-lr, delta, w);
        p[i] = w;
        put16<T16>(p16, i, w);
    }
}

// torch.optim.RMSprop, single-tensor form (not centered): square_avg starts at zeros, eps outside the sqrt, the momentum
// buffer holds g / avg and the lr multiplies it at the weight update
template <typename T16>
__global__ void rmsprop_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ sq,
                               float* __restrict__ mom, size_t n, float lr, float alpha, float eps, float wd, float momentum,
                               float grad_scale, const float* __restrict__ gscale_dev, const int* __restrict__ skip,
                               void* __restrict__ p16, const float* __restrict__ lr_dev) {
    if (skip && *skip) return;
    const float s = eff_scale(grad_scale, gscale_dev);
    if (lr_dev) lr = *lr_dev;
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (size_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        float w = p[i];
        const float gg = fmaf(wd, w, g[i] * s);
        const float sa = fmaf(alpha, sq[i], (1.f - alpha) * gg * gg);
        sq[i] = sa;
        const float avg = sqrtf(sa) + eps;
        if (momentum > 0.f) {
            const float b = fmaf(momentum, mom[i], gg / avg);
            mom[i] = b;
            w = fmaf(-lr, b, w);
        } else {
            w = fmaf(-lr, gg / avg, w);
        }
        p[i] = w;
        put16<T16>(p16, i, w);
    }
}

// ---- per-tensor sum of squares ---------------------------------------------------------------------------------------------
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__global__ void __launch_bounds__(LW_THREADS) sumsq_chunks_kernel(const float* __restrict__ g, const LwChunk* __restrict__ table,
                                                                 double* __restrict__ partial, float grad_scale,
                                                                 const float* __restrict__ gscale_dev,
                                                                 const int* __restrict__ skip) {
    if (skip && *skip) return;
    __shared__ double s_w[LW_THREADS / 32];
    const float s = eff_scale(grad_scale, gscale_dev);
    const LwChunk c = table[blockIdx.x];
    const float* src = g + c.off;
    double acc = 0.0;
    for (int i = threadIdx.x; i < c.len; i += LW_THREADS) {
        const double x = (double)(src[i] * s);          // the unscaled fp32 gradient, squared exactly in fp64
        acc = fma(x, x, acc);
    }
    acc = warp_sum_d(acc);
    if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
#pragma unroll
        for (int w = 0; w < LW_THREADS / 32; w++) t += s_w[w];
        partial[blockIdx.x] = t;
    }
}

// one warp per tensor: lane l adds the partials l, l + 32, ... of the tensor's chunks, then a fixed butterfly
__global__ void sumsq_tensors_kernel(const double* __restrict__ partial, const int* __restrict__ chunk0, int n_tensors,
                                     float* __restrict__ sumsq, const int* __restrict__ skip) {
    if (skip && *skip) return;
    const int t = blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (t >= n_tensors) return;
    double acc = 0.0;
    for (int c = chunk0[t] + lane; c < chunk0[t + 1]; c += 32) acc += partial[c];
    acc = warp_sum_d(acc);
    if (lane == 0) sumsq[t] = (float)acc;
}

// ---- NovoGrad (novograd.py:29-77) --------------------------------------------------------------------------------------------
// Per-tensor part, one CTA. state[0] = initialised flag (cleared at construction, set by the first applied step), state[1] =
// "this step initialised" for the update kernels. On the step that initialises (:30-46) v = ||g||^2, grad_ema starts at
// ||g||^2 and the step count restarts at 1. Then (:58-72) grad_ema = b2 grad_ema + (1-b2) ||g||^2, ghat = g / (sqrt(grad_ema)
// + eps), v = b2 v + (1-b2) ||ghat||^2. ||ghat||^2 is taken as ||g||^2 / (sqrt(grad_ema) + eps)^2 instead of a second pass
// over the tensor: equal in exact arithmetic, within a few fp32 roundings of the reference's norm of the scaled tensor.
// coef[2t] = 1 / (||g|| + eps) (the initial m), coef[2t + 1] = 1 / ((sqrt(grad_ema) + eps) (sqrt(v) + eps)).
__global__ void novograd_prepare_kernel(const float* __restrict__ sumsq, float* __restrict__ v, float* __restrict__ grad_ema,
                                        float* __restrict__ coef, int* __restrict__ state, int* __restrict__ step_dev,
                                        int n_tensors, float b2, float eps, const int* __restrict__ skip) {
    if (skip && *skip) return;
    const bool fresh = state[0] == 0;
    for (int t = threadIdx.x; t < n_tensors; t += blockDim.x) {
        const float n2 = sumsq[t];
        float ge, vv;
        if (fresh) {
            ge = n2;
            vv = n2;
            coef[2 * t] = 1.f / (sqrtf(n2) + eps);
        } else {
            ge = fmaf(b2, grad_ema[t], (1.f - b2) * n2);
            vv = v[t];
        }
        const float r = 1.f / (sqrtf(ge) + eps);
        vv = fmaf(b2, vv, (1.f - b2) * (n2 * r * r));
        v[t] = vv;
        grad_ema[t] = ge;
        coef[2 * t + 1] = r / (sqrtf(vv) + eps);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        if (fresh) {
            state[0] = 1;
            *step_dev = 1;                 // state['step'] = 0 at initialisation, then += 1
        }
        state[1] = fresh ? 1 : 0;
    }
}

// m = b1 m + ghat / (sqrt(v) + eps) + wd p (m's initial value on the initialising step: g / (||g|| + eps) + wd p);
// p -= lr sqrt(1 - b2^t) / (1 - b1^t) m. wd is the constructor's decay (self._wd), not the group's.
template <typename T16>
__global__ void novograd_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                const LwChunk* __restrict__ table, int n_chunks, const float* __restrict__ coef,
                                const int* __restrict__ state, float lr, double b1, double b2, float wd, float grad_scale,
                                const float* __restrict__ gscale_dev, const int* __restrict__ skip, void* __restrict__ p16,
                                const float* __restrict__ lr_dev, const int* __restrict__ step_dev) {
    if (skip && *skip) return;
    const float s = eff_scale(grad_scale, gscale_dev);
    if (lr_dev) lr = *lr_dev;
    const double t = (double)*step_dev;
    const float step_size = (float)((double)lr * sqrt(1.0 - pow(b2, t)) / (1.0 - pow(b1, t)));
    const bool fresh = state[1] != 0;
    const float fb1 = (float)b1;
    for (int ci = blockIdx.x; ci < n_chunks; ci += gridDim.x) {
        const LwChunk c = table[ci];
        const float a0 = fresh ? coef[2 * c.tensor] : 0.f, a1 = coef[2 * c.tensor + 1];
        for (int j = threadIdx.x; j < c.len; j += blockDim.x) {
            const size_t i = (size_t)c.off + j;
            const float gg = g[i] * s;
            float w = p[i];
            const float dp = wd * w;
            const float mp = fresh ? fmaf(gg, a0, dp) : m[i];
            const float mm = fmaf(fb1, mp, fmaf(gg, a1, dp));
            m[i] = mm;
            w = fmaf(-step_size, mm, w);
            p[i] = w;
            put16<T16>(p16, i, w);
        }
    }
}

// ---- NvNovoGrad (nvnovograd.py:91-115) ----------------------------------------------------------------------------------------
// exp_avg_sq (per tensor) is copied from ||g||^2 while it is exactly 0 and is an EMA after that; denom = sqrt(exp_avg_sq) + eps
__global__ void nvnovograd_prepare_kernel(const float* __restrict__ sumsq, float* __restrict__ exp_avg_sq,
                                          float* __restrict__ denom, int n_tensors, float b2, float eps,
                                          const int* __restrict__ skip) {
    if (skip && *skip) return;
    for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < n_tensors; t += gridDim.x * blockDim.x) {
        const float n2 = sumsq[t];
        float e = exp_avg_sq[t];
        e = e == 0.f ? n2 : fmaf(e, b2, (1.f - b2) * n2);
        exp_avg_sq[t] = e;
        denom[t] = sqrtf(e) + eps;
    }
}

// g / denom + wd p (the group's decay), exp_avg = b1 exp_avg + that, p -= lr exp_avg (no bias correction)
template <typename T16>
__global__ void nvnovograd_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                  const LwChunk* __restrict__ table, int n_chunks, const float* __restrict__ denom, float lr,
                                  float b1, float wd, float grad_scale, const float* __restrict__ gscale_dev,
                                  const int* __restrict__ skip, void* __restrict__ p16, const float* __restrict__ lr_dev) {
    if (skip && *skip) return;
    const float s = eff_scale(grad_scale, gscale_dev);
    if (lr_dev) lr = *lr_dev;
    for (int ci = blockIdx.x; ci < n_chunks; ci += gridDim.x) {
        const LwChunk c = table[ci];
        const float d = denom[c.tensor];
        for (int j = threadIdx.x; j < c.len; j += blockDim.x) {
            const size_t i = (size_t)c.off + j;
            float w = p[i];
            const float gg = fmaf(wd, w, (g[i] * s) / d);
            const float mm = fmaf(b1, m[i], gg);
            m[i] = mm;
            w = fmaf(-lr, mm, w);
            p[i] = w;
            put16<T16>(p16, i, w);
        }
    }
}

int flat_grid(long long n) {
    long long b = (n + 255) / 256;
    if (b > DFD_SMS * 8) b = DFD_SMS * 8;
    return (int)(b < 1 ? 1 : b);
}

}  // namespace

#define DISPATCH_16(dt, ...)                                          \
    if ((dt) == DFD_DT_FP16) { typedef __half T16; __VA_ARGS__; }     \
    else { typedef bf16 T16; __VA_ARGS__; }

extern "C" {

int dfd_radam_step(float* p, const float* g, float* m, float* v, long long n, float lr, double b1, double b2, float eps,
                   float wd, float grad_scale, const float* gscale_dev, const int* skip, void* p16, int dt,
                   const float* lr_dev, const float* lr0_dev, const int* step_dev, void* stream) {
    if (n <= 0) return DFD_OK;
    if (!step_dev) return dfd_set_error(DFD_ERR_ARG, "dfd_radam_step: step_dev is required");
    DISPATCH_16(dt, (radam_kernel<T16><<<flat_grid(n), 256, 0, (cudaStream_t)stream>>>(p, g, m, v, (size_t)n, lr, b1, b2, eps, wd, grad_scale, gscale_dev, skip, p16, lr_dev, lr0_dev, step_dev)));
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

int dfd_adadelta_step(float* p, const float* g, float* sq, float* acc, long long n, float lr, float rho, float eps, float wd,
                      float grad_scale, const float* gscale_dev, const int* skip, void* p16, int dt, const float* lr_dev,
                      void* stream) {
    if (n <= 0) return DFD_OK;
    DISPATCH_16(dt, (adadelta_kernel<T16><<<flat_grid(n), 256, 0, (cudaStream_t)stream>>>(p, g, sq, acc, (size_t)n, lr, rho, eps, wd, grad_scale, gscale_dev, skip, p16, lr_dev)));
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

int dfd_rmsprop_step(float* p, const float* g, float* sq, float* mom, long long n, float lr, float alpha, float eps, float wd,
                     float momentum, float grad_scale, const float* gscale_dev, const int* skip, void* p16, int dt,
                     const float* lr_dev, void* stream) {
    if (n <= 0) return DFD_OK;
    if (momentum > 0.f && !mom) return dfd_set_error(DFD_ERR_ARG, "dfd_rmsprop_step: momentum without a buffer");
    DISPATCH_16(dt, (rmsprop_kernel<T16><<<flat_grid(n), 256, 0, (cudaStream_t)stream>>>(p, g, sq, mom, (size_t)n, lr, alpha, eps, wd, momentum, grad_scale, gscale_dev, skip, p16, lr_dev)));
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

int dfd_tensor_sumsq(const float* g, const void* table, int n_chunks, const int* chunk0, int n_tensors, double* partial,
                     float* sumsq, float grad_scale, const float* gscale_dev, const int* skip, void* stream) {
    if (n_chunks <= 0 || n_tensors <= 0) return dfd_set_error(DFD_ERR_ARG, "dfd_tensor_sumsq: empty table");
    cudaStream_t st = (cudaStream_t)stream;
    sumsq_chunks_kernel<<<n_chunks, LW_THREADS, 0, st>>>(g, (const LwChunk*)table, partial, grad_scale, gscale_dev, skip);
    DFD_LAUNCH_CHECK();
    sumsq_tensors_kernel<<<cdiv(n_tensors, 8), 256, 0, st>>>(partial, chunk0, n_tensors, sumsq, skip);
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

int dfd_novograd_prepare(const float* sumsq, float* v, float* grad_ema, float* coef, int* state, int* step_dev, int n_tensors,
                         float b2, float eps, const int* skip, void* stream) {
    if (n_tensors <= 0) return dfd_set_error(DFD_ERR_ARG, "dfd_novograd_prepare: no tensors");
    novograd_prepare_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(sumsq, v, grad_ema, coef, state, step_dev, n_tensors, b2, eps,
                                                                  skip);
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

int dfd_novograd_step(float* p, const float* g, float* m, const void* table, int n_chunks, const float* coef, const int* state,
                      float lr, double b1, double b2, float wd, float grad_scale, const float* gscale_dev, const int* skip,
                      void* p16, int dt, const float* lr_dev, const int* step_dev, void* stream) {
    if (n_chunks <= 0) return DFD_OK;
    const int grid = n_chunks < DFD_SMS * 8 ? n_chunks : DFD_SMS * 8;
    DISPATCH_16(dt, (novograd_kernel<T16><<<grid, LW_THREADS, 0, (cudaStream_t)stream>>>(p, g, m, (const LwChunk*)table, n_chunks, coef, state, lr, b1, b2, wd, grad_scale, gscale_dev, skip, p16, lr_dev, step_dev)));
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

int dfd_nvnovograd_prepare(const float* sumsq, float* exp_avg_sq, float* denom, int n_tensors, float b2, float eps,
                           const int* skip, void* stream) {
    if (n_tensors <= 0) return dfd_set_error(DFD_ERR_ARG, "dfd_nvnovograd_prepare: no tensors");
    nvnovograd_prepare_kernel<<<cdiv(n_tensors, 256), 256, 0, (cudaStream_t)stream>>>(sumsq, exp_avg_sq, denom, n_tensors, b2,
                                                                                       eps, skip);
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

int dfd_nvnovograd_step(float* p, const float* g, float* m, const void* table, int n_chunks, const float* denom, float lr,
                        float b1, float wd, float grad_scale, const float* gscale_dev, const int* skip, void* p16, int dt,
                        const float* lr_dev, void* stream) {
    if (n_chunks <= 0) return DFD_OK;
    const int grid = n_chunks < DFD_SMS * 8 ? n_chunks : DFD_SMS * 8;
    DISPATCH_16(dt, (nvnovograd_kernel<T16><<<grid, LW_THREADS, 0, (cudaStream_t)stream>>>(p, g, m, (const LwChunk*)table, n_chunks, denom, lr, b1, wd, grad_scale, gscale_dev, skip, p16, lr_dev)));
    DFD_LAUNCH_CHECK();
    return DFD_OK;
}

}  // extern "C"
