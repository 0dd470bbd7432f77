// Fused optimizer step for the training loop that drives the hot path (train.py:324-331):
//   clip_grad_norm_ (global L2 norm over every gradient)  ->  RAdam.step (radam.py:44-122).
// The reference walks the parameters in Python: per tensor two fp32 copies, ~10 elementwise launches and a copy
// back (radam.py:56-122) -- ~600 launches and ~15 passes over the 220 MB of parameters per step.  Here parameters,
// gradients and both moments live in flat fp32 buffers (flowtron_b200/radam.py), so a step is: one partial-sums
// launch per contiguous gradient segment, one tiny finalize launch (norm + clip coefficient, kept on the device: no
// host sync), one update launch per segment.  HBM-bound: reads p, g, m, v and writes p, m, v = 28 B per parameter.
#include "ptx.cuh"
#include "ft_internal.h"

namespace ft {

constexpr int SUMSQ_BLOCKS = 1024;      // partials per segment (ft_sumsq_partials writes exactly this many floats)
constexpr int OPT_THREADS = 256;

__global__ void __launch_bounds__(OPT_THREADS)
sumsq_partials_kernel(const float* __restrict__ x, long long n, float* __restrict__ partials) {
    float s = 0.f;
    const long long stride = static_cast<long long>(gridDim.x) * OPT_THREADS;
    const long long i0 = static_cast<long long>(blockIdx.x) * OPT_THREADS + threadIdx.x;
    if ((reinterpret_cast<uintptr_t>(x) & 15) == 0) {
        const long long n4 = n >> 2;
        const float4* x4 = reinterpret_cast<const float4*>(x);
        for (long long i = i0; i < n4; i += stride) {
            const float4 v = x4[i];
            s = fmaf(v.x, v.x, s); s = fmaf(v.y, v.y, s); s = fmaf(v.z, v.z, s); s = fmaf(v.w, v.w, s);
        }
        for (long long i = (n4 << 2) + i0; i < n; i += stride) s = fmaf(x[i], x[i], s);
    } else {
        for (long long i = i0; i < n; i += stride) s = fmaf(x[i], x[i], s);
    }
    __shared__ float red[OPT_THREADS / 32];
#pragma unroll
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x < 32) {
        float t = threadIdx.x < OPT_THREADS / 32 ? red[threadIdx.x] : 0.f;
#pragma unroll
        for (int o = 16; o; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
        if (threadIdx.x == 0) partials[blockIdx.x] = t;
    }
}

// out[0] = total L2 norm, out[1] = min(1, max_norm / (norm + 1e-6))   (torch.nn.utils.clip_grad_norm_)
__global__ void __launch_bounds__(OPT_THREADS)
clip_coef_kernel(const float* __restrict__ partials, int n_partials, float max_norm, float* __restrict__ out) {
    double s = 0.0;
    for (int i = threadIdx.x; i < n_partials; i += OPT_THREADS) s += static_cast<double>(partials[i]);
    __shared__ double red[OPT_THREADS / 32];
#pragma unroll
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < OPT_THREADS / 32; ++w) t += red[w];
        const float norm = static_cast<float>(sqrt(t));
        out[0] = norm;
        out[1] = fminf(1.0f, max_norm / (norm + 1e-6f));
    }
}

struct RAdamScalars { float beta1, beta2, omb1, omb2, eps, wd_lr, step_size; int use_denom; };

__device__ __forceinline__ void radam_one(float& p, float g, float& m, float& v, const RAdamScalars& a) {
    v = fmaf(a.omb2 * g, g, v * a.beta2);              // exp_avg_sq.mul_(beta2).addcmul_(1 - beta2, grad, grad)   radam.py:78
    m = fmaf(a.omb1, g, m * a.beta1);                  // exp_avg.mul_(beta1).add_(1 - beta1, grad)                :79
    if (a.wd_lr != 0.f) p = fmaf(-a.wd_lr, p, p);      // p.add_(-weight_decay * lr, p)                            :109-112
    if (a.use_denom) p = fmaf(-a.step_size, m / (sqrtf(v) + a.eps), p);     // addcdiv_(-step_size, exp_avg, denom) :115-117
    else p = fmaf(-a.step_size, m, p);                 // add_(-step_size, exp_avg)                                :119
}

__global__ void __launch_bounds__(OPT_THREADS)
radam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v, long long n,
             RAdamScalars a, const float* __restrict__ grad_coef) {
    const float gc = grad_coef ? grad_coef[0] : 1.0f;
    const long long stride = static_cast<long long>(gridDim.x) * OPT_THREADS;
    const long long i0 = static_cast<long long>(blockIdx.x) * OPT_THREADS + threadIdx.x;
    const bool al = ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(m) |
                      reinterpret_cast<uintptr_t>(v)) & 15) == 0;
    long long done = 0;
    if (al) {
        const long long n4 = n >> 2;
        float4* p4 = reinterpret_cast<float4*>(p);
        const float4* g4 = reinterpret_cast<const float4*>(g);
        float4* m4 = reinterpret_cast<float4*>(m);
        float4* v4 = reinterpret_cast<float4*>(v);
        for (long long i = i0; i < n4; i += stride) {
            float4 pp = p4[i], mm = m4[i], vv = v4[i];
            const float4 gg = g4[i];
            radam_one(pp.x, gg.x * gc, mm.x, vv.x, a);
            radam_one(pp.y, gg.y * gc, mm.y, vv.y, a);
            radam_one(pp.z, gg.z * gc, mm.z, vv.z, a);
            radam_one(pp.w, gg.w * gc, mm.w, vv.w, a);
            p4[i] = pp; m4[i] = mm; v4[i] = vv;
        }
        done = n4 << 2;
    }
    for (long long i = done + i0; i < n; i += stride) {
        float pp = p[i], mm = m[i], vv = v[i];
        radam_one(pp, g[i] * gc, mm, vv, a);
        p[i] = pp; m[i] = mm; v[i] = vv;
    }
}

// Capturable form (CUDA graphs): the step count lives on the device, so N_sma / step_size (radam.py:87-107) are evaluated by
// the kernel (one thread per block, fp64 like the Python floats of the reference) instead of being baked into the launch.
struct RAdamHyper { double beta1, beta2, eps, wd, lr; };

__global__ void __launch_bounds__(OPT_THREADS)
radam_dev_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v, long long n,
                 RAdamHyper h, const int* __restrict__ step_dev, const float* __restrict__ grad_coef) {
    __shared__ RAdamScalars sa;
    if (threadIdx.x == 0) {
        const double t = static_cast<double>(step_dev[0] + 1);           // this update is step t (state['step'] += 1 first, :81)
        const double beta2_t = pow(h.beta2, t);
        const double n_sma_max = 2.0 / (1.0 - h.beta2) - 1.0;
        const double n_sma = n_sma_max - 2.0 * t * beta2_t / (1.0 - beta2_t);
        double step_size;
        if (n_sma >= 5.0)
            step_size = h.lr * sqrt((1.0 - beta2_t) * (n_sma - 4.0) / (n_sma_max - 4.0) * (n_sma - 2.0) / n_sma * n_sma_max /
                                    (n_sma_max - 2.0)) / (1.0 - pow(h.beta1, t));
        else
            step_size = h.lr / (1.0 - pow(h.beta1, t));
        RAdamScalars a;
        a.beta1 = static_cast<float>(h.beta1); a.beta2 = static_cast<float>(h.beta2);
        a.omb1 = static_cast<float>(1.0 - h.beta1); a.omb2 = static_cast<float>(1.0 - h.beta2); a.eps = static_cast<float>(h.eps);
        a.wd_lr = static_cast<float>(h.wd * h.lr); a.step_size = static_cast<float>(step_size); a.use_denom = n_sma >= 5.0;
        sa = a;
    }
    __syncthreads();
    const RAdamScalars a = sa;
    const float gc = grad_coef ? grad_coef[0] : 1.0f;
    const long long stride = static_cast<long long>(gridDim.x) * OPT_THREADS;
    const long long i0 = static_cast<long long>(blockIdx.x) * OPT_THREADS + threadIdx.x;
    const bool al = ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(m) |
                      reinterpret_cast<uintptr_t>(v)) & 15) == 0;
    long long done = 0;
    if (al) {
        const long long n4 = n >> 2;
        float4* p4 = reinterpret_cast<float4*>(p);
        const float4* g4 = reinterpret_cast<const float4*>(g);
        float4* m4 = reinterpret_cast<float4*>(m);
        float4* v4 = reinterpret_cast<float4*>(v);
        for (long long i = i0; i < n4; i += stride) {
            float4 pp = p4[i], mm = m4[i], vv = v4[i];
            const float4 gg = g4[i];
            radam_one(pp.x, gg.x * gc, mm.x, vv.x, a);
            radam_one(pp.y, gg.y * gc, mm.y, vv.y, a);
            radam_one(pp.z, gg.z * gc, mm.z, vv.z, a);
            radam_one(pp.w, gg.w * gc, mm.w, vv.w, a);
            p4[i] = pp; m4[i] = mm; v4[i] = vv;
        }
        done = n4 << 2;
    }
    for (long long i = done + i0; i < n; i += stride) {
        float pp = p[i], mm = m[i], vv = v[i];
        radam_one(pp, g[i] * gc, mm, vv, a);
        p[i] = pp; m[i] = mm; v[i] = vv;
    }
}
__global__ void step_increment_kernel(int* step_dev) { step_dev[0] += 1; }

static int grid_1d(long long work_items, int cap) {
    long long b = (work_items + OPT_THREADS - 1) / OPT_THREADS;
    if (b < 1) b = 1;
    if (b > cap) b = cap;
    return static_cast<int>(b);
}

}  // namespace ft

extern "C" {

int ft_sumsq_partials(const float* x, long long n, float* partials, void* stream) {
    if (!x || !partials || n < 0) return ft::ft_set_error("ft_sumsq_partials: bad argument");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    ft::sumsq_partials_kernel<<<ft::SUMSQ_BLOCKS, ft::OPT_THREADS, 0, st>>>(x, n, partials);
    ft::ft_count_launch(1);
    return ft::ft_check_launch("sumsq_partials_kernel");
}

int ft_clip_coef(const float* partials, int n_partials, float max_norm, float* norm_coef, void* stream) {
    if (!partials || !norm_coef || n_partials <= 0) return ft::ft_set_error("ft_clip_coef: bad argument");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    ft::clip_coef_kernel<<<1, ft::OPT_THREADS, 0, st>>>(partials, n_partials, max_norm, norm_coef);
    ft::ft_count_launch(1);
    return ft::ft_check_launch("clip_coef_kernel");
}

int ft_radam_step(float* p, const float* g, float* m, float* v, long long n, double beta1, double beta2, double eps,
                  double weight_decay_lr, double step_size, int use_denom, const float* grad_coef, void* stream) {
    if (!p || !g || !m || !v || n < 0) return ft::ft_set_error("ft_radam_step: bad argument");
    if (n == 0) return 0;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    ft::RAdamScalars a;
    // scalars arrive in double like the Python floats the reference passes to each fp32 op (1 - beta is formed in
    // double there, radam.py:78-79) and are rounded to fp32 once
    a.beta1 = static_cast<float>(beta1); a.beta2 = static_cast<float>(beta2);
    a.omb1 = static_cast<float>(1.0 - beta1); a.omb2 = static_cast<float>(1.0 - beta2); a.eps = static_cast<float>(eps);
    a.wd_lr = static_cast<float>(weight_decay_lr); a.step_size = static_cast<float>(step_size); a.use_denom = use_denom;
    // 132 SMs (H100 SXM) x 8 resident CTAs of 256 threads, 4 elements per thread-iteration
    ft::radam_kernel<<<ft::grid_1d((n + 3) / 4, 132 * 8), ft::OPT_THREADS, 0, st>>>(p, g, m, v, n, a, grad_coef);
    ft::ft_count_launch(1);
    return ft::ft_check_launch("radam_kernel");
}

}  // extern "C"

extern "C" {

/* RAdam update with the step count on the device (graph-capturable): uses step_dev[0] + 1 as this update's step; the caller
 * bumps the counter once per optimizer step with ft_step_increment after every segment has been updated. */
int ft_radam_step_dev(float* p, const float* g, float* m, float* v, long long n, double beta1, double beta2, double eps,
                      double weight_decay, double lr, const int* step_dev, const float* grad_coef, void* stream) {
    if (!p || !g || !m || !v || !step_dev || n < 0) return ft::ft_set_error("ft_radam_step_dev: bad argument");
    if (n == 0) return 0;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    ft::RAdamHyper h{beta1, beta2, eps, weight_decay, lr};
    ft::radam_dev_kernel<<<ft::grid_1d((n + 3) / 4, 132 * 8), ft::OPT_THREADS, 0, st>>>(p, g, m, v, n, h, step_dev, grad_coef);
    ft::ft_count_launch(1);
    return ft::ft_check_launch("radam_dev_kernel");
}

int ft_step_increment(int* step_dev, void* stream) {
    if (!step_dev) return ft::ft_set_error("ft_step_increment: NULL argument");
    ft::step_increment_kernel<<<1, 1, 0, static_cast<cudaStream_t>(stream)>>>(step_dev);
    ft::ft_count_launch(1);
    return ft::ft_check_launch("step_increment_kernel");
}

}  // extern "C"
