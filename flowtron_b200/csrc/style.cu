// Posterior mean of a set of reference z for style transfer (the reference's inference_style_transfer.ipynb): the z of K
// reference utterances, averaged frame by frame ('batch') or over their own frames and then over the K ('time_and_batch'),
// and shrunk by scale = ratio / (ratio + 1).
//
// z is Flowtron.forward's flow output [T, B, M] (row t*B + b), so Flowtron.encode's result is read in place.  Both modes
// accumulate in fp32 with Kahan compensation in a fixed order and no atomics, so every run (and every CUDA-graph replay)
// gives the same bits; the time means of mode 1 stay within fp32 rounding of a float64 sum at any length.  The work is a
// few MB of reads, so both kernels are latency-bound: each thread issues its loads several rows or frames ahead of the
// ordered sums that consume them.
#include "ft_internal.h"
#include "../../include/flowtron_b200.h"

namespace ft {

constexpr int STYLE_THREADS = 128;     // mode 0: one thread per mel channel (M <= 128), one CTA per output frame
constexpr int STYLE_BATCH = 8;         // loads issued ahead of their (ordered) sums
constexpr int STYLE_MLANES = 4;        // mode 1: 4 channels per CTA (20 CTAs at M = 80) ...
constexpr int STYLE_SLICES = 256;      // ... x 256 frame slices: 1024 threads

struct Kahan {
    float s = 0.f, c = 0.f;
    __device__ __forceinline__ void add(float x) {
        const float y = x - c;
        const float t = s + y;
        c = (t - s) - y;
        s = t;
    }
};

// mode 0: out[m, t] = scale * (1/B) sum_b z[t mod out_lens[b], b, m].  CTA t, thread m; rows are summed in order b = 0..B-1,
// their loads issued STYLE_BATCH rows ahead.
__global__ void __launch_bounds__(STYLE_THREADS)
posterior_mean_batch_kernel(const float* __restrict__ z, int B, int M, const int* __restrict__ out_lens, int n_frames,
                            float scale, float* __restrict__ out) {
    const int m = threadIdx.x, t = blockIdx.x;
    if (m >= M) return;
    Kahan acc;
    for (int b0 = 0; b0 < B; b0 += STYLE_BATCH) {
        float v[STYLE_BATCH];
#pragma unroll
        for (int j = 0; j < STYLE_BATCH; ++j) {
            const int b = b0 + j;
            v[j] = b < B ? z[(static_cast<long long>(t % out_lens[b]) * B + b) * M + m] : 0.f;
        }
#pragma unroll
        for (int j = 0; j < STYLE_BATCH; ++j)
            if (b0 + j < B) acc.add(v[j]);
    }
    out[static_cast<long long>(m) * n_frames + t] = scale * (acc.s / static_cast<float>(B));
}

// mode 1: out[m] = scale * (1/B) sum_b (1/out_lens[b]) sum_{t < out_lens[b]} z[t, b, m].  CTA x takes channels
// [4x, 4x + 4); slice s of its 1024 threads takes frames t = s, s + 256, ... of every row, in order, and keeps
// sum_b (its share of row b) / out_lens[b]; the 256 slice sums are then added in a fixed tree.
__global__ void __launch_bounds__(STYLE_MLANES * STYLE_SLICES)
posterior_mean_time_kernel(const float* __restrict__ z, int B, int M, const int* __restrict__ out_lens, float scale,
                           float* __restrict__ out) {
    __shared__ float part[STYLE_SLICES][STYLE_MLANES];
    const int lane = threadIdx.x % STYLE_MLANES, slice = threadIdx.x / STYLE_MLANES;
    const int m = blockIdx.x * STYLE_MLANES + lane;
    Kahan rows;
    if (m < M) {
        const long long step = static_cast<long long>(STYLE_SLICES) * B * M;
        for (int b = 0; b < B; ++b) {
            const int len = out_lens[b];
            const float* zb = z + (static_cast<long long>(slice) * B + b) * M + m;
            Kahan frames;
            for (int t0 = slice; t0 < len; t0 += STYLE_SLICES * STYLE_BATCH) {
                float v[STYLE_BATCH];
                const float* p = zb + static_cast<long long>((t0 - slice) / STYLE_SLICES) * step;
#pragma unroll
                for (int j = 0; j < STYLE_BATCH; ++j) v[j] = t0 + j * STYLE_SLICES < len ? p[j * step] : 0.f;
#pragma unroll
                for (int j = 0; j < STYLE_BATCH; ++j)
                    if (t0 + j * STYLE_SLICES < len) frames.add(v[j]);
            }
            rows.add(frames.s / static_cast<float>(len));
        }
    }
    part[slice][lane] = rows.s;
    __syncthreads();
    for (int h = STYLE_SLICES / 2; h > 0; h >>= 1) {
        if (slice < h) part[slice][lane] += part[slice + h][lane];
        __syncthreads();
    }
    if (slice == 0 && m < M) out[m] = scale * (part[0][lane] / static_cast<float>(B));
}

}  // namespace ft

extern "C" {

int ft_posterior_mean(const float* z, int T, int B, int M, const int* out_lens, int n_frames, int mode, float scale,
                      float* out, void* stream) {
    using namespace ft;
    if (!z || !out_lens || !out) return ft_set_error("ft_posterior_mean: NULL argument");
    if (B < 1) return ft_set_error("ft_posterior_mean: B < 1");
    if (T < 1) return ft_set_error("ft_posterior_mean: T < 1");
    if (n_frames < 1) return ft_set_error("ft_posterior_mean: n_frames < 1");
    if (M < 1 || M > STYLE_THREADS) return ft_set_error("ft_posterior_mean: M must lie in [1, 128]");
    if (mode != 0 && mode != 1) return ft_set_error("ft_posterior_mean: mode must be 0 (batch) or 1 (time_and_batch)");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    TimeScope ts(mode == 0 ? "posterior_mean_batch" : "posterior_mean_time", n_frames, B, M, st);
    if (mode == 0) {
        posterior_mean_batch_kernel<<<n_frames, STYLE_THREADS, 0, st>>>(z, B, M, out_lens, n_frames, scale, out);
    } else {
        const int grid = (M + STYLE_MLANES - 1) / STYLE_MLANES;
        posterior_mean_time_kernel<<<grid, STYLE_MLANES * STYLE_SLICES, 0, st>>>(z, B, M, out_lens, scale, out);
    }
    ft_count_launch(1);
    return ft_check_launch(mode == 0 ? "posterior_mean_batch_kernel" : "posterior_mean_time_kernel");
}

}  // extern "C"
