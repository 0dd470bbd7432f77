// Synthesis side of the Gaussian-mixture prior (FlowtronLoss gm_loss=True, flowtron.py:217-230): a sampler that draws z from
// the per-element mixture the flows were trained to map mels to, and the component responsibilities of a given z.
//
// Sampler: element (b, c, t) of z [B, M, T] takes component k (forced, or drawn from prob[b] by inverting its running sum) and
// z = mean[b|0, c, k] + sigma exp(log_var / 2) eps, eps from Box-Muller.  Its three 24-bit uniforms come from the counter
// hash the encoders' dropout uses (splitmix64 over (seed, counter, element)), with counter = 4 state[1] + draw and element =
// (b M + c) 2^32 + t: nothing depends on B or on the padded T, so a row equals its B = 1 call and a numpy restatement
// reproduces the draws.  A one-thread launch then advances state[1], as enc_rng_advance_kernel does for the dropout masks.
//
// Responsibilities: one warp per (b, m) and frame chunk, lane k = component, the posterior formed in log space with the
// NLL kernels' max shift (gmm.cu); per-chunk sums land in caller scratch and one thread per (b, k) adds them in a fixed
// order, so a row does not depend on the other rows, on B or on the padded length.
#include <cstdint>

#include "ft_internal.h"
#include "../../include/flowtron_b200.h"

namespace ft {
namespace {

constexpr int GS_MAX_K = FT_GMM_MAX_COMPONENTS;
constexpr int GS_MAX_M = 80;
constexpr int GS_FRAMES = 32;        // sampler: frames per CTA (one per lane) ...
constexpr int GS_SLICES = 8;         // ... x channel slices (one per warp)
constexpr int GR_CHUNK = 32;         // responsibilities: frames per warp
constexpr int GR_WARPS = 8;          // mel channels per CTA

// the dropout masks' hash (encoder.cu), restated here so encoder.cu's kernels stay as they are
__device__ __forceinline__ uint32_t hash3(uint64_t seed, uint64_t ctr, uint64_t idx) {
    uint64_t z = seed + 0x9E3779B97F4A7C15ull * (ctr + 1) + idx * 0xD1B54A32D192ED03ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return static_cast<uint32_t>((z ^ (z >> 31)) >> 32);
}
__device__ __forceinline__ float unit24(uint32_t h) { return static_cast<float>(h >> 8) * 0x1p-24f; }   // [0, 1)

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

struct SampleArgs {
    const float* mean; const float* log_var; int per_row;      // [B or 1, M, K]
    const float* prob; const int* n_frames; const int* component;
    int T, M, K; float sigma;
    const unsigned long long* rng; float* z;                   // z [B, M, T]
};

// grid (ceil(T / 32), B), block (32, 8): lane = frame, warp = channel slice; row b's means, standard deviations and the
// running sum of its weights are staged in shared memory first.
__global__ void __launch_bounds__(GS_FRAMES * GS_SLICES) gmm_sample_kernel(SampleArgs a) {
    __shared__ float s_mu[GS_MAX_M * GS_MAX_K], s_sd[GS_MAX_M * GS_MAX_K], cdf[GS_MAX_K];
    __shared__ float s_total;
    __shared__ int s_last;
    const int b = blockIdx.y, t = blockIdx.x * GS_FRAMES + threadIdx.x, tid = threadIdx.y * GS_FRAMES + threadIdx.x;
    const int MK = a.M * a.K;
    const long long po = static_cast<long long>(a.per_row ? b : 0) * MK;
    for (int i = tid; i < MK; i += GS_FRAMES * GS_SLICES) {
        s_mu[i] = a.mean[po + i];
        s_sd[i] = expf(0.5f * a.log_var[po + i]);
    }
    if (tid == 0) {                      // running sum in component order; the last component with positive weight
        float c = 0.f;
        int last = 0;
        for (int k = 0; k < a.K; ++k) {
            const float p = a.prob[b * a.K + k];
            c += p;
            cdf[k] = c;
            if (p > 0.f) last = k;
        }
        s_total = c;
        s_last = last;
    }
    __syncthreads();
    if (t >= a.T) return;
    const int n = min(a.n_frames[b], a.T);
    const int forced = a.component ? a.component[b] : -1;
    const unsigned long long seed = a.rng[0], ctr = a.rng[1] * 4;
    for (int c = threadIdx.y; c < a.M; c += GS_SLICES) {
        float* out = a.z + (static_cast<long long>(b) * a.M + c) * a.T + t;
        if (t >= n) { *out = 0.f; continue; }
        const uint64_t idx = (static_cast<uint64_t>(b * a.M + c) << 32) | static_cast<uint32_t>(t);
        int k = forced;
        if (k < 0 || k >= a.K) {
            // first k whose running sum exceeds u * total: never a zero-weight component; past the end (rounding) the last one
            // with positive weight
            const float x = unit24(hash3(seed, ctr, idx)) * s_total;
            k = s_last;
            for (int j = 0; j < a.K; ++j)
                if (x < cdf[j]) { k = j; break; }
        }
        const float u1 = static_cast<float>((hash3(seed, ctr + 1, idx) >> 8) + 1u) * 0x1p-24f;     // (0, 1]
        const float u2 = unit24(hash3(seed, ctr + 2, idx));
        const float eps = sqrtf(-2.f * logf(u1)) * cospif(2.f * u2);
        *out = s_mu[c * a.K + k] + a.sigma * s_sd[c * a.K + k] * eps;
    }
}

__global__ void gmm_rng_advance_kernel(unsigned long long* rng) { rng[1] += 1; }

struct RespArgs {
    const float* z; const int* lens; int T, B, M, K;
    const float* mean; const float* log_var; int per_row;      // [B or 1, M, K]
    const float* prob;                                         // [B, K]
};

// grid (chunks, B, ceil(M / 8)); part[((b M + m) chunks + chunk) K + k] = sum over the chunk's valid frames of the posterior
// of component k (+0 for a chunk past the row's length)
__global__ void __launch_bounds__(GR_WARPS * 32) gmm_resp_kernel(RespArgs a, float* __restrict__ part) {
    const int chunk = blockIdx.x, b = blockIdx.y, m = blockIdx.z * GR_WARPS + (threadIdx.x >> 5), k = threadIdx.x & 31;
    if (m >= a.M) return;
    const bool on = k < a.K;
    float c0 = 0.f, mu = 0.f, iv = 0.f;
    if (on) {
        const long long o = (static_cast<long long>(a.per_row ? b : 0) * a.M + m) * a.K + k;
        const float lv = a.log_var[o];
        c0 = logf(a.prob[b * a.K + k]) - 0.5f * lv;
        mu = a.mean[o];
        iv = expf(-lv);
    }
    const int t1 = min(min(a.lens[b], a.T), (chunk + 1) * GR_CHUNK);
    float s = 0.f;
    for (int t = chunk * GR_CHUNK; t < t1; ++t) {
        const float d = a.z[(static_cast<long long>(t) * a.B + b) * a.M + m] - mu;
        const float ak = on ? c0 - 0.5f * d * d * iv : -INFINITY;
        const float mx = warp_max(ak);
        const float ls = logf(warp_sum(on ? expf(ak - mx) : 0.f));
        if (on) s += expf((ak - mx) - ls);
    }
    if (on) part[((static_cast<long long>(b) * a.M + m) * gridDim.x + chunk) * a.K + k] = s;
}

// grid B, 32 threads: resp[b, k] = (sum over m, then over chunks, in index order) / (min(len, T) M)
__global__ void __launch_bounds__(32) gmm_resp_final_kernel(const float* __restrict__ part, int chunks, const int* __restrict__ lens,
                                                            int T, int M, int K, float* __restrict__ resp) {
    const int b = blockIdx.x, k = threadIdx.x;
    if (k >= K) return;
    const float* p = part + static_cast<long long>(b) * M * chunks * K + k;
    float s = 0.f;
    for (long long i = 0; i < static_cast<long long>(M) * chunks; ++i) s += p[i * K];
    resp[b * K + k] = s / static_cast<float>(min(lens[b], T) * M);
}

int check_desc(const FtGmmDesc* d) {
    if (!d) return ft_set_error("gmm sample: NULL descriptor");
    if (d->K < 1 || d->K > GS_MAX_K) return ft_set_error("gmm sample: n_components must be in [1, 32]");
    if (d->M < 1 || d->M > GS_MAX_M || d->T < 1 || d->B < 1) return ft_set_error("gmm sample: bad shape (M must be in [1, 80])");
    return 0;
}

}  // namespace
}  // namespace ft

extern "C" {

int ft_gmm_sample(const FtGmmDesc* d, const float* mean, const float* log_var, const float* prob, const int* n_frames,
                  const int* component, float sigma, unsigned long long* rng_state, float* z, void* stream) {
    using namespace ft;
    FT_TRY(check_desc(d));
    if (!mean || !log_var || !prob || !n_frames || !rng_state || !z) return ft_set_error("ft_gmm_sample: NULL argument");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    SampleArgs a{mean, log_var, d->per_row, prob, n_frames, component, d->T, d->M, d->K, sigma, rng_state, z};
    gmm_sample_kernel<<<dim3((d->T + GS_FRAMES - 1) / GS_FRAMES, d->B), dim3(GS_FRAMES, GS_SLICES), 0, st>>>(a);
    ft_count_launch(1);
    FT_TRY(ft_check_launch("gmm_sample_kernel"));
    gmm_rng_advance_kernel<<<1, 1, 0, st>>>(rng_state);
    ft_count_launch(1);
    return ft_check_launch("gmm_rng_advance_kernel");
}

int ft_gmm_responsibilities(const FtGmmDesc* d, const float* z, const int* out_lens, const float* mean, const float* log_var,
                            const float* prob, float* resp, void* scratch, void* stream) {
    using namespace ft;
    FT_TRY(check_desc(d));
    if (!z || !out_lens || !mean || !log_var || !prob || !resp || !scratch) return ft_set_error("ft_gmm_responsibilities: NULL argument");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    RespArgs a{z, out_lens, d->T, d->B, d->M, d->K, mean, log_var, d->per_row, prob};
    const int chunks = (d->T + GR_CHUNK - 1) / GR_CHUNK;
    float* part = static_cast<float*>(scratch);
    gmm_resp_kernel<<<dim3(chunks, d->B, (d->M + GR_WARPS - 1) / GR_WARPS), GR_WARPS * 32, 0, st>>>(a, part);
    ft_count_launch(1);
    FT_TRY(ft_check_launch("gmm_resp_kernel"));
    gmm_resp_final_kernel<<<d->B, 32, 0, st>>>(part, chunks, out_lens, d->T, d->M, d->K, resp);
    ft_count_launch(1);
    return ft_check_launch("gmm_resp_final_kernel");
}

}  // extern "C"
