// Gaussian-mixture NLL of the Flowtron prior (FlowtronLoss with gm_loss=True, flowtron.py:217-235) and its gradient.
//
// Per valid element (t < out_lens[b], b, m) with a_k = log prob_bk - log_var_bmk / 2 - (z_tbm - mean_bmk)^2 / (2 exp log_var_bmk):
//   nll = -sum logsumexp_k a_k
// (the reference's max-shifted form: no sigma, no 2 pi).  One warp per (b, m) and frame chunk, lane k = mixture component
// (K <= 32), so the logsumexp is a max and a sum over the warp with every a_k shifted by the true maximum: stable for any log_var.
// Every sum has a fixed order and there are no atomics: partial sums per (frame chunk, b, m) land in caller scratch and a second
// launch adds them up in index order, so graph replays are bit-identical.
#include "ft_internal.h"
#include "../../include/flowtron_b200.h"

namespace ft {

constexpr int GMM_CHUNK = 32;        // frames per warp
constexpr int GMM_WARPS = 8;         // mel channels per CTA
constexpr int GMM_MAX_K = 32;

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

struct GmmArgs {
    const float* z; const int* lens; int T, B, M, K;
    const float* mean; const float* log_var; int per_row;     // [B or 1, M, K]
    const float* prob;                                         // [B, K]
};

// this lane's component constants for (b, m): log prob - log_var / 2, -log_var / 2, log prob, mean, exp(-log_var); lanes >= K
// get a = -inf
struct GmmLane { float c0, hl, lp, mu, iv; bool on; };
__device__ __forceinline__ GmmLane gmm_lane(const GmmArgs& a, int b, int m, int k) {
    GmmLane g{0.f, 0.f, 0.f, 0.f, 0.f, k < a.K};
    if (g.on) {
        const long long o = (static_cast<long long>(a.per_row ? b : 0) * a.M + m) * a.K + k;
        const float lv = a.log_var[o];
        g.hl = -0.5f * lv;
        g.lp = logf(a.prob[b * a.K + k]);
        g.c0 = g.lp + g.hl;
        g.mu = a.mean[o];
        g.iv = expf(-lv);
    }
    return g;
}

// grid (chunks, B, ceil(M / 8)); part[(b * M + m) * chunks + chunk] = sum over the chunk's valid frames of logsumexp_k a_k
__global__ void __launch_bounds__(GMM_WARPS * 32) gmm_reduce_kernel(GmmArgs a, float* __restrict__ part) {
    const int chunk = blockIdx.x, b = blockIdx.y, m = blockIdx.z * GMM_WARPS + (threadIdx.x >> 5), k = threadIdx.x & 31;
    if (m >= a.M) return;
    const GmmLane g = gmm_lane(a, b, m, k);
    const int t1 = min(min(a.lens[b], a.T), (chunk + 1) * GMM_CHUNK);
    float s = 0.f;
    for (int t = chunk * GMM_CHUNK; t < t1; ++t) {
        const float d = a.z[(static_cast<long long>(t) * a.B + b) * a.M + m] - g.mu;
        const float ak = g.on ? g.c0 - 0.5f * d * d * g.iv : -INFINITY;
        const float mx = warp_max(ak);
        s += mx + logf(warp_sum(g.on ? expf(ak - mx) : 0.f));
    }
    if (k == 0) part[(static_cast<long long>(b) * a.M + m) * gridDim.x + chunk] = s;
}

// one CTA: sums[0] = -sum of the partials (the NLL), sums[1] = number of valid frames (sum of min(out_lens, T))
__global__ void gmm_reduce_final_kernel(const float* __restrict__ part, long long n, const int* __restrict__ lens, int B, int T,
                                        float* __restrict__ sums) {
    __shared__ float sm[256];
    float s = 0.f;
    for (long long i = threadIdx.x; i < n; i += 256) s += part[i];
    sm[threadIdx.x] = s;
    __syncthreads();
    for (int w = 128; w; w >>= 1) {
        if (threadIdx.x < w) sm[threadIdx.x] += sm[threadIdx.x + w];
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        float nf = 0.f;
        for (int b = 0; b < B; ++b) nf += static_cast<float>(min(lens[b], T));
        sums[0] = -sm[0];
        sums[1] = nf;
    }
}

// grid B, 128 threads: rows[b] = -(sum over m of (sum over chunks of the row's partials, in chunk order)), the m terms added
// in channel order by one thread.  Only row b's partials are read, and chunks past its length hold +0, so the value does not
// depend on the other rows, on B or on the padded length.
__global__ void __launch_bounds__(128) gmm_rows_final_kernel(const float* __restrict__ part, int chunks, int M,
                                                             float* __restrict__ rows) {
    __shared__ float sm[128];
    const int b = blockIdx.x;
    float s = 0.f;
    if (threadIdx.x < M) {
        const float* p = part + (static_cast<long long>(b) * M + threadIdx.x) * chunks;
        for (int c = 0; c < chunks; ++c) s += p[c];
    }
    sm[threadIdx.x] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        float r = 0.f;
        for (int m = 0; m < M; ++m) r += sm[m];
        rows[b] = -r;
    }
}

// Gradient of g * nll.  Per valid element, r_k = exp(a_k - lse), e_k = exp(a_k - log prob_k - lse), u_k = (z - mean_k) exp(-log_var_k):
//   dz = g sum_k r_k u_k ;  dmean_k = -g sum_t r_k u_k ;  dlog_var_k = g sum_t (r_k - r_k u_k (z - mean_k)) / 2 ;  dprob_k = -g sum_{t,m} e_k
// (e_k, not r_k / prob_k, so a vanishing prob_k has a finite gradient).  dz is written for every frame (zero past the length); the
// per-chunk sums of e, r u and r u (z - mean) go to part [(b, m, k), chunk, 3] for gmm_grad_final_kernel.
__global__ void __launch_bounds__(GMM_WARPS * 32) gmm_grad_kernel(GmmArgs a, const float* __restrict__ g_nll, float* __restrict__ dz,
                                                                  float* __restrict__ part) {
    const int chunk = blockIdx.x, b = blockIdx.y, m = blockIdx.z * GMM_WARPS + (threadIdx.x >> 5), k = threadIdx.x & 31;
    if (m >= a.M) return;
    const GmmLane g = gmm_lane(a, b, m, k);
    const float gn = g_nll[0];
    const int len = min(a.lens[b], a.T), t0 = chunk * GMM_CHUNK, t1 = min(a.T, t0 + GMM_CHUNK);
    float se = 0.f, su = 0.f, sv = 0.f;
    for (int t = t0; t < t1; ++t) {
        const long long zi = (static_cast<long long>(t) * a.B + b) * a.M + m;
        if (t >= len) { if (k == 0) dz[zi] = 0.f; continue; }
        const float d = a.z[zi] - g.mu;
        const float ak = g.on ? g.c0 - 0.5f * d * d * g.iv : -INFINITY;
        // a_k - lse is formed as (a_k - max) - log(sum): a_k and lse can both be ~1e8 (log_var -20) and differ by a little
        const float mx = warp_max(ak);
        const float ls = logf(warp_sum(g.on ? expf(ak - mx) : 0.f));
        const float r = g.on ? expf((ak - mx) - ls) : 0.f;
        const float u = d * g.iv;
        const float dzs = warp_sum(r * u);
        if (k == 0) dz[zi] = gn * dzs;
        if (g.on) {
            se += g.lp > -INFINITY ? expf((ak - mx) - ls - g.lp) : expf((g.hl - 0.5f * d * d * g.iv - mx) - ls);
            su += r * u;
            sv += r * u * d;
        }
    }
    if (g.on) {
        float* p = part + ((((static_cast<long long>(b) * a.M + m) * a.K + k) * gridDim.x + chunk) * 3);
        p[0] = se; p[1] = su; p[2] = sv;
    }
}

// grid B, 256 threads: dmean / dlog_var [B, M, K] (per-row Gaussians only) and dprob [B, K], the chunks added in order
__global__ void gmm_grad_final_kernel(GmmArgs a, const float* __restrict__ part, int chunks, const float* __restrict__ g_nll,
                                      float* __restrict__ dmean, float* __restrict__ dlog_var, float* __restrict__ dprob) {
    __shared__ float se_mk[GMM_MAX_K][81];
    const int b = blockIdx.x;
    const float gn = g_nll[0];
    for (int i = threadIdx.x; i < a.M * a.K; i += blockDim.x) {
        const int m = i / a.K, k = i - m * a.K;
        const float* p = part + (static_cast<long long>(b) * a.M * a.K + i) * chunks * 3;
        float se = 0.f, su = 0.f, sv = 0.f;
        for (int c = 0; c < chunks; ++c) { se += p[3 * c]; su += p[3 * c + 1]; sv += p[3 * c + 2]; }
        se_mk[k][m] = se;
        if (dmean) {
            const float pk = a.prob[b * a.K + k];
            dmean[static_cast<long long>(b) * a.M * a.K + i] = -gn * su;
            dlog_var[static_cast<long long>(b) * a.M * a.K + i] = 0.5f * gn * (pk * se - sv);
        }
    }
    __syncthreads();
    if (threadIdx.x < a.K) {
        float s = 0.f;
        for (int m = 0; m < a.M; ++m) s += se_mk[threadIdx.x][m];
        dprob[b * a.K + threadIdx.x] = -gn * s;
    }
}

static int check_gmm(const FtGmmDesc* d) {
    if (!d) return ft_set_error("gmm: NULL descriptor");
    if (d->K < 1 || d->K > GMM_MAX_K) return ft_set_error("gmm: n_components must be in [1, 32]");
    if (d->M < 1 || d->M > 80 || d->T < 1 || d->B < 1) return ft_set_error("gmm: bad shape (M must be in [1, 80])");
    return 0;
}
static int gmm_chunks(const FtGmmDesc* d) { return (d->T + GMM_CHUNK - 1) / GMM_CHUNK; }

}  // namespace ft

extern "C" {

size_t ft_gmm_nll_scratch_bytes(const FtGmmDesc* d) {
    if (ft::check_gmm(d)) return 0;
    return sizeof(float) * static_cast<size_t>(ft::gmm_chunks(d)) * d->B * d->M * d->K * 3 + 256;
}

int ft_gmm_nll_reduce(const FtGmmDesc* d, const float* z, const int* out_lens, const float* mean, const float* log_var,
                      const float* prob, float* sums, void* scratch, void* stream) {
    using namespace ft;
    if (check_gmm(d)) return -1;
    if (!z || !out_lens || !mean || !log_var || !prob || !sums || !scratch) return ft_set_error("ft_gmm_nll_reduce: NULL argument");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    GmmArgs a{z, out_lens, d->T, d->B, d->M, d->K, mean, log_var, d->per_row, prob};
    const int chunks = gmm_chunks(d);
    float* part = static_cast<float*>(scratch);
    gmm_reduce_kernel<<<dim3(chunks, d->B, (d->M + GMM_WARPS - 1) / GMM_WARPS), GMM_WARPS * 32, 0, st>>>(a, part);
    ft_count_launch(1);
    if (ft_check_launch("gmm_reduce_kernel")) return -1;
    gmm_reduce_final_kernel<<<1, 256, 0, st>>>(part, static_cast<long long>(chunks) * d->B * d->M, out_lens, d->B, d->T, sums);
    ft_count_launch(1);
    return ft_check_launch("gmm_reduce_final_kernel");
}

int ft_gmm_nll_rows(const FtGmmDesc* d, const float* z, const int* out_lens, const float* mean, const float* log_var,
                    const float* prob, float* rows_out, void* scratch, void* stream) {
    using namespace ft;
    if (check_gmm(d)) return -1;
    if (!z || !out_lens || !mean || !log_var || !prob || !rows_out || !scratch) return ft_set_error("ft_gmm_nll_rows: NULL argument");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    GmmArgs a{z, out_lens, d->T, d->B, d->M, d->K, mean, log_var, d->per_row, prob};
    const int chunks = gmm_chunks(d);
    float* part = static_cast<float*>(scratch);
    gmm_reduce_kernel<<<dim3(chunks, d->B, (d->M + GMM_WARPS - 1) / GMM_WARPS), GMM_WARPS * 32, 0, st>>>(a, part);
    ft_count_launch(1);
    if (ft_check_launch("gmm_reduce_kernel")) return -1;
    gmm_rows_final_kernel<<<d->B, 128, 0, st>>>(part, chunks, d->M, rows_out);
    ft_count_launch(1);
    return ft_check_launch("gmm_rows_final_kernel");
}

int ft_gmm_nll_grad(const FtGmmDesc* d, const float* z, const int* out_lens, const float* mean, const float* log_var,
                    const float* prob, const float* g_nll, float* dz, float* dmean, float* dlog_var, float* dprob, void* scratch,
                    void* stream) {
    using namespace ft;
    if (check_gmm(d)) return -1;
    if (!z || !out_lens || !mean || !log_var || !prob || !g_nll || !dz || !dprob || !scratch) return ft_set_error("ft_gmm_nll_grad: NULL argument");
    if ((dmean == nullptr) != (dlog_var == nullptr)) return ft_set_error("ft_gmm_nll_grad: dmean and dlog_var go together");
    if (dmean && !d->per_row) return ft_set_error("ft_gmm_nll_grad: shared Gaussians have no gradient here (fixed buffers)");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    GmmArgs a{z, out_lens, d->T, d->B, d->M, d->K, mean, log_var, d->per_row, prob};
    const int chunks = gmm_chunks(d);
    float* part = static_cast<float*>(scratch);
    gmm_grad_kernel<<<dim3(chunks, d->B, (d->M + GMM_WARPS - 1) / GMM_WARPS), GMM_WARPS * 32, 0, st>>>(a, g_nll, dz, part);
    ft_count_launch(1);
    if (ft_check_launch("gmm_grad_kernel")) return -1;
    gmm_grad_final_kernel<<<d->B, 256, 0, st>>>(a, part, chunks, g_nll, dmean, dlog_var, dprob);
    ft_count_launch(1);
    return ft_check_launch("gmm_grad_final_kernel");
}

}  // extern "C"
