// Hard alignments from attention log-probabilities: a batched monotonic alignment search (MAS, the Viterbi step of "One
// TTS Alignment to Rule Them All") and the one-hot maps of a row of per-token durations.
//
// ft_mas_align, utterance b (Tb = out_lens[b] frames, Lb = in_lens[b] tokens), s[t][l] = logp[b, t', l] with t' = t, or
// t' = Tb-1-t for an AR_Back_Step's flipped time:
//   Q[0][0] = s[0][0], Q[0][l > 0] = -inf;   Q[t][l] = s[t][l] + max(Q[t-1][l], Q[t-1][l-1])   (Q[t-1][-1] = -inf)
// and the path back from (Tb-1, Lb-1) moves to l-1 only where Q[t-1][l-1] > Q[t-1][l] (ties stay on the token).  One
// CTA per utterance, like the attention-CTC kernel: thread tid owns states tid + j * blockDim (j < NS), the Q row is
// double-buffered in shared memory (one __syncthreads per frame), logp is loaded MAS_PREFETCH frames ahead of its use, and
// each warp packs its 32 backpointer bits of a frame into one word with __ballot_sync (caller scratch, [T][W] words per
// row, W = ceil(L / 32)).  The add is __fadd_rn and the max a strict compare, so the path is bit-for-bit that of a float32
// restatement.  The backtrace is a serial chain: it runs in chunks of MAS_CHUNK frames, over which l falls by at most
// MAS_CHUNK - 1, so the MAS_STAGE words per frame it can touch are staged in shared memory by the whole CTA first and one
// thread then walks the chunk without a dependent global load per frame.
#include <math_constants.h>

#include "ft_internal.h"
#include "../../include/flowtron_b200.h"

namespace ft {

constexpr int MAS_MAX_THREADS = 256;
constexpr int MAS_NS_LONG = 4;             // states per thread past 256 tokens: 4 * 256 = FT_MAX_TEXT_LEN
constexpr int MAS_PREFETCH = 8;            // frames of logp in flight ahead of the recursion
constexpr int MAS_CHUNK = 128;             // backtrace frames per staging round
constexpr int MAS_STAGE = (MAS_CHUNK - 1 + 31) / 32 + 1;   // words per frame a chunk can touch
static_assert(MAS_NS_LONG * MAS_MAX_THREADS >= FT_MAX_TEXT_LEN, "MAS states must fit in one block");

constexpr int D2A_THREADS = 256;           // ft_durations_to_attn: 4 tokens per thread in the prefix sum
constexpr int D2A_ROWS = 64;               // output rows per CTA
static_assert(4 * D2A_THREADS >= FT_MAX_TEXT_LEN, "durations must fit in one block");

template <int NS>
__global__ void __launch_bounds__(MAS_MAX_THREADS)
mas_kernel(const float* __restrict__ logp, const int* __restrict__ in_lens, const int* __restrict__ out_lens, int T, int L,
           int reversed, int* __restrict__ durations, int* __restrict__ token_of_frame, unsigned* __restrict__ bp_scratch) {
    __shared__ float qbuf[2][FT_MAX_TEXT_LEN + 1];      // Q[t-1] / Q[t]; index l + 1, index 0 is the -inf of l = -1
    __shared__ int dur[FT_MAX_TEXT_LEN];
    __shared__ unsigned stage[MAS_CHUNK][MAS_STAGE];
    __shared__ int tokc[MAS_CHUNK];
    __shared__ int s_l, s_cnt;
    const int b = blockIdx.x, tid = threadIdx.x, nth = blockDim.x, lane = tid & 31, warp = tid >> 5;
    int Lb = in_lens[b], Tb = out_lens[b];
    Lb = Lb < 0 ? 0 : (Lb > L ? L : Lb);
    Tb = Tb < 0 ? 0 : (Tb > T ? T : Tb);
    const bool path = Lb > 0 && Tb >= Lb;
    int* tok_out = token_of_frame + static_cast<long long>(b) * T;
    for (int l = tid; l < L; l += nth) dur[l] = 0;
    for (int t = path ? Tb + tid : tid; t < T; t += nth) tok_out[t] = -1;
    if (!path) {
        for (int l = tid; l < L; l += nth) durations[static_cast<long long>(b) * L + l] = 0;
        return;
    }
    const int W = (L + 31) >> 5;
    const float* x = logp + static_cast<long long>(b) * T * L;
    unsigned* bp = bp_scratch + static_cast<long long>(b) * T * W;
    auto row = [&](int t) -> long long { return static_cast<long long>(reversed ? Tb - 1 - t : t) * L; };
    const float NEG = -CUDART_INF_F;

    // ---- forward recursion
    bool live[NS];
    float q[NS];
#pragma unroll
    for (int j = 0; j < NS; ++j) {
        const int l = tid + j * nth;
        live[j] = l < Lb;
        q[j] = (l == 0) ? x[row(0)] : NEG;
        if (live[j]) qbuf[0][l + 1] = q[j];
    }
    if (tid == 0) qbuf[0][0] = qbuf[1][0] = NEG;
    float v[MAS_PREFETCH][NS];
#pragma unroll
    for (int k = 0; k < MAS_PREFETCH; ++k)
#pragma unroll
        for (int j = 0; j < NS; ++j)
            v[k][j] = (live[j] && 1 + k < Tb) ? x[row(1 + k) + tid + j * nth] : 0.f;
    __syncthreads();
    int cur = 1;
    for (int t0 = 1; t0 < Tb; t0 += MAS_PREFETCH) {
#pragma unroll
        for (int k = 0; k < MAS_PREFETCH; ++k) {
            const int t = t0 + k;
            if (t >= Tb) break;
            const float* prev = qbuf[cur ^ 1];
            float* next = qbuf[cur];
#pragma unroll
            for (int j = 0; j < NS; ++j) {
                const int l = tid + j * nth;
                const float up = live[j] ? prev[l] : NEG;           // Q[t-1][l-1]
                const bool mv = up > q[j];
                const float val = live[j] ? __fadd_rn(v[k][j], mv ? up : q[j]) : NEG;
                if (live[j] && t + MAS_PREFETCH < Tb) v[k][j] = x[row(t + MAS_PREFETCH) + l];
                const unsigned word = __ballot_sync(0xffffffffu, live[j] && mv);
                const int l0 = j * nth + warp * 32;
                if (lane == 0 && l0 < Lb) bp[static_cast<long long>(t) * W + (l0 >> 5)] = word;
                q[j] = val;
                if (live[j]) next[l + 1] = val;
            }
            __syncthreads();
            cur ^= 1;
        }
    }

    // ---- backtrace from (Tb-1, Lb-1), MAS_CHUNK frames per round
    const int Wb = (Lb + 31) >> 5;
    if (tid == 0) { s_l = Lb - 1; s_cnt = 0; }
    for (int t_hi = Tb - 1; t_hi >= 0; t_hi -= MAS_CHUNK) {
        __syncthreads();
        const int lh = s_l;
        const int t_lo = t_hi - MAS_CHUNK + 1 > 0 ? t_hi - MAS_CHUNK + 1 : 0;
        const int w0 = (lh - MAS_CHUNK + 1 > 0 ? lh - MAS_CHUNK + 1 : 0) >> 5;
        for (int i = tid; i < MAS_CHUNK * MAS_STAGE; i += nth) {
            const int k = i / MAS_STAGE, w = i % MAS_STAGE, t = t_hi - k;
            if (t >= t_lo && t >= 1 && w0 + w < Wb) stage[k][w] = bp[static_cast<long long>(t) * W + w0 + w];
        }
        __syncthreads();
        if (tid == 0) {
            int l = lh, cnt = s_cnt;
            for (int t = t_hi; t >= t_lo; --t) {
                tokc[t_hi - t] = l;
                ++cnt;
                if (t > 0 && ((stage[t_hi - t][(l >> 5) - w0] >> (l & 31)) & 1u)) {
                    dur[l] = cnt;
                    cnt = 0;
                    --l;
                }
            }
            if (t_lo == 0) dur[l] = cnt;
            s_l = l;
            s_cnt = cnt;
        }
        __syncthreads();
        for (int k = tid; k <= t_hi - t_lo; k += nth) tok_out[t_hi - k] = tokc[k];
    }
    __syncthreads();
    for (int l = tid; l < L; l += nth) durations[static_cast<long long>(b) * L + l] = dur[l];
}

// One-hot maps of per-token durations.  CTA (b, y) computes row b's inclusive prefix sums cum[l] = sum_{k <= l} d_k over
// its in_lens[b] tokens (negative durations count as 0), then writes rows i in [64 y, 64 y + 64) of out[b]: generation step
// i is natural frame j = i, or n_b - 1 - i when reversed, and belongs to the first token l with cum[l] > j.
__global__ void __launch_bounds__(D2A_THREADS)
durations_to_attn_kernel(const int* __restrict__ durations, const int* __restrict__ in_lens, int L, int Ta, int reversed,
                         float* __restrict__ out) {
    __shared__ int cum[4 * D2A_THREADS];
    __shared__ int wsum[D2A_THREADS / 32];
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    int Lb = in_lens[b];
    Lb = Lb < 0 ? 0 : (Lb > L ? L : Lb);
    const int* d = durations + static_cast<long long>(b) * L;
    int v[4], s = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int l = 4 * tid + k;
        const int dl = l < Lb ? d[l] : 0;
        s += dl > 0 ? dl : 0;
        v[k] = s;
    }
    int incl = s;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += y;
    }
    if (lane == 31) wsum[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        int w = lane < D2A_THREADS / 32 ? wsum[lane] : 0;
#pragma unroll
        for (int o = 1; o < D2A_THREADS / 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, w, o);
            if (lane >= o) w += y;
        }
        if (lane < D2A_THREADS / 32) wsum[lane] = w;
    }
    __syncthreads();
    const int off = (warp > 0 ? wsum[warp - 1] : 0) + incl - s;
#pragma unroll
    for (int k = 0; k < 4; ++k) cum[4 * tid + k] = off + v[k];
    __syncthreads();
    const int n = wsum[D2A_THREADS / 32 - 1];
    float* o = out + static_cast<long long>(b) * Ta * L;
    const int i_end = min(Ta, (blockIdx.y + 1) * D2A_ROWS);
    for (int i = blockIdx.y * D2A_ROWS + warp; i < i_end; i += D2A_THREADS / 32) {
        int tok = -1;
        if (i < n) {
            const int j = reversed ? n - 1 - i : i;
            int lo = 0, hi = Lb - 1;                    // cum[Lb - 1] = n > j: the answer lies in [0, Lb - 1]
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (cum[mid] > j) hi = mid; else lo = mid + 1;
            }
            tok = lo;
        }
        float* r = o + static_cast<long long>(i) * L;
        for (int l = lane; l < L; l += 32) r[l] = l == tok ? 1.f : 0.f;
    }
}

}  // namespace ft

extern "C" {

size_t ft_mas_align_scratch_bytes(int B, int T, int L) {
    if (B <= 0 || T <= 0 || L <= 0) return 0;
    return static_cast<size_t>(B) * T * ((static_cast<size_t>(L) + 31) / 32) * sizeof(unsigned);
}

int ft_mas_align(const float* logp, const int* in_lens, const int* out_lens, int B, int T, int L, int time_reversed,
                 int* durations, int* token_of_frame, void* scratch, void* stream) {
    using namespace ft;
    if (!logp || !in_lens || !out_lens || !durations || !token_of_frame || !scratch)
        return ft_set_error("ft_mas_align: NULL argument");
    if (B <= 0 || T <= 0 || L <= 0) return 0;
    if (L > FT_MAX_TEXT_LEN) return ft_set_error("ft_mas_align: L > FT_MAX_TEXT_LEN (1024) not supported");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const bool longk = L > MAS_MAX_THREADS;
    const int per = longk ? MAS_NS_LONG : 1;
    const int threads = ((L + per - 1) / per + 31) / 32 * 32;
    TimeScope ts("mas_align", T, B, L, st);
    auto kern = longk ? mas_kernel<MAS_NS_LONG> : mas_kernel<1>;
    kern<<<B, threads, 0, st>>>(logp, in_lens, out_lens, T, L, time_reversed ? 1 : 0, durations, token_of_frame,
                                static_cast<unsigned*>(scratch));
    ft_count_launch(1);
    return ft_check_launch("mas_kernel");
}

int ft_durations_to_attn(const int* durations, const int* in_lens, int B, int L, int Ta, int time_reversed, float* out,
                         void* stream) {
    using namespace ft;
    if (!durations || !in_lens || !out) return ft_set_error("ft_durations_to_attn: NULL argument");
    if (B <= 0 || L <= 0 || Ta <= 0) return 0;
    if (L > FT_MAX_TEXT_LEN) return ft_set_error("ft_durations_to_attn: L > FT_MAX_TEXT_LEN (1024) not supported");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    TimeScope ts("durations_to_attn", Ta, B, L, st);
    const dim3 grid(B, (Ta + D2A_ROWS - 1) / D2A_ROWS);
    durations_to_attn_kernel<<<grid, D2A_THREADS, 0, st>>>(durations, in_lens, L, Ta, time_reversed ? 1 : 0, out);
    ft_count_launch(1);
    return ft_check_launch("durations_to_attn_kernel");
}

}  // extern "C"
