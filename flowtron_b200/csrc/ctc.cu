// Batched attention-CTC loss (AttentionCTCLoss, flowtron.py:155-182, called per flow from FlowtronLoss :245-274) with its
// gradient, one CTA per utterance -- the reference loops over the batch in Python with .item() host syncs, pads a blank
// column, slices, log_softmaxes and calls nn.CTCLoss once per utterance.
//
// Utterance b (Tq = out_lens[b] frames, K = in_lens[b] tokens): classes c = 0 (blank, constant logit blank_logprob) and
// c = 1..K (logit attn_logprob[b, t, c-1]); lp[t,c] = log_softmax_c; target = 1, 2, ..., K (every token once, in order), so
// the extended sequence is blank,1,blank,2,...,K,blank (S = 2K+1 states) and the skip transition s-2 -> s is always allowed
// for token states.  Standard log-space alpha/beta recursions (Graves 2006):
//   alpha_t(s) = lp[t, l_s] + LSE(alpha_{t-1}(s), alpha_{t-1}(s-1), [s odd] alpha_{t-1}(s-2)),   nll = -LSE(alpha_T(S-1), alpha_T(S-2))
//   d nll / d logit[t,k] = exp(lp[t,k]) - exp(alpha_t(2k-1) + beta_t(2k-1) + nll - lp[t,k])       (same expression ATen returns)
// cost[b] = nll / K (nn.CTCLoss reduction='mean' divides by the target length), 0 with zero gradient if nll is inf
// (zero_infinity=True).  For AR_Back_Step flows attn_logprob is in the flow's flipped time (row q = len-1-t holds natural
// frame t): the reference un-rolls and un-flips it (:250-256); here it is an index map.
// Thread s owns state s; alpha_{t-1} / beta_{t+1} live in a double-buffered shared array (two leading / trailing -inf pads
// make s-1, s-2 / s+1, s+2 unconditional); alpha for all t is parked in global scratch [T, S] per utterance and read back by
// the SAME thread in the beta sweep.  One __syncthreads per time step, all utterances in parallel.  Texts longer than 271
// tokens (2L + 1 > 544 states) run attn_ctc_long_kernel, the same recursions with 4 states per thread (2L + 1 <= 2049 for
// L <= FT_MAX_TEXT_LEN = 1024).
#include <math_constants.h>

#include "ft_internal.h"
#include "../../include/flowtron_b200.h"

namespace ft {

constexpr int CTC_THREADS = 544;            // >= 2 * 256 + 1 states (L <= 256), 17 warps
constexpr int CTC_NS_LONG = 4;              // states per thread of attn_ctc_long_kernel: 4 * 544 >= 2 * FT_MAX_TEXT_LEN + 1
static_assert(CTC_NS_LONG * CTC_THREADS >= 2 * FT_MAX_TEXT_LEN + 1, "CTC states must fit in one block");

__device__ __forceinline__ float lse3(float a, float b, float c) {
    const float m = fmaxf(a, fmaxf(b, c));
    if (m == -CUDART_INF_F) return -CUDART_INF_F;
    return m + logf(expf(a - m) + expf(b - m) + expf(c - m));
}

__global__ void __launch_bounds__(CTC_THREADS)
attn_ctc_kernel(const float* __restrict__ logprob, const int* __restrict__ in_lens, const int* __restrict__ out_lens, int T, int L,
                int reversed, float blank, float* __restrict__ cost, float* __restrict__ dlogprob, float* __restrict__ alpha_scratch) {
    extern __shared__ float sm[];
    const int b = blockIdx.x, tid = threadIdx.x;
    int K = in_lens[b], Tq = out_lens ? out_lens[b] : T;
    K = K < 0 ? 0 : (K > L ? L : K);
    Tq = Tq < 0 ? 0 : (Tq > T ? T : Tq);
    const int S = 2 * K + 1;
    float* lse = sm;                                   // [T]
    float* buf0 = sm + T;                              // [S + 4]  (2 pads each side)
    float* buf1 = buf0 + (2 * L + 1) + 4;
    __shared__ float s_nll;
    const float* x = logprob + static_cast<long long>(b) * T * L;
    float* dx = dlogprob + static_cast<long long>(b) * T * L;
    float* al = alpha_scratch + static_cast<long long>(b) * T * (2 * L + 1);
    const float NEG = -CUDART_INF_F;

    for (int i = tid; i < T * L; i += blockDim.x) dx[i] = 0.f;
    if (K == 0 || Tq == 0) { if (tid == 0) cost[b] = 0.f; return; }
    // ---- phase 0: lse[t] = log sum_c exp(logit[t,c]) over blank + K tokens (warp per row)
    {
        const int lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
        for (int t = warp; t < Tq; t += nw) {
            const float* row = x + static_cast<long long>(reversed ? Tq - 1 - t : t) * L;
            float m = blank;
            for (int k = lane; k < K; k += 32) m = fmaxf(m, row[k]);
#pragma unroll
            for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
            float s = lane == 0 ? expf(blank - m) : 0.f;
            for (int k = lane; k < K; k += 32) s += expf(row[k] - m);
#pragma unroll
            for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            if (lane == 0) lse[t] = m + logf(s);
        }
    }
    for (int i = tid; i < 2 * ((2 * L + 1) + 4); i += blockDim.x) buf0[i] = NEG;
    __syncthreads();
    const int s = tid;
    const bool live = s < S;
    const bool tok = (s & 1) != 0;                       // token state: label k = (s+1)/2, column k-1
    const int col = (s - 1) >> 1;
    auto logit = [&](int t) -> float {
        return tok ? x[static_cast<long long>(reversed ? Tq - 1 - t : t) * L + col] : blank;
    };
    // ---- phase 1: alpha
    float* prev = buf0; float* cur = buf1;
    float lp_t = live ? logit(0) - lse[0] : NEG;
    if (live) {
        const float a0 = (s <= 1) ? lp_t : NEG;
        prev[s + 2] = a0;
        al[s] = a0;
    }
    float nxt = (live && Tq > 1) ? logit(1) : 0.f;
    __syncthreads();
    for (int t = 1; t < Tq; ++t) {
        const float u = nxt;
        if (live && t + 1 < Tq) nxt = logit(t + 1);      // prefetch the next step's logit under this step's math
        if (live) {
            const float v2 = (tok && s >= 3) ? prev[s] : NEG;
            const float a = (u - lse[t]) + lse3(prev[s + 2], prev[s + 1], v2);
            cur[s + 2] = a;
            al[static_cast<long long>(t) * S + s] = a;
        }
        __syncthreads();
        float* tmp = prev; prev = cur; cur = tmp;
    }
    if (tid == 0) {
        const float a1 = prev[S - 1 + 2], a2 = S > 1 ? prev[S - 2 + 2] : NEG;
        const float m = fmaxf(a1, a2);
        s_nll = (m == NEG) ? CUDART_INF_F : -(m + logf(expf(a1 - m) + expf(a2 - m)));
    }
    __syncthreads();
    const float nll = s_nll;
    if (!(nll < CUDART_INF_F)) { if (tid == 0) cost[b] = 0.f; return; }       // zero_infinity: loss 0, gradient 0 (dx is zero)
    if (tid == 0) cost[b] = nll / static_cast<float>(K);
    // ---- phase 2: beta + gradient (time descending).  Pads: index s+2 -> s+1 at +3, s+2 at +4 (always in range, -inf beyond S)
    __syncthreads();
    for (int i = tid; i < 2 * ((2 * L + 1) + 4); i += blockDim.x) buf0[i] = NEG;
    __syncthreads();
    prev = buf0; cur = buf1;
    const float invK = 1.f / static_cast<float>(K);
    {
        const int t = Tq - 1;
        const float u = live ? logit(t) : 0.f;
        if (live) {
            const float lp = u - lse[t];
            const float be = (s >= S - 2) ? lp : NEG;
            prev[s + 2] = be;
            if (tok) {
                const float a = al[static_cast<long long>(t) * S + s];
                dx[static_cast<long long>(reversed ? Tq - 1 - t : t) * L + col] = (expf(lp) - expf(a + be + nll - lp)) * invK;
            }
        }
    }
    nxt = (live && Tq > 1) ? logit(Tq - 2) : 0.f;
    __syncthreads();
    for (int t = Tq - 2; t >= 0; --t) {
        const float u = nxt;
        if (live && t > 0) nxt = logit(t - 1);
        if (live) {
            const float lp = u - lse[t];
            const float v2 = (tok && s + 2 < S) ? prev[s + 4] : NEG;
            const float be = lp + lse3(prev[s + 2], prev[s + 3], v2);
            cur[s + 2] = be;
            if (tok) {
                const float a = al[static_cast<long long>(t) * S + s];
                dx[static_cast<long long>(reversed ? Tq - 1 - t : t) * L + col] = (expf(lp) - expf(a + be + nll - lp)) * invK;
            }
        }
        __syncthreads();
        float* tmp = prev; prev = cur; cur = tmp;
    }
}

// Texts past 271 tokens: the same recursions with NS states per thread (state s[j] = tid + j * CTC_THREADS).
template <int NS>
__global__ void __launch_bounds__(CTC_THREADS)
attn_ctc_long_kernel(const float* __restrict__ logprob, const int* __restrict__ in_lens, const int* __restrict__ out_lens, int T, int L,
                int reversed, float blank, float* __restrict__ cost, float* __restrict__ dlogprob, float* __restrict__ alpha_scratch) {
    extern __shared__ float sm[];
    const int b = blockIdx.x, tid = threadIdx.x;
    int K = in_lens[b], Tq = out_lens ? out_lens[b] : T;
    K = K < 0 ? 0 : (K > L ? L : K);
    Tq = Tq < 0 ? 0 : (Tq > T ? T : Tq);
    const int S = 2 * K + 1;
    float* lse = sm;                                   // [T]
    float* buf0 = sm + T;                              // [S + 4]  (2 pads each side)
    float* buf1 = buf0 + (2 * L + 1) + 4;
    __shared__ float s_nll;
    const float* x = logprob + static_cast<long long>(b) * T * L;
    float* dx = dlogprob + static_cast<long long>(b) * T * L;
    float* al = alpha_scratch + static_cast<long long>(b) * T * (2 * L + 1);
    const float NEG = -CUDART_INF_F;

    for (int i = tid; i < T * L; i += blockDim.x) dx[i] = 0.f;
    if (K == 0 || Tq == 0) { if (tid == 0) cost[b] = 0.f; return; }
    // ---- phase 0: lse[t] = log sum_c exp(logit[t,c]) over blank + K tokens (warp per row)
    {
        const int lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
        for (int t = warp; t < Tq; t += nw) {
            const float* row = x + static_cast<long long>(reversed ? Tq - 1 - t : t) * L;
            float m = blank;
            for (int k = lane; k < K; k += 32) m = fmaxf(m, row[k]);
#pragma unroll
            for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
            float s = lane == 0 ? expf(blank - m) : 0.f;
            for (int k = lane; k < K; k += 32) s += expf(row[k] - m);
#pragma unroll
            for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            if (lane == 0) lse[t] = m + logf(s);
        }
    }
    for (int i = tid; i < 2 * ((2 * L + 1) + 4); i += blockDim.x) buf0[i] = NEG;
    __syncthreads();
    // state s[j] = tid + j * CTC_THREADS
    bool live[NS], tok[NS];
    int col[NS];
#pragma unroll
    for (int j = 0; j < NS; ++j) {
        const int s = tid + j * CTC_THREADS;
        live[j] = s < S;
        tok[j] = (s & 1) != 0;                           // token state: label k = (s+1)/2, column k-1
        col[j] = (s - 1) >> 1;
    }
    auto logit = [&](int j, int t) -> float {
        return tok[j] ? x[static_cast<long long>(reversed ? Tq - 1 - t : t) * L + col[j]] : blank;
    };
    // ---- phase 1: alpha
    float* prev = buf0; float* cur = buf1;
    float nxt[NS];
#pragma unroll
    for (int j = 0; j < NS; ++j) {
        const int s = tid + j * CTC_THREADS;
        const float lp_t = live[j] ? logit(j, 0) - lse[0] : NEG;
        if (live[j]) {
            const float a0 = (s <= 1) ? lp_t : NEG;
            prev[s + 2] = a0;
            al[s] = a0;
        }
        nxt[j] = (live[j] && Tq > 1) ? logit(j, 1) : 0.f;
    }
    __syncthreads();
    for (int t = 1; t < Tq; ++t) {
#pragma unroll
        for (int j = 0; j < NS; ++j) {
            const int s = tid + j * CTC_THREADS;
            const float u = nxt[j];
            if (live[j] && t + 1 < Tq) nxt[j] = logit(j, t + 1);      // prefetch the next step's logit under this step's math
            if (live[j]) {
                const float v2 = (tok[j] && s >= 3) ? prev[s] : NEG;
                const float a = (u - lse[t]) + lse3(prev[s + 2], prev[s + 1], v2);
                cur[s + 2] = a;
                al[static_cast<long long>(t) * S + s] = a;
            }
        }
        __syncthreads();
        float* tmp = prev; prev = cur; cur = tmp;
    }
    if (tid == 0) {
        const float a1 = prev[S - 1 + 2], a2 = S > 1 ? prev[S - 2 + 2] : NEG;
        const float m = fmaxf(a1, a2);
        s_nll = (m == NEG) ? CUDART_INF_F : -(m + logf(expf(a1 - m) + expf(a2 - m)));
    }
    __syncthreads();
    const float nll = s_nll;
    if (!(nll < CUDART_INF_F)) { if (tid == 0) cost[b] = 0.f; return; }       // zero_infinity: loss 0, gradient 0 (dx is zero)
    if (tid == 0) cost[b] = nll / static_cast<float>(K);
    // ---- phase 2: beta + gradient (time descending).  Pads: index s+2 -> s+1 at +3, s+2 at +4 (always in range, -inf beyond S)
    __syncthreads();
    for (int i = tid; i < 2 * ((2 * L + 1) + 4); i += blockDim.x) buf0[i] = NEG;
    __syncthreads();
    prev = buf0; cur = buf1;
    const float invK = 1.f / static_cast<float>(K);
#pragma unroll
    for (int j = 0; j < NS; ++j) {
        const int s = tid + j * CTC_THREADS;
        const int t = Tq - 1;
        const float u = live[j] ? logit(j, t) : 0.f;
        if (live[j]) {
            const float lp = u - lse[t];
            const float be = (s >= S - 2) ? lp : NEG;
            prev[s + 2] = be;
            if (tok[j]) {
                const float a = al[static_cast<long long>(t) * S + s];
                dx[static_cast<long long>(reversed ? Tq - 1 - t : t) * L + col[j]] = (expf(lp) - expf(a + be + nll - lp)) * invK;
            }
        }
        nxt[j] = (live[j] && Tq > 1) ? logit(j, Tq - 2) : 0.f;
    }
    __syncthreads();
    for (int t = Tq - 2; t >= 0; --t) {
#pragma unroll
        for (int j = 0; j < NS; ++j) {
            const int s = tid + j * CTC_THREADS;
            const float u = nxt[j];
            if (live[j] && t > 0) nxt[j] = logit(j, t - 1);
            if (live[j]) {
                const float lp = u - lse[t];
                const float v2 = (tok[j] && s + 2 < S) ? prev[s + 4] : NEG;
                const float be = lp + lse3(prev[s + 2], prev[s + 3], v2);
                cur[s + 2] = be;
                if (tok[j]) {
                    const float a = al[static_cast<long long>(t) * S + s];
                    dx[static_cast<long long>(reversed ? Tq - 1 - t : t) * L + col[j]] = (expf(lp) - expf(a + be + nll - lp)) * invK;
                }
            }
        }
        __syncthreads();
        float* tmp = prev; prev = cur; cur = tmp;
    }
}

}  // namespace ft

extern "C" {

size_t ft_attn_ctc_scratch_bytes(int B, int T, int L) {
    return static_cast<size_t>(B) * T * (2 * static_cast<size_t>(L) + 1) * sizeof(float) + 256;
}

int ft_attn_ctc_loss(const float* attn_logprob, const int* in_lens, const int* out_lens, int B, int T, int L, int time_reversed,
                     float blank_logprob, float* cost, float* d_attn_logprob, void* scratch, void* stream) {
    using namespace ft;
    if (!attn_logprob || !in_lens || !cost || !d_attn_logprob || !scratch) return ft_set_error("ft_attn_ctc_loss: NULL argument");
    if (B <= 0 || T <= 0 || L <= 0) return 0;
    if (L > FT_MAX_TEXT_LEN) return ft_set_error("ft_attn_ctc_loss: L > FT_MAX_TEXT_LEN (1024) not supported");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t smem = sizeof(float) * (static_cast<size_t>(T) + 2 * ((2 * L + 1) + 4));
    if (smem > 200 * 1024) return ft_set_error("ft_attn_ctc_loss: T too large for the shared-memory lse table");
    auto kern = 2 * L + 1 <= CTC_THREADS ? attn_ctc_kernel : attn_ctc_long_kernel<CTC_NS_LONG>;
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    TimeScope ts("attn_ctc", T, B, L, st);
    kern<<<B, CTC_THREADS, smem, st>>>(attn_logprob, in_lens, out_lens, T, L, time_reversed, blank_logprob, cost, d_attn_logprob,
                                       static_cast<float*>(scratch));
    ft_count_launch(1);
    return ft_check_launch("attn_ctc_kernel");
}

}  // extern "C"
