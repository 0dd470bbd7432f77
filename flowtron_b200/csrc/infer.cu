// Autoregressive inference of one flow (AR_Step.infer, flowtron.py:775-828) as ONE persistent cooperative
// kernel: the per-frame chain  attention_lstm -> Q -> score/softmax/context -> lstm x2 -> dense x2 -> conv ->
// (z - b)/exp(log_s) -> gate  runs for all T frames without returning to the host (the reference issues ~25
// launches and one host sync per frame, and re-projects K/V every frame; here K/V are projected once).
//
// Design:
//   * every matrix-vector phase runs on the TENSOR CORES with the batch as the M = 16 rows of mma.sync.m16n8k16 and 8 weight
//     rows as N, so batches up to 16 cost what B = 1 costs.  Why warp-level mma.sync and not wgmma: a wgmma instruction
//     needs M >= 64 rows and its B operand in shared memory -- for an N <= 16 matvec that is 2.5-3 KB of shared-memory operand
//     reads (20+ clk) per K = 16 plus a shared-memory staging pass for 54 MB of weights per frame, while mma.sync takes the
//     weights straight from L2 into registers (one 16-byte load per lane per 32 k) with no padding rows.  The phase is bound
//     by L2 latency/bandwidth, not by tensor throughput, either way;
//   * weights are re-packed ONCE per call into the order the lanes consume them: [task (8 rows)][k-block of 32][row][32 k]
//     fp16, input and recurrent matrices of an LSTM fused along K (zero padded), so a warp instruction reads 512 contiguous
//     bytes and issues 8 of them back to back (4 KB in flight per warp, 16 warps per SM);
//   * a task's K range is split over the warps of a CTA (partial accumulators meet in shared memory), so all 16 warps of
//     every SM stream weights in every phase;
//   * a warp's share of the NEXT phase's weights is prefetched into registers before it waits for that phase's inputs (weights
//     do not depend on them), and so are the lane's biases, cell states and residual frame; scores run over all warps of the
//     grid (query rows staged in shared memory), then one (utterance, 64- or 128-channel slice) context item per CTA with the
//     softmax (+ prior posterior) recomputed per item; the gate logit of utterance b is computed by CTA b off the critical path;
//   * NO grid barriers (nine barriers and staging round trips per frame would take a large share of the frame): the
//     DATA IS THE FLAG.  Every exchanged activation lives in a ring of 3 frame slots pre-filled with a sentinel (0xFFFF per
//     fp16, 0xFFFFFFFF per fp32 word: bit patterns no conversion produces); producers store results with st.relaxed.gpu and
//     reset the same elements of the NEXT slot to the sentinel; consumers fetch the very words they need into shared memory
//     (cp.async.cg rounds) and re-fetch the packets that still contain a sentinel.  A hand-over costs one L2 store + one L2 load instead of
//     membar + atomic + poll + barrier + load.  A slot is reset two frames after its last reader: every read is followed by a
//     store that all CTAs consume within one frame, and one gpu-scope fence per thread per frame makes that chain formal
//     (tools/trace_infer.py prints the phase table).
// Same operand precision as the training kernels (fp16 operands, fp32 accumulate/state).
#include "ptx.cuh"
#include "ft_internal.h"
#include "../../include/flowtron_b200.h"

namespace ft {

constexpr int IH = 1024, IG = 4096;
constexpr int INF_THREADS = 512, INF_WARPS = 16;
constexpr int KMAX = 1664 + 1024;              // widest phase input: [d ; h0]
constexpr int KP = KMAX + 32;                  // activation row pitch (halfs): 5440 B = 64 mod 128 -> conflict-free 16-byte reads
constexpr int XPAD = 96;                       // the 80 mel channels of the attention LSTM's input, padded to 3 k-blocks
constexpr int LMAX = 256;                      // keys of the short-text kernels (one row of scores in registers per lane)
constexpr int LMAX_LONG = FT_MAX_TEXT_LEN;     // keys of the long-text kernels (the row staged in shared memory)

struct InferParams {
    int T, B, L, M, A, E, D;
    // packed fp16 weights ([task][k-block][8 rows][32 k]) and packed fp32 biases ([task][8])
    const __half *wA, *w0, *w1, *wq, *wd1, *wd2, *wc;
    const float *bA, *b0, *b1, *bd1, *bd2, *bc;
    const float *v, *wg, *bg;
    const float* Kp; const float* Vp;      // [L*B, A] projected once
    const float* residual;                 // [T,B,M] natural time order
    const float* prior;                    // [B,T,L] (row i used at frame i) or null
    // kForced: forced alignments (flowtron.py:585-588, 797), batch-major [B,Ta,L], each row in its flow's own generation
    // order; step i of utterance b reads keys l < in_lens[b] of row (b, i) while i < frame_lens[b]: every other weight is 0
    // whatever the buffer holds
    const float* attn_forced;
    float inv_temperature, gate_threshold;
    int has_gate;
    // keys l >= in_lens[b] take no part in the softmax; utterance b generates at most frame_lens[b] frames (null: L / T);
    // reversed: frame i reads residual row frame_lens[b] - 1 - i
    const int* in_lens;
    const int* frame_lens;
    int reversed;
    // outputs
    float* out;                            // [T,B,M]
    float* attn_out;                       // [T,B,L]
    int* n_frames;                         // [B]
    // state (global scratch).  Exchanged tensors are rings of 3 frame slots (slot = frame % 3) initialised to the sentinel
    // (slot 2 of the recurrent ones to zero: the state before frame 0); cell states are private to their producing lanes.
    float *cA, *c0, *c1;
    // (slot-0 pointers; slot k of every ring lies k * slot_bytes further: no dynamically indexed arrays in the parameter struct,
    //  which would move it to local memory)
    long long slot_bytes, rep_bytes;       // the tensors every CTA reads exist in NREP replicas (rep_bytes apart): see the header
    float *hA, *q, *e;                     // fp32: attention-LSTM output (gate), query, scores
    __half *hA16, *h016, *h116, *ctx16, *y116, *y216, *x16;   // fp16 [B][K]: what the next phases consume
    float* ctx32;                          // fp32 context (gate)
    uint32_t* alive;                       // [B] per slot: 1 while the sample keeps generating after this frame, 0 once stopped
    int* status;
    long long* trace;                      // debug: [T][32] clock64 stamps of CTA 0 (tools/trace_infer.py), or null
    int Ta;                                // rows per utterance of attn_forced
};

static long long* g_infer_trace = nullptr;
#define IT_TRACE(slot) do { if (p.trace && blockIdx.x == 0 && threadIdx.x == 0) p.trace[i * 32 + (slot)] = clock64(); } while (0)

constexpr uint32_t SENT = 0xFFFFFFFFu;
constexpr int NREP = 1;                        // replicas of the all-to-all exchanged tensors (CTA c reads replica c % NREP); more replicas
                                               // spread the reads of the same lines over more L2 slices but add stores
#define SL(ptr, k) (reinterpret_cast<decltype(ptr)>(reinterpret_cast<char*>(ptr) + (k)))     /* ring slot: k = slot index * slot_bytes */
__device__ __forceinline__ uint32_t ld_rlx_u32(const void* p) {
    uint32_t v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_rlx_u32(void* p, uint32_t v) { asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ void st_rlx_u16(void* p, uint16_t v) { asm volatile("st.relaxed.gpu.global.u16 [%0], %1;" ::"l"(p), "h"(v) : "memory"); }
__device__ __forceinline__ void st_rlx_f32(float* p, float v) { st_rlx_u32(p, __float_as_uint(v)); }
__device__ __forceinline__ void st_rlx_h(__half* p, float v) { st_rlx_u16(p, __half_as_ushort(__float2half_rn(v))); }
__device__ __forceinline__ void st_rlx_h2(__half* p, float a, float b) {
    const __half2 h = __floats2half2_rn(a, b);
    st_rlx_u32(p, *reinterpret_cast<const uint32_t*>(&h));
}
// any fp16 element of the 16-byte packet still the sentinel?
__device__ __forceinline__ bool sent16(const uint4& v) { return (__vcmpeq2(v.x, SENT) | __vcmpeq2(v.y, SENT) | __vcmpeq2(v.z, SENT) | __vcmpeq2(v.w, SENT)) != 0u; }
__device__ __forceinline__ float poll_f32(const float* g, int* status, int code) {
    uint32_t v = ld_rlx_u32(g);
    if (v == SENT) {
        const long long t0 = clock64();
        do {
            v = ld_rlx_u32(g);
            if (clock64() - t0 > FT_WATCHDOG_CYCLES) watchdog_fail(status, code);
        } while (v == SENT);
    }
    return __uint_as_float(v);
}

// Inputs of a phase: up to three ring-slot tensors [B, pitch] (written by the producing phases' epilogues on other SMs) -> shared
// memory rows of KP halfs at element columns cA / cB / cC (kF32: fp32 elements, rows of KP / 2 floats).  Round = every pending
// 16-byte packet of this thread is fetched with cp.async.cg (L2, no registers, all in flight at once), then checked in shared
// memory; packets that still hold a sentinel element are fetched again next round.  While a thread's FIRST packet is not valid
// it is the only one fetched (a failed round of everything moves B x K x 2 bytes per CTA for nothing: 11 MB over the grid at
// B = 16); the 512 first packets of a CTA sample all producers.  Batch rows >= B stay zero.  K, pitch, columns: multiples of
// the 16-byte packet.  Callers finish with __syncthreads().
// B <= 8 variant: a thread has at most ~3 packets, so plain index arithmetic is cheapest (the shift / mask set-up of the variant
// below costs more than it saves at such small batches).
template <bool kF32>
__device__ __forceinline__ void stage3_small(__half* sx, int cA, const void* srcA, int KA, int pitchA, int cB, const void* srcB, int KB, int pitchB,
                                             int cC, const void* srcC, int KC, int pitchC, int B, int* status) {
    constexpr int EPP = kF32 ? 4 : 8, EB = kF32 ? 4 : 2;          // elements per packet, bytes per element
    const int k8A = KA / EPP, k8B = KB / EPP, k8C = KC / EPP, totA = B * k8A, totB = totA + B * k8B, total = totB + B * k8C;
    uint32_t pend = 0;                                            // bit u: packet threadIdx.x + u * INF_THREADS not valid yet
    for (int u = 0, idx = threadIdx.x; idx < total; ++u, idx += INF_THREADS) pend |= 1u << u;
    long long t0 = 0;
    while (pend) {
        const uint32_t want = (pend & 1u) ? 1u : pend;
#pragma unroll 1
        for (int pass = 0; pass < 2; ++pass) {
            for (int u = 0, idx = threadIdx.x; idx < total; ++u, idx += INF_THREADS) {
                if (want >> u & 1u) {
                    const int q = idx < totA ? 0 : (idx < totB ? 1 : 2);
                    const int j = idx - (q == 0 ? 0 : (q == 1 ? totA : totB)), k8 = q == 0 ? k8A : (q == 1 ? k8B : k8C);
                    const int b = j / k8, i8 = j - b * k8;
                    uint8_t* dst = reinterpret_cast<uint8_t*>(sx) + b * (KP * 2) + (q == 0 ? cA : (q == 1 ? cB : cC)) * EB + 16 * i8;
                    if (pass == 0) {
                        const uint8_t* g = static_cast<const uint8_t*>(q == 0 ? srcA : (q == 1 ? srcB : srcC)) +
                                           static_cast<long long>(b) * (q == 0 ? pitchA : (q == 1 ? pitchB : pitchC)) * EB + 16 * i8;
                        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst)), "l"(g) : "memory");
                    } else {
                        const uint4 v = *reinterpret_cast<const uint4*>(dst);
                        const bool bad = kF32 ? (v.x == SENT || v.y == SENT || v.z == SENT || v.w == SENT) : sent16(v);
                        if (!bad) pend &= ~(1u << u);
                    }
                }
            }
            if (pass == 0) {
                asm volatile("cp.async.commit_group;" ::: "memory");
                asm volatile("cp.async.wait_group 0;" ::: "memory");
            }
        }
        if (pend) {
            if (t0 == 0) t0 = clock64();
            else if (clock64() - t0 > FT_WATCHDOG_CYCLES) watchdog_fail(status, 302);
        }
    }
}

template <bool kF32>
__device__ __forceinline__ void stage3_big(__half* sx, int cA, const void* srcA, int KA, int pitchA, int cB, const void* srcB, int KB, int pitchB,
                                           int cC, const void* srcC, int KC, int pitchC, int B, int* status) {
    constexpr int EPP = kF32 ? 4 : 8, EB = kF32 ? 4 : 2;          // elements per packet, bytes per element
    // thread -> (packet column i8 = tid & (kp - 1), row group tid / kp) per source, kp = packets per row rounded up to a power of
    // two (shift / mask arithmetic only: divisions would dominate the instruction issue of a round of the B = 16 loops); a source
    // needs `it` = ceil(B / (512 / kp)) iterations, pending bit = 4 * source + iteration (B <= 16, kp <= 512: it <= 4 when kp <= 128;
    // wider rows use up to 8 bits, sources are then limited to what fits in 32 bits)
    const void* src[3] = {srcA, srcB, srcC};
    const int col[3] = {cA, cB, cC}, pitch[3] = {pitchA, pitchB, pitchC};
    int k8[3] = {KA / EPP, KB / EPP, KC / EPP}, sh[3], nit[3], bit0[3];
    uint32_t pend = 0;
    int nb = 0;
#pragma unroll
    for (int q = 0; q < 3; ++q) {
        int kp = 1, s2 = 0;
        while (kp < k8[q]) { kp <<= 1; ++s2; }
        sh[q] = s2;
        const int rows_per = INF_THREADS >> s2;                   // rows covered per iteration
        nit[q] = k8[q] ? (B + rows_per - 1) / rows_per : 0;
        bit0[q] = nb;
        for (int it = 0; it < nit[q]; ++it) {
            const int b = (threadIdx.x >> s2) + it * rows_per, i8 = threadIdx.x & (kp - 1);
            if (b < B && i8 < k8[q]) pend |= 1u << (nb + it);
        }
        nb += nit[q];
    }
    long long t0 = 0;
    const uint32_t canary = pend & (0u - pend);                   // the thread's first packet: fetched alone until it is valid
    while (pend) {
        const uint32_t want = (pend & canary) ? canary : pend;
#pragma unroll 1
        for (int pass = 0; pass < 2; ++pass) {
#pragma unroll
            for (int q = 0; q < 3; ++q) {
                const int rows_per = INF_THREADS >> sh[q], i8 = threadIdx.x & ((1 << sh[q]) - 1);
                for (int it = 0; it < nit[q]; ++it) {
                    const uint32_t bit = 1u << (bit0[q] + it);
                    if (want & bit) {
                        const int b = (threadIdx.x >> sh[q]) + it * rows_per;
                        uint8_t* dst = reinterpret_cast<uint8_t*>(sx) + b * (KP * 2) + col[q] * EB + 16 * i8;
                        if (pass == 0) {
                            const uint8_t* g = static_cast<const uint8_t*>(src[q]) + static_cast<long long>(b) * pitch[q] * EB + 16 * i8;
                            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst)), "l"(g) : "memory");
                        } else {
                            const uint4 v = *reinterpret_cast<const uint4*>(dst);
                            const bool bad = kF32 ? (v.x == SENT || v.y == SENT || v.z == SENT || v.w == SENT) : sent16(v);
                            if (!bad) pend &= ~bit;
                        }
                    }
                }
            }
            if (pass == 0) {
                asm volatile("cp.async.commit_group;" ::: "memory");
                asm volatile("cp.async.wait_group 0;" ::: "memory");
            }
        }
        if (pend) {
            if (t0 == 0) t0 = clock64();
            else if (clock64() - t0 > FT_WATCHDOG_CYCLES) watchdog_fail(status, 302);
        }
    }
}

template <bool kF32, bool kBig>
__device__ __forceinline__ void stage3(__half* sx, int cA, const void* srcA, int KA, int pitchA, int cB, const void* srcB, int KB, int pitchB,
                                       int cC, const void* srcC, int KC, int pitchC, int B, int* status) {
    if (kBig) stage3_big<kF32>(sx, cA, srcA, KA, pitchA, cB, srcB, KB, pitchB, cC, srcC, KC, pitchC, B, status);
    else stage3_small<kF32>(sx, cA, srcA, KA, pitchA, cB, srcB, KB, pitchB, cC, srcC, KC, pitchC, B, status);
}

// d[16 batch x 8 rows] += sum over k-blocks [m0, m1) of  x[batch][k] * W[row][k].  Wt: this task's packed weights
// ([k-block][8 rows][32 k]); lane (n = lane/4, j = lane%4) owns row n and the 8 k values 8j..8j+7 of every block; the k order
// inside a block is a fixed permutation shared by both operands (any bijection is a valid contraction order):
// MMA step s in {0,1} of a block uses halfs 4s..4s+3 of the lane's chunk as its (k, k+1, k+8, k+9) slots.
template <bool kB16>
__device__ __forceinline__ void mv_partial(const __half* __restrict__ Wt, int m0, int m1, const __half* sx, int lane, float (&d)[4]) {
    constexpr int U = 10;
    const uint4* wp = reinterpret_cast<const uint4*>(Wt) + lane;             // block m: + 32 m   (lane = 4 n + j: 16 bytes each)
    const __half* a_lo = sx + (lane >> 2) * KP + 8 * (lane & 3);
    const __half* a_hi = a_lo + 8 * KP;
    for (int m = m0; m < m1; m += U) {
        uint4 w[U];
#pragma unroll
        for (int u = 0; u < U; ++u) w[u] = (m + u < m1) ? __ldg(wp + 32 * (m + u)) : make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
        for (int u = 0; u < U; ++u) {
            if (m + u < m1) {
                const uint4 lo = *reinterpret_cast<const uint4*>(a_lo + 32 * (m + u));
                uint4 hi = make_uint4(0u, 0u, 0u, 0u);
                if (kB16) hi = *reinterpret_cast<const uint4*>(a_hi + 32 * (m + u));
                mma16816(d, lo.x, hi.x, lo.y, hi.y, w[u].x, w[u].y);
                mma16816(d, lo.z, hi.z, lo.w, hi.w, w[u].z, w[u].w);
            }
        }
    }
}

// Weights do not depend on the activations a phase waits for: the first PFN k-blocks of a warp's share of the NEXT phase are
// loaded into registers BEFORE the grid barrier and land while the CTA waits instead of costing load round trips after it.
constexpr int PFN = 11;
struct Prefetch { uint4 w[PFN]; };
__device__ __forceinline__ void mv_prefetch(Prefetch& pf, const __half* __restrict__ W, int n_tasks, int nm, int S) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int tpc = INF_WARPS / S;
    const int tl = warp / S, split = warp - tl * S;
    const int task = blockIdx.x * tpc + tl;
    const int m0 = nm * split / S, m1 = nm * (split + 1) / S;
    const uint4* wp = reinterpret_cast<const uint4*>(W + static_cast<long long>(task) * nm * 256) + lane;
#pragma unroll
    for (int u = 0; u < PFN; ++u) pf.w[u] = (task < n_tasks && m0 + u < m1) ? __ldg(wp + 32 * (m0 + u)) : make_uint4(0u, 0u, 0u, 0u);
}

// One matrix-vector phase: n_tasks tasks of 8 rows, nm k-blocks, each task split over S warps of a CTA.  epi(task, d) is
// called by the task's first warp (all 32 lanes) with the complete accumulator fragment:
//   d[0], d[1] = batch row lane/4, rows 2j, 2j+1 of the task (j = lane%4);  d[2], d[3] = batch row lane/4 + 8, same rows.
// pf: the prefetched first PFN blocks of this warp's share of the FIRST pass (mv_prefetch with the same arguments).
template <bool kB16, class Epi>
__device__ __forceinline__ void mv_phase(const __half* __restrict__ W, int n_tasks, int nm, int S, float* spart, const __half* sx,
                                         const Prefetch& pf, Epi epi) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int tpc = INF_WARPS / S;
    const int tl = warp / S, split = warp - tl * S;
    bool first = true;
    for (int base = blockIdx.x * tpc; base < n_tasks; base += gridDim.x * tpc) {       // CTA-uniform trip count
        const int task = base + tl;
        float d[4] = {0.f, 0.f, 0.f, 0.f};
        if (task < n_tasks) {
            int m0 = nm * split / S;
            const int m1 = nm * (split + 1) / S;
            if (first) {
                const __half* a_lo = sx + (lane >> 2) * KP + 8 * (lane & 3);
                const __half* a_hi = a_lo + 8 * KP;
#pragma unroll
                for (int u = 0; u < PFN; ++u) {
                    if (m0 + u < m1) {
                        const uint4 lo = *reinterpret_cast<const uint4*>(a_lo + 32 * (m0 + u));
                        uint4 hi = make_uint4(0u, 0u, 0u, 0u);
                        if (kB16) hi = *reinterpret_cast<const uint4*>(a_hi + 32 * (m0 + u));
                        mma16816(d, lo.x, hi.x, lo.y, hi.y, pf.w[u].x, pf.w[u].y);
                        mma16816(d, lo.z, hi.z, lo.w, hi.w, pf.w[u].z, pf.w[u].w);
                    }
                }
                m0 = (m0 + PFN < m1) ? m0 + PFN : m1;
            }
            mv_partial<kB16>(W + static_cast<long long>(task) * nm * 256, m0, m1, sx, lane, d);
            if (S > 1) *reinterpret_cast<float4*>(spart + (warp * 32 + lane) * 4) = make_float4(d[0], d[1], d[2], d[3]);
        }
        if (S > 1) {
            __syncthreads();
            if (task < n_tasks && split == 0) {
                for (int s2 = 1; s2 < S; ++s2) {
                    const float4 v = *reinterpret_cast<const float4*>(spart + ((warp + s2) * 32 + lane) * 4);
                    d[0] += v.x; d[1] += v.y; d[2] += v.z; d[3] += v.w;
                }
            }
        }
        if (task < n_tasks && split == 0) epi(task, d, first);
        if (S > 1) __syncthreads();
        first = false;
    }
}

// LSTM cell for task = 2 units x 4 gates (rows i0,f0,g0,o0,i1,f1,g1,o1): lane j holds (i,f) [j even] or (g,o) [j odd] of unit j/2.
// h goes to ring slot `h16` (and `hnew`, fp32, when given); the same elements of the next slot are reset to the sentinel.
// cpre / bpre: the lane's cell states and biases, loaded before the phase waited for its inputs (first pass only).
__device__ __forceinline__ void lstm_epi(const InferParams& p, int task, float (&d)[4], const float* bias, float* c, float* hnew, float* hnew_next,
                                         __half* h16, __half* h16_next, bool first, const float (&cpre)[2], const float (&bpre)[2]) {
    const int lane = threadIdx.x & 31, j = lane & 3, r = lane >> 2;
    const float b0 = first ? bpre[0] : bias[task * 8 + 2 * j], b1 = first ? bpre[1] : bias[task * 8 + 2 * j + 1];
    float v[4] = {d[0] + b0, d[1] + b1, d[2] + b0, d[3] + b1};
    float o[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) o[i] = __shfl_xor_sync(0xffffffffu, v[i], 1);          // partner lane holds the other gate pair
    if ((j & 1) == 0) {
        const int u = 2 * task + (j >> 1);
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            const int b = r + 8 * half;
            if (b < p.B) {
                const float gi = sigmoid_f(v[2 * half]), gf = sigmoid_f(v[2 * half + 1]);
                const float gg = tanh_f(o[2 * half]), go = sigmoid_f(o[2 * half + 1]);
                const float cn = gf * (first ? cpre[half] : c[b * IH + u]) + gi * gg;
                const float h = go * tanh_f(cn);
#pragma unroll
                for (int rr = 0; rr < NREP; ++rr) {
                    st_rlx_h(SL(h16, rr * p.rep_bytes) + b * IH + u, h);
                    st_rlx_u16(SL(h16_next, rr * p.rep_bytes) + b * IH + u, 0xFFFFu);
                }
                if (hnew) { st_rlx_f32(hnew + b * IH + u, h); st_rlx_u32(hnew_next + b * IH + u, SENT); }
                c[b * IH + u] = cn;
            }
        }
    }
}
// the loads lstm_epi wants early: this lane's biases and cell states for the first task of its warp (S = 4: 4 tasks per CTA)
__device__ __forceinline__ void lstm_pre(const InferParams& p, const float* bias, const float* c, float (&cpre)[2], float (&bpre)[2]) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, j = lane & 3, r = lane >> 2;
    const int task = blockIdx.x * 4 + (warp >> 2);
    cpre[0] = cpre[1] = bpre[0] = bpre[1] = 0.f;
    if ((warp & 3) == 0 && task < IH / 2) {
        bpre[0] = bias[task * 8 + 2 * j]; bpre[1] = bias[task * 8 + 2 * j + 1];
        if ((j & 1) == 0) {
            const int u = 2 * task + (j >> 1);
            if (r < p.B) cpre[0] = c[r * IH + u];
            if (r + 8 < p.B) cpre[1] = c[(r + 8) * IH + u];
        }
    }
}

// Residual of frame i, utterance b, channel m.  Frames past the utterance's budget are never read (0: such frames are not
// emitted); a reversed flow reads its own frames back to front.
__device__ __forceinline__ float residual_at(const InferParams& p, int i, int b, int m) {
    const int n = p.frame_lens ? p.frame_lens[b] : p.T;
    if (i >= n) return 0.f;
    const int t = p.reversed ? n - 1 - i : i;
    return p.residual[(static_cast<long long>(t) * p.B + b) * p.M + m];
}

// kForced: the forced weights of utterance b at generation step i (row (b, i) of the batch-major buffer) and how many of its
// keys are read: in_lens[b], none once the row's frame budget is spent.
__device__ __forceinline__ const float* forced_row(const InferParams& p, int i, int b, int Lb, int& Lf) {
    Lf = (p.frame_lens && i >= p.frame_lens[b]) ? 0 : Lb;
    return p.attn_forced + (static_cast<long long>(b) * p.Ta + i) * p.L;
}

// Long texts (kLong, L > LMAX): warp 0 runs the same softmax / prior posterior / forced alignment over the row staged in
// shared memory, 32 keys per pass, instead of holding it in registers.  Each lane handles the same keys in the same order
// as the register path, so the two agree bit for bit where both apply.
template <bool kForced>
__device__ __forceinline__ void attn_row_long(const InferParams& p, float* se, int i, int b, long long cur, int Lb) {
    const int lane = threadIdx.x & 31;
    if (!kForced) {
        float mx = -INFINITY;
        for (int l = lane; l < p.L; l += 32) {
            const float x = l < Lb ? poll_f32(SL(p.e, cur) + b * p.L + l, p.status, 303) : -INFINITY;
            se[l] = x;
            mx = fmaxf(mx, x);
        }
#pragma unroll
        for (int o = 16; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        float sum = 0.f;
        for (int l = lane; l < p.L; l += 32) { const float x = l < Lb ? expf(se[l] - mx) : 0.f; se[l] = x; sum += x; }
#pragma unroll
        for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
        const float inv = 1.f / sum;
        for (int l = lane; l < p.L; l += 32) se[l] *= inv;
        if (p.prior) {
            float m2 = -INFINITY;
            for (int l = lane; l < Lb; l += 32) {
                const float pr = p.prior[(static_cast<long long>(b) * p.T + i) * p.L + l];
                const float x = logf(se[l] + 1e-20f) + logf(pr + 1e-20f);
                se[l] = x;
                m2 = fmaxf(m2, x);
            }
#pragma unroll
            for (int o = 16; o; o >>= 1) m2 = fmaxf(m2, __shfl_xor_sync(0xffffffffu, m2, o));
            float s2 = 0.f;
            for (int l = lane; l < p.L; l += 32) { const float x = l < Lb ? expf(se[l] - m2) : 0.f; se[l] = x; s2 += x; }
#pragma unroll
            for (int o = 16; o; o >>= 1) s2 += __shfl_xor_sync(0xffffffffu, s2, o);
            const float inv2 = 1.f / s2;
            for (int l = lane; l < p.L; l += 32) se[l] *= inv2;
        }
    } else {
        int Lf;
        const float* fr = forced_row(p, i, b, Lb, Lf);
        for (int l = lane; l < p.L; l += 32) se[l] = l < Lf ? fr[l] : 0.f;
    }
}

// Context of utterance b, channels [CW s, CW s + CW) (CW = 64 or 128), inside one CTA: warp 0 turns the scores into attention weights (softmax,
// prior posterior -- or the forced alignment), all 16 warps then take L/16 keys each (every V load of the CTA in flight at
// once), partial sums meet in shared memory.  Writes ctx (fp16 for lstm layer 0, fp32 for the gate) and, from slice 0, the
// attention weights.  (One CTA per utterance doing all 640 channels would pull 256 KB through one SM.)
template <int CW, bool kLong, bool kForced>
__device__ __forceinline__ void context_item(const InferParams& p, float* sf, int i, int b, int s, long long cur, long long nxt) {
    constexpr int NV = CW / 32;                                    // channels per lane
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float* se = sf; float* sp = sf + (kLong ? LMAX_LONG : LMAX);   // attn [LMAX or LMAX_LONG], partials [16 warps][CW]
    const int Lb = p.in_lens ? p.in_lens[b] : p.L;                 // key mask: tokens l >= Lb get weight 0 (as if L were Lb)
    if (kLong && warp == 0) {
        attn_row_long<kForced>(p, se, i, b, cur, Lb);
        if (s == 0)
            for (int l = lane; l < p.L; l += 32) p.attn_out[(static_cast<long long>(i) * p.B + b) * p.L + l] = se[l];
    } else if (warp == 0) {
        float w[8];
        if (!kForced) {                                           // softmax over L in registers: lane holds l = lane + 32 jj
            float mx = -INFINITY;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
                const int l = lane + 32 * jj;
                w[jj] = -INFINITY;
                if (l < Lb) w[jj] = poll_f32(SL(p.e, cur) + b * p.L + l, p.status, 303);
                mx = fmaxf(mx, w[jj]);
            }
#pragma unroll
            for (int o = 16; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
            float sum = 0.f;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) { w[jj] = (lane + 32 * jj < Lb) ? expf(w[jj] - mx) : 0.f; sum += w[jj]; }
#pragma unroll
            for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
            const float inv = 1.f / sum;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) w[jj] *= inv;
            if (p.prior) {
                float m2 = -INFINITY;
#pragma unroll
                for (int jj = 0; jj < 8; ++jj) {
                    const int l = lane + 32 * jj;
                    if (l < Lb) {
                        const float pr = p.prior[(static_cast<long long>(b) * p.T + i) * p.L + l];
                        w[jj] = logf(w[jj] + 1e-20f) + logf(pr + 1e-20f);
                        m2 = fmaxf(m2, w[jj]);
                    }
                }
#pragma unroll
                for (int o = 16; o; o >>= 1) m2 = fmaxf(m2, __shfl_xor_sync(0xffffffffu, m2, o));
                float s2 = 0.f;
#pragma unroll
                for (int jj = 0; jj < 8; ++jj) { w[jj] = (lane + 32 * jj < Lb) ? expf(w[jj] - m2) : 0.f; s2 += w[jj]; }
#pragma unroll
                for (int o = 16; o; o >>= 1) s2 += __shfl_xor_sync(0xffffffffu, s2, o);
                const float inv2 = 1.f / s2;
#pragma unroll
                for (int jj = 0; jj < 8; ++jj) w[jj] *= inv2;
            }
        } else {
            int Lf;
            const float* fr = forced_row(p, i, b, Lb, Lf) + lane;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) w[jj] = lane + 32 * jj < Lf ? __ldg(fr + 32 * jj) : 0.f;
        }
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
            const int l = lane + 32 * jj;
            if (l < p.L) { se[l] = w[jj]; if (s == 0) p.attn_out[(static_cast<long long>(i) * p.B + b) * p.L + l] = w[jj]; }
        }
    }
    __syncthreads();
    {   // warp w: keys w, w + 16, ...; lane: channels CW s + NV lane .. + NV - 1
        float acc[NV];
#pragma unroll
        for (int e = 0; e < NV; ++e) acc[e] = 0.f;
        constexpr int CU = 8;
        for (int l0 = warp; l0 < Lb; l0 += CU * INF_WARPS) {
            float v[CU][NV];
#pragma unroll
            for (int u = 0; u < CU; ++u) {
                const int l = l0 + u * INF_WARPS;
                const float* vr = p.Vp + (static_cast<long long>(l) * p.B + b) * p.A + CW * s + NV * lane;
                if (l < Lb) {
                    if (NV == 2) { const float2 t = *reinterpret_cast<const float2*>(vr); v[u][0] = t.x; v[u][1] = t.y; }
                    else { const float4 t = *reinterpret_cast<const float4*>(vr); v[u][0] = t.x; v[u][1] = t.y; v[u][NV - 2] = t.z; v[u][NV - 1] = t.w; }
                } else {
#pragma unroll
                    for (int e = 0; e < NV; ++e) v[u][e] = 0.f;
                }
            }
#pragma unroll
            for (int u = 0; u < CU; ++u) {
                const int l = l0 + u * INF_WARPS;
                const float w = l < Lb ? se[l] : 0.f;
#pragma unroll
                for (int e = 0; e < NV; ++e) acc[e] = fmaf(w, v[u][e], acc[e]);
            }
        }
#pragma unroll
        for (int e = 0; e < NV; ++e) sp[warp * CW + NV * lane + e] = acc[e];
    }
    __syncthreads();
    if (threadIdx.x < CW) {
        float c = 0.f;
#pragma unroll
        for (int w2 = 0; w2 < INF_WARPS; ++w2) c += sp[w2 * CW + threadIdx.x];
        const int o = b * p.A + CW * s + threadIdx.x;
#pragma unroll
        for (int rr = 0; rr < NREP; ++rr) { st_rlx_h(SL(p.ctx16, cur + rr * p.rep_bytes) + o, c); st_rlx_u16(SL(p.ctx16, nxt + rr * p.rep_bytes) + o, 0xFFFFu); }
        st_rlx_f32(SL(p.ctx32, cur) + o, c); st_rlx_u32(SL(p.ctx32, nxt) + o, SENT);
    }
    __syncthreads();
}

// kB16: batches of 9-16 utterances (the mma's upper 8 rows are live).  kLong: texts of LMAX < L <= LMAX_LONG keys
// (context_item's softmax over a shared-memory row).  kForced: attention weights given in attn_forced, so the query / score
// phases are not compiled in.
template <bool kB16, bool kLong, bool kForced>
__global__ void __launch_bounds__(INF_THREADS, 1)
infer_kernel(InferParams p) {
    extern __shared__ __align__(16) uint8_t smem_raw[];
    __half* sx = reinterpret_cast<__half*>(smem_raw);                          // [16][KP] fp16 activations of the phase
    float* spart = reinterpret_cast<float*>(sx + 16 * KP);                     // [16 warps][32 lanes][4] partial accumulators
    float* sf = spart + INF_WARPS * 128;                                       // attention scratch: attn[LMAX or LMAX_LONG], partials[16][128]
    __shared__ int s_alive[16], s_nfr[16];                                     // every CTA tracks every sample's gate state
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int i = threadIdx.x; i < 16 * KP; i += INF_THREADS) sx[i] = __float2half_rn(0.f);     // batch rows >= B: zero forever
    if (threadIdx.x < 16) { s_alive[threadIdx.x] = threadIdx.x < p.B; s_nfr[threadIdx.x] = 0; }
    __syncthreads();

    const int nmA = (XPAD + IH) / 32, nm0 = (p.D + IH) / 32, nm1 = 2 * IH / 32, nmd = IH / 32;
    const int gw = blockIdx.x * INF_WARPS + warp, nw = gridDim.x * INF_WARPS;
    // which phases this CTA has tasks in (CTAs without a task skip the phase's staging: nothing they read would be followed
    // by a store, and the ring-slot reuse argument relies on read -> store chains)
    const bool act_lstm = static_cast<int>(blockIdx.x) * 4 < IH / 2, act_q = static_cast<int>(blockIdx.x) < p.A / 8;
    const bool act_dense = static_cast<int>(blockIdx.x) < IH / 8, act_conv = static_cast<int>(blockIdx.x) < p.M / 4;
    // context work items: (utterance, channel slice); 64-channel slices unless that needs a second pass over the grid
    const bool wide_ctx = (p.A % 128 == 0) && p.B * (p.A / 64) > static_cast<int>(gridDim.x);
    Prefetch pf;
    mv_prefetch(pf, p.wA, IH / 2, nmA, 4);
    for (int i = 0; i < p.T; ++i) {
        const long long cur = (i % 3) * p.slot_bytes, prv = ((i + 2) % 3) * p.slot_bytes, nxt = ((i + 1) % 3) * p.slot_bytes;
        // all samples stopped?  (s_alive: the flags every CTA read before the previous frame's last phase -- identical everywhere)
        bool any = false;
        for (int b = 0; b < p.B; ++b) any |= (s_alive[b] != 0);
        if (!any) break;
        __threadfence();                         // one gpu-scope fence per thread per frame: see the header (slot reuse)
        float cpre[2], bpre[2];
        const long long cur_r = cur + (blockIdx.x % NREP) * p.rep_bytes, prv_r = prv + (blockIdx.x % NREP) * p.rep_bytes;   // this CTA's replica

        // ---- P1 attention_lstm step on the previous output frame (zeros at i == 0): x = [out_{i-1} (80 -> 96) ; hA_{i-1}]
        IT_TRACE(0);
        lstm_pre(p, p.bA, p.cA, cpre, bpre);
        if (act_lstm) {
            if (threadIdx.x < 16 * 2) *reinterpret_cast<uint4*>(sx + (threadIdx.x >> 1) * KP + p.M + 8 * (threadIdx.x & 1)) = make_uint4(0u, 0u, 0u, 0u);
            stage3<false, kB16>(sx, 0, SL(p.x16, prv_r), p.M, XPAD, XPAD, SL(p.hA16, prv_r), IH, IH, 0, nullptr, 0, 0, p.B, p.status);
        }
        __syncthreads();
        IT_TRACE(1);
        mv_phase<kB16>(p.wA, IH / 2, nmA, 4, spart, sx, pf, [&](int task, float (&d)[4], bool first) {
            lstm_epi(p, task, d, p.bA, p.cA, SL(p.hA, cur), SL(p.hA, nxt), SL(p.hA16, cur), SL(p.hA16, nxt), first, cpre, bpre);
        });
        if (kForced) mv_prefetch(pf, p.w0, IH / 2, nm0, 4); else mv_prefetch(pf, p.wq, p.A / 8, nmd, INF_WARPS);
        IT_TRACE(2);

        if (!kForced) {
            // ---- P2 query projection (no bias)
            if (act_q) stage3<false, kB16>(sx, 0, SL(p.hA16, cur_r), IH, IH, 0, nullptr, 0, 0, 0, nullptr, 0, 0, p.B, p.status);
            __syncthreads();
            IT_TRACE(4);
            mv_phase<kB16>(p.wq, p.A / 8, nmd, INF_WARPS, spart, sx, pf, [&](int task, float (&d)[4], bool) {
                const int j = lane & 3, r = lane >> 2;
#pragma unroll
                for (int half = 0; half < 2; ++half) {
                    const int b = r + 8 * half;
                    if (b < p.B && (half == 0 || kB16)) {
                        const int o = b * p.A + 8 * task + 2 * j;
#pragma unroll
                        for (int rr = 0; rr < NREP; ++rr) {
                            const long long ro = rr * p.rep_bytes;
                            st_rlx_f32(SL(p.q, cur + ro) + o, d[2 * half]); st_rlx_f32(SL(p.q, cur + ro) + o + 1, d[2 * half + 1]);
                            st_rlx_u32(SL(p.q, nxt + ro) + o, SENT); st_rlx_u32(SL(p.q, nxt + ro) + o + 1, SENT);
                        }
                    }
                }
            });
            mv_prefetch(pf, p.w0, IH / 2, nm0, 4);       // lstm layer 0's weights ride through the attention phases
            IT_TRACE(5);
            // ---- P3a scores e[b,l] = v . tanh(q[b] + K[l,b]) / temperature over ALL warps of the grid (no key mask in
            //      inference, flowtron.py:800-803); the query rows are staged in shared memory first (fp32, rows of KP/2 floats)
            if (static_cast<int>(blockIdx.x) * INF_WARPS < p.B * p.L)
                stage3<true, kB16>(sx, 0, SL(p.q, cur_r), p.A, p.A, 0, nullptr, 0, 0, 0, nullptr, 0, 0, p.B, p.status);
            __syncthreads();
            {
                const float* sq = reinterpret_cast<const float*>(sx);
                for (int t = gw; t < p.B * p.L; t += nw) {
                    const int b = t / p.L, l = t - b * p.L;
                    const float* kr = p.Kp + (static_cast<long long>(l) * p.B + b) * p.A;
                    const float* qr = sq + b * (KP / 2);
                    float sc = 0.f;
                    for (int a0 = 0; a0 < p.A; a0 += 256) {                      // 8 independent loads in flight
                        float kv[8];
#pragma unroll
                        for (int u = 0; u < 8; ++u) { const int a = a0 + 32 * u + lane; kv[u] = a < p.A ? kr[a] : 0.f; }
#pragma unroll
                        for (int u = 0; u < 8; ++u) { const int a = a0 + 32 * u + lane; if (a < p.A) sc = fmaf(p.v[a], tanh_f(qr[a] + kv[u]), sc); }
                    }
#pragma unroll
                    for (int o = 16; o; o >>= 1) sc += __shfl_xor_sync(0xffffffffu, sc, o);
                    if (lane == 0) { st_rlx_f32(SL(p.e, cur) + t, sc * p.inv_temperature); st_rlx_u32(SL(p.e, nxt) + t, SENT); }
                }
            }
            __syncthreads();                         // sx is re-staged below
            IT_TRACE(6);
        }
        // ---- P3b softmax + context, one (utterance, channel slice) item per CTA
        if (wide_ctx) { for (int it = blockIdx.x; it < p.B * (p.A / 128); it += gridDim.x) context_item<128, kLong, kForced>(p, sf, i, it / (p.A / 128), it % (p.A / 128), cur, nxt); }
        else          { for (int it = blockIdx.x; it < p.B * (p.A / 64); it += gridDim.x) context_item<64, kLong, kForced>(p, sf, i, it / (p.A / 64), it % (p.A / 64), cur, nxt); }
        IT_TRACE(7);
        // ---- P4 lstm layer 0 on [hA ; ctx ; h0_{i-1}]
        lstm_pre(p, p.b0, p.c0, cpre, bpre);
        if (act_lstm) stage3<false, kB16>(sx, 0, SL(p.hA16, cur_r), IH, IH, IH, SL(p.ctx16, cur_r), p.A, p.A, p.D, SL(p.h016, prv_r), IH, IH, p.B, p.status);
        __syncthreads();
        IT_TRACE(9);
        mv_phase<kB16>(p.w0, IH / 2, nm0, 4, spart, sx, pf, [&](int task, float (&d)[4], bool first) {
            lstm_epi(p, task, d, p.b0, p.c0, nullptr, nullptr, SL(p.h016, cur), SL(p.h016, nxt), first, cpre, bpre);
        });
        mv_prefetch(pf, p.w1, IH / 2, nm1, 4);
        IT_TRACE(10);
        if (static_cast<int>(blockIdx.x) < p.B) {
            // gate decision of utterance b = blockIdx.x for this frame, off the critical path (consumed before the conv phase):
            // w_g . [hA ; ctx] in fp32 (the frame that trips the gate IS emitted, flowtron.py:823-826)
            const int b = blockIdx.x;
            if (p.has_gate) {
                float sg = 0.f;
                for (int kk = threadIdx.x; kk < p.D; kk += INF_THREADS) {
                    const float x = kk < IH ? poll_f32(SL(p.hA, cur) + b * IH + kk, p.status, 304)
                                            : poll_f32(SL(p.ctx32, cur) + b * p.A + (kk - IH), p.status, 307);
                    sg = fmaf(p.wg[kk], x, sg);
                }
#pragma unroll
                for (int o = 16; o; o >>= 1) sg += __shfl_xor_sync(0xffffffffu, sg, o);
                if (lane == 0) sf[warp] = sg;
            }
            __syncthreads();
            if (threadIdx.x == 0) {
                const bool was_alive = s_alive[b] != 0;
                bool alive = was_alive;
                if (p.has_gate) {
                    float tot = 0.f;
                    for (int w2 = 0; w2 < INF_WARPS; ++w2) tot += sf[w2];
                    if (was_alive && sigmoid_f(tot + p.bg[0]) > p.gate_threshold) alive = false;
                }
                if (p.frame_lens && i + 1 >= p.frame_lens[b]) alive = false;       // the row's frame budget is spent
                if (was_alive) p.n_frames[b] = i + 1;
                st_rlx_u32(SL(p.alive, cur) + b, alive ? 1u : 0u);
                st_rlx_u32(SL(p.alive, nxt) + b, SENT);
            }
            __syncthreads();
        }
        // ---- P5 lstm layer 1 on [h0 ; h1_{i-1}]
        lstm_pre(p, p.b1, p.c1, cpre, bpre);
        if (act_lstm) stage3<false, kB16>(sx, 0, SL(p.h016, cur_r), IH, IH, IH, SL(p.h116, prv_r), IH, IH, 0, nullptr, 0, 0, p.B, p.status);
        __syncthreads();
        IT_TRACE(12);
        mv_phase<kB16>(p.w1, IH / 2, nm1, 4, spart, sx, pf, [&](int task, float (&d)[4], bool first) {
            lstm_epi(p, task, d, p.b1, p.c1, nullptr, nullptr, SL(p.h116, cur), SL(p.h116, nxt), first, cpre, bpre);
        });
        mv_prefetch(pf, p.wd1, IH / 8, nmd, INF_WARPS);
        IT_TRACE(13);
        // ---- P6/P7 dense layers (tanh)
        auto dense = [&](const __half* W, const float* bias, const __half* x, __half* y, __half* y_next) {
            const int j = lane & 3;
            const float pb0 = act_dense ? bias[blockIdx.x * 8 + 2 * j] : 0.f, pb1 = act_dense ? bias[blockIdx.x * 8 + 2 * j + 1] : 0.f;   // S = 16: task == CTA
            if (act_dense) stage3<false, kB16>(sx, 0, x, IH, IH, 0, nullptr, 0, 0, 0, nullptr, 0, 0, p.B, p.status);
            __syncthreads();
            mv_phase<kB16>(W, IH / 8, nmd, INF_WARPS, spart, sx, pf, [&](int task, float (&d)[4], bool first) {
                const int r = lane >> 2;
                const float b0 = first ? pb0 : bias[task * 8 + 2 * j], b1 = first ? pb1 : bias[task * 8 + 2 * j + 1];
#pragma unroll
                for (int half = 0; half < 2; ++half) {
                    const int b = r + 8 * half;
                    if (b < p.B && (half == 0 || kB16)) {
                        const int o = b * IH + 8 * task + 2 * j;
                        const float y0 = tanh_f(d[2 * half] + b0), y1 = tanh_f(d[2 * half + 1] + b1);
#pragma unroll
                        for (int rr = 0; rr < NREP; ++rr) { st_rlx_h2(SL(y, rr * p.rep_bytes) + o, y0, y1); st_rlx_u32(SL(y_next, rr * p.rep_bytes) + o, SENT); }
                    }
                }
            });
        };
        dense(p.wd1, p.bd1, SL(p.h116, cur_r), SL(p.y116, cur), SL(p.y116, nxt));
        mv_prefetch(pf, p.wd2, IH / 8, nmd, INF_WARPS);
        IT_TRACE(15);
        dense(p.wd2, p.bd2, SL(p.y116, cur_r), SL(p.y216, cur), SL(p.y216, nxt));
        mv_prefetch(pf, p.wc, p.M / 4, nmd, INF_WARPS);
        IT_TRACE(17);
        // ---- P8 conv + inverse affine: out = (residual - b) / exp(log_s); task rows = (log_s, b) of 4 consecutive channels
        if (threadIdx.x < p.B) {
            // the samples' gate decisions of this frame (written by CTA b after lstm layer 0, long ago)
            const float fl = poll_f32(reinterpret_cast<const float*>(SL(p.alive, cur)) + threadIdx.x, p.status, 306);
            if (s_alive[threadIdx.x]) s_nfr[threadIdx.x] = i + 1;
            s_alive[threadIdx.x] = __float_as_uint(fl) != 0u;
        }
        float rpre[2] = {0.f, 0.f}, cb0 = 0.f, cb1 = 0.f;                 // residual and conv biases of this lane's outputs (S = 16: task == CTA)
        if (act_conv && warp == 0) {
            const int j = lane & 3, r = lane >> 2, m = 4 * blockIdx.x + j;
            cb0 = p.bc[blockIdx.x * 8 + 2 * j]; cb1 = p.bc[blockIdx.x * 8 + 2 * j + 1];
            if (r < p.B) rpre[0] = residual_at(p, i, r, m);
            if (kB16 && r + 8 < p.B) rpre[1] = residual_at(p, i, r + 8, m);
        }
        if (act_conv) stage3<false, kB16>(sx, 0, SL(p.y216, cur_r), IH, IH, 0, nullptr, 0, 0, 0, nullptr, 0, 0, p.B, p.status);
        __syncthreads();
        IT_TRACE(18);
        mv_phase<kB16>(p.wc, p.M / 4, nmd, INF_WARPS, spart, sx, pf, [&](int task, float (&d)[4], bool first) {
            const int j = lane & 3, r = lane >> 2;
            const int m = 4 * task + j;
            const float bl = first ? cb0 : p.bc[task * 8 + 2 * j], bb = first ? cb1 : p.bc[task * 8 + 2 * j + 1];
#pragma unroll
            for (int half = 0; half < 2; ++half) {
                const int b = r + 8 * half;
                if (b < p.B && (half == 0 || kB16)) {
                    const long long ro = (static_cast<long long>(i) * p.B + b) * p.M;
                    // a sample that stopped at an earlier frame emits zeros; the frame that trips the gate is still emitted
                    // (s_nfr: updated above from the flags every CTA read)
                    const bool emit = (i < s_nfr[b]);
                    const float res = first ? rpre[half] : residual_at(p, i, b, m);
                    const float val = (res - (d[2 * half + 1] + bb)) / expf(d[2 * half] + bl);
                    p.out[ro + m] = emit ? val : 0.f;
#pragma unroll
                    for (int rr = 0; rr < NREP; ++rr) {
                        st_rlx_h(SL(p.x16, cur + rr * p.rep_bytes) + b * XPAD + m, val);
                        st_rlx_u16(SL(p.x16, nxt + rr * p.rep_bytes) + b * XPAD + m, 0xFFFFu);
                    }
                }
            }
        });
        mv_prefetch(pf, p.wA, IH / 2, nmA, 4);           // next frame's attention LSTM
        IT_TRACE(19);
    }
}

// ------------------------------------------------------------------------------------------------ weight packing
// dst[task][m][n][kk] (fp16) <- W[row(task, n)][32 m + kk] over the virtual K = [A part (Ka real columns, padded to Kap) ; B part]
//   kind 0: LSTM      row = (n % 4) * 1024 + 2 task + n / 4        (rows i0,f0,g0,o0,i1,f1,g1,o1)
//   kind 1: dense     row = 8 task + n
//   kind 2: conv pair row = (n % 2) * M + 4 task + n / 2           (log_s, b of 4 consecutive channels)
// bias_dst[task][n] = b1[row] (+ b2[row])
__global__ void pack_weights_kernel(__half* __restrict__ dst, float* __restrict__ bias_dst, const float* __restrict__ WA, int Ka, int Kap,
                                    const float* __restrict__ WB, int Kb, const float* __restrict__ b1, const float* __restrict__ b2,
                                    int n_tasks, int nm, int kind, int M) {
    const long long total = static_cast<long long>(n_tasks) * nm * 256;
    for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int kk = static_cast<int>(i & 31), n = static_cast<int>((i >> 5) & 7);
        const long long tm = i >> 8;
        const int m = static_cast<int>(tm % nm), task = static_cast<int>(tm / nm);
        const int row = kind == 0 ? (n & 3) * IH + 2 * task + (n >> 2) : kind == 1 ? 8 * task + n : (n & 1) * M + 4 * task + (n >> 1);
        const int k = 32 * m + kk;
        float v = 0.f;
        if (k < Kap) { if (k < Ka) v = WA[static_cast<long long>(row) * Ka + k]; }
        else if (WB && k - Kap < Kb) v = WB[static_cast<long long>(row) * Kb + (k - Kap)];
        dst[i] = __float2half_rn(v);
        if (m == 0 && kk == 0 && bias_dst) bias_dst[task * 8 + n] = (b1 ? b1[row] : 0.f) + (b2 ? b2[row] : 0.f);
    }
}

static int pack(__half* dst, float* bias_dst, const float* WA, int Ka, int Kap, const float* WB, int Kb, const float* b1, const float* b2,
                int n_tasks, int nm, int kind, int M, cudaStream_t st) {
    const long long total = static_cast<long long>(n_tasks) * nm * 256;
    int blocks = static_cast<int>((total + 255) / 256);
    if (blocks > 132 * 16) blocks = 132 * 16;     // 16 CTAs per SM of an H100 SXM
    pack_weights_kernel<<<blocks, 256, 0, st>>>(dst, bias_dst, WA, Ka, Kap, WB, Kb, b1, b2, n_tasks, nm, kind, M);
    ft_count_launch(1);
    return ft_check_launch("pack_weights_kernel");
}

// ------------------------------------------------------------------------------------------------ host
struct InferScratch {
    __half *wA, *w0, *w1, *wq, *wd1, *wd2, *wc;
    float *bA, *b0, *b1, *bd1, *bd2, *bc;
    uint16_t *wk, *wv, *text16;
    float *Kp, *Vp, *state;
    int* ints;
    size_t state_floats, total;
};

static InferScratch plan_infer(const FtArStepDesc& d, uint8_t* base) {
    InferScratch s;
    Workspace ws; ws.base = base;
    const int M = d.n_mel, A = d.n_attn, E = d.n_text, D = IH + A;
    auto w16 = [&](size_t tasks, size_t nm) { return ws.get<__half>(tasks * nm * 256); };
    s.wA = w16(IH / 2, (XPAD + IH) / 32);
    s.w0 = w16(IH / 2, (D + IH) / 32);
    s.w1 = w16(IH / 2, 2 * IH / 32);
    s.wq = w16(A / 8, IH / 32);
    s.wd1 = w16(IH / 8, IH / 32);
    s.wd2 = w16(IH / 8, IH / 32);
    s.wc = w16(M / 4, IH / 32);
    s.bA = ws.get<float>(IG); s.b0 = ws.get<float>(IG); s.b1 = ws.get<float>(IG);
    s.bd1 = ws.get<float>(IH); s.bd2 = ws.get<float>(IH); s.bc = ws.get<float>(2 * M);
    s.wk = ws.get<uint16_t>(size_t(A) * E);
    s.wv = ws.get<uint16_t>(size_t(A) * E);
    s.text16 = ws.get<uint16_t>(size_t(d.L) * d.B * E);
    s.Kp = ws.get<float>(size_t(d.L) * d.B * A);
    s.Vp = ws.get<float>(size_t(d.L) * d.B * A);
    // state: cell states cA, c0, c1 (3 x B*IH fp32), then the exchange rings (3 frame slots each): hA32 (B*IH), q (B*A), e (B*L),
    // alive (B) as 32-bit words; hA16, h016, h116, y116, y216 (B*IH), d16 (B*D), x16 (B*96) as fp16 (counted in floats, each piece
    // padded to 16 bytes)
    s.state_floats = size_t(d.B) * 3 * IH + 3 * (size_t(d.B) * (IH + A + d.L + 1) + 24) +
                     3 * 8 /* NREP */ * ((size_t(d.B) * (5 * IH + A + XPAD) + 1) / 2 + size_t(d.B) * A + 40) + 256;
    s.state = ws.get<float>(s.state_floats);
    s.ints = nullptr;
    s.total = ws.off;
    return s;
}

// After the persistent kernel: row (i, b) with i >= n_frames[b] gets zero attention weights; a reversed flow's emitted frames
// are flipped within n_frames[b] (frame j <-> n - 1 - j, swapped by the CTA that owns the lower of the two rows).
__global__ void infer_finish_kernel(float* __restrict__ out, float* __restrict__ attn_out, const int* __restrict__ n_frames,
                                    int T, int B, int M, int L, int reversed) {
    for (int row = blockIdx.x; row < T * B; row += gridDim.x) {
        const int i = row / B, b = row - i * B, n = n_frames[b];
        if (i >= n) {
            for (int l = threadIdx.x; l < L; l += blockDim.x) attn_out[static_cast<long long>(row) * L + l] = 0.f;
        } else if (reversed && 2 * i + 1 < n) {
            float* x = out + static_cast<long long>(row) * M;
            float* y = out + (static_cast<long long>(n - 1 - i) * B + b) * M;
            for (int m = threadIdx.x; m < M; m += blockDim.x) { const float t = x[m]; x[m] = y[m]; y[m] = t; }
        }
    }
}

static int infer_impl(const FtArStepDesc* d, const FtArStepWeights* w, const float* residual, const float* text,
                      const int* in_lens, const int* frame_lens, const float* attn_prior, const float* attn_forced, int Ta,
                      float gate_threshold, float* out, float* attn_out, int* n_frames, void* scratch, void* stream) {
    if (!d || !w || !residual || !text || !out || !attn_out || !n_frames || !scratch) return ft_set_error("ft_ar_step_infer: NULL argument");
    if (attn_forced && (Ta < 1 || (!frame_lens && Ta < d->T)))
        return ft_set_error("ft_ar_step_infer: attn_forced must cover every frame budget (Ta >= max frame_lens)");
    if (d->n_hidden != IH) return ft_set_error("infer: n_hidden must be 1024");
    if (d->L > LMAX_LONG) return ft_set_error("infer: L > FT_MAX_TEXT_LEN (1024) not supported");
    if (d->B > 16) return ft_set_error("infer: batch > 16 per call not supported (run the batch in slices of 16)");
    if (d->n_mel > XPAD || d->n_mel % 8 || d->n_attn % 64 || d->n_text % 8 || d->n_attn > 4 * INF_THREADS)
        return ft_set_error("infer: n_mel <= 96 and %8, n_attn %64 and <= 2048, n_text %8 required");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    InferScratch s = plan_infer(*d, static_cast<uint8_t*>(scratch));
    const int M = d->n_mel, A = d->n_attn, E = d->n_text, D = IH + A, B = d->B;
    const long long RL = static_cast<long long>(d->L) * B;
    // weights in consumption order (fp16), LSTM input + recurrent matrices fused along K, biases pre-added
    FT_TRY(pack(s.wA, s.bA, w->attn_lstm_w_ih, M, XPAD, w->attn_lstm_w_hh, IH, w->attn_lstm_b_ih, w->attn_lstm_b_hh, IH / 2, (XPAD + IH) / 32, 0, M, st));
    FT_TRY(pack(s.w0, s.b0, w->lstm_w_ih0, D, D, w->lstm_w_hh0, IH, w->lstm_b_ih0, w->lstm_b_hh0, IH / 2, (D + IH) / 32, 0, M, st));
    FT_TRY(pack(s.w1, s.b1, w->lstm_w_ih1, IH, IH, w->lstm_w_hh1, IH, w->lstm_b_ih1, w->lstm_b_hh1, IH / 2, 2 * IH / 32, 0, M, st));
    FT_TRY(pack(s.wq, nullptr, w->att_query, IH, IH, nullptr, 0, nullptr, nullptr, A / 8, IH / 32, 1, M, st));
    FT_TRY(pack(s.wd1, s.bd1, w->dense_w0, IH, IH, nullptr, 0, w->dense_b0, nullptr, IH / 8, IH / 32, 1, M, st));
    FT_TRY(pack(s.wd2, s.bd2, w->dense_w1, IH, IH, nullptr, 0, w->dense_b1, nullptr, IH / 8, IH / 32, 1, M, st));
    FT_TRY(pack(s.wc, s.bc, w->conv_w, IH, IH, nullptr, 0, w->conv_b, nullptr, M / 4, IH / 32, 2, M, st));
    FT_TRY(launch_cast(w->att_key, 2, s.wk, 0, static_cast<long long>(A) * E, st));
    FT_TRY(launch_cast(w->att_value, 2, s.wv, 0, static_cast<long long>(A) * E, st));
    FT_TRY(launch_cast(text, 2, s.text16, 0, RL * E, st));
    // K / V projections once per utterance (the reference recomputes them every frame, flowtron.py:568-570)
    FT_TRY(gemm_nt(st, RL, A, E, s.text16, E, s.wk, E, s.Kp, A));
    FT_TRY(gemm_nt(st, RL, A, E, s.text16, E, s.wv, E, s.Vp, A));
    FT_CU(cudaMemsetAsync(out, 0, sizeof(float) * d->T * B * M, st), "infer");
    FT_CU(cudaMemsetAsync(attn_out, 0, sizeof(float) * d->T * B * d->L, st), "infer");
    FT_CU(cudaMemsetAsync(n_frames, 0, sizeof(int) * B, st), "infer");

    InferParams p;
    p.T = d->T; p.B = B; p.L = d->L; p.M = M; p.A = A; p.E = E; p.D = D;
    p.wA = s.wA; p.w0 = s.w0; p.w1 = s.w1; p.wq = s.wq; p.wd1 = s.wd1; p.wd2 = s.wd2; p.wc = s.wc;
    p.bA = s.bA; p.b0 = s.b0; p.b1 = s.b1; p.bd1 = s.bd1; p.bd2 = s.bd2; p.bc = s.bc;
    p.v = w->att_v; p.wg = w->gate_w; p.bg = w->gate_b;
    p.Kp = s.Kp; p.Vp = s.Vp; p.residual = residual; p.prior = d->has_prior ? attn_prior : nullptr;
    p.attn_forced = attn_forced; p.Ta = Ta;
    p.in_lens = in_lens; p.frame_lens = frame_lens; p.reversed = d->reversed ? 1 : 0;
    p.inv_temperature = 1.0f / d->temperature; p.gate_threshold = gate_threshold;
    p.has_gate = d->has_gate && w->gate_w;
    p.out = out; p.attn_out = attn_out; p.n_frames = n_frames;
    float* f = s.state;
    auto take = [&](size_t n) { float* r = f; f += (n + 3) & ~size_t(3); return r; };     // 16-byte aligned pieces (16-byte polls)
    const size_t BH = static_cast<size_t>(B) * IH;
    auto take16 = [&](size_t n) { return reinterpret_cast<__half*>(take((n + 1) / 2)); };
    p.cA = take(BH); p.c0 = take(BH); p.c1 = take(BH);
    float* ring0 = f;                                            // everything from here on is exchanged: sentinel-filled
    // slot layout: [replicated tensors] x NREP, then the tensors only a few CTAs read
    p.hA16 = take16(BH); p.h016 = take16(BH); p.h116 = take16(BH); p.y116 = take16(BH); p.y216 = take16(BH);
    p.ctx16 = take16(static_cast<size_t>(B) * A); p.x16 = take16(static_cast<size_t>(B) * XPAD); p.q = take(static_cast<size_t>(B) * A);
    p.rep_bytes = (f - ring0) * static_cast<long long>(sizeof(float));
    f = ring0 + NREP * (f - ring0);
    p.hA = take(BH); p.e = take(static_cast<size_t>(B) * d->L); p.ctx32 = take(static_cast<size_t>(B) * A);
    p.alive = reinterpret_cast<uint32_t*>(take(B));
    p.slot_bytes = (f - ring0) * static_cast<long long>(sizeof(float));
    f = ring0 + 3 * (f - ring0);
    if (static_cast<size_t>(f - s.state) > s.state_floats) return ft_set_error("infer: scratch plan overflow");
    FT_CU(cudaMemsetAsync(s.state, 0, (ring0 - s.state) * sizeof(float), st), "infer");
    FT_CU(cudaMemsetAsync(ring0, 0xFF, (f - ring0) * sizeof(float), st), "infer");
    // the state before frame 0 (slot 2 = frame -1): zero hidden states and a zero previous output frame
    for (int rr = 0; rr < NREP; ++rr) {
        auto slot2 = [&](void* ptr) { return static_cast<char*>(ptr) + 2 * p.slot_bytes + rr * p.rep_bytes; };
        FT_CU(cudaMemsetAsync(slot2(p.hA16), 0, BH * 2, st), "infer");
        FT_CU(cudaMemsetAsync(slot2(p.h016), 0, BH * 2, st), "infer");
        FT_CU(cudaMemsetAsync(slot2(p.h116), 0, BH * 2, st), "infer");
        FT_CU(cudaMemsetAsync(slot2(p.x16), 0, static_cast<size_t>(B) * XPAD * 2, st), "infer");
    }
    p.status = ft_status_word();
    p.trace = g_infer_trace;
    int dev = 0, sms = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (sms < B) return ft_set_error("infer: fewer SMs than utterances");
    const bool long_text = d->L > LMAX;
    using Kernel = void (*)(InferParams);
    static const Kernel kernels[2][2][2] = {{{infer_kernel<false, false, false>, infer_kernel<false, false, true>}, {infer_kernel<false, true, false>, infer_kernel<false, true, true>}},
                                            {{infer_kernel<true, false, false>, infer_kernel<true, false, true>}, {infer_kernel<true, true, false>, infer_kernel<true, true, true>}}};
    void* fn = reinterpret_cast<void*>(kernels[B > 8][long_text][attn_forced != nullptr]);
    const int smem = 16 * KP * 2 + INF_WARPS * 128 * 4 + ((long_text ? LMAX_LONG : LMAX) + INF_WARPS * 128 + 64) * 4;
    cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    TimeScope ts("infer", d->T, B, d->L, st);
    void* args[] = {&p};
    cudaError_t e = cudaLaunchCooperativeKernel(fn, dim3(sms), dim3(INF_THREADS), args, smem, st);
    if (e != cudaSuccess) return ft_set_error(cudaGetErrorString(e));
    ft_count_launch(1);
    if (ft_check_launch("infer_kernel") != 0) return -1;
    // frames are generated back to front by a reversed flow: flip each row within its own n_frames (the B = 1 flip), and clear
    // the attention rows of frames a stopped utterance computed but did not emit
    const int rows = d->T * B;
    if (rows <= 0) return 0;
    infer_finish_kernel<<<rows < 4096 ? rows : 4096, 128, 0, st>>>(out, attn_out, n_frames, d->T, B, M, d->L, p.reversed);
    ft_count_launch(1);
    return ft_check_launch("infer_finish_kernel");
}


}  // namespace ft

extern "C" {

/* debug: device buffer [T][32] receiving clock64 stamps of CTA 0 of the next ft_ar_step_infer launches (NULL disables) */
void ft_debug_set_infer_trace(long long* buf) { ft::g_infer_trace = buf; }

size_t ft_ar_step_infer_scratch_bytes(const FtArStepDesc* d) { return ft::plan_infer(*d, nullptr).total + 256; }

int ft_ar_step_infer(const FtArStepDesc* d, const FtArStepWeights* w, const float* residual, const float* text, const int* in_lens,
                     const int* frame_lens, const float* attn_prior, const float* attn_forced, int Ta, float gate_threshold,
                     float* out, float* attn_out, int* n_frames, void* scratch, void* stream) {
    return ft::infer_impl(d, w, residual, text, in_lens, frame_lens, attn_prior, attn_forced, Ta, gate_threshold, out, attn_out,
                          n_frames, scratch, stream);
}

}  // extern "C"
