// Persistent LSTM recurrence kernels for sm_90a (forward and BPTT), hidden size 1024.
//
// Reference semantics: torch.nn.LSTM as used by AR_Step (flowtron.py:654-655, 671-695): gate order
// i,f,g,o; c' = s(f) c + s(i) tanh(g); h' = s(o) tanh(c'); zero initial state; outputs are 0 at
// t >= len (pack_padded/pad_packed).  The input projection W_ih x + b_ih + b_hh is a plain GEMM done
// beforehand (gemm.cu); these kernels run the T-step dependency chain without returning to the host.
//
// Forward (lstm_fwd_kernel), one cooperative launch of 64 CTAs (U = 16 hidden units each), or of 128 CTAs (U = 8) for
// the attention LSTM with its input projection folded in:
//   * CTA c owns hidden units [Uc, Uc+U): its 4U rows of W_hh (4 gates x U units, fp16, 128 / 64 KB) are
//     TMA-loaded once and stay resident in shared memory as the wgmma A operand (M = 64, 4U real rows).
//   * every step: h_{t-1} ([B,1024] fp16, read straight out of the layer's output tensor) arrives through
//     TWO 3-D TMA loads (8 K-chunks each, box {64 elems, B rows, 8 chunks}: the smem image is chunk-major
//     SWIZZLE_128B K-major tiles, the wgmma B operand with N = B rounded up to 16 / 32); the CTA's one
//     warpgroup accumulates the 4U gate pre-activations in registers, hands them through shared memory to
//     the thread that owns each (batch row, unit pair), adds the input projection, applies the cell in fp32
//     (cell state lives in registers for the whole sequence), store h_t (fp16) and publish ONE release per
//     CTA into a per-(step, chunk) counter; consumers poll the 16 counters in parallel (one lane each),
//     fence the async proxy, and issue the next loads.  gates / c for the backward pass are stored AFTER
//     the release so they stay off the critical path.
// Backward (lstm_bwd4_kernel), 16 clusters of 4 CTAs: dh_{t-1} = dG_t W_hh split over the four gates, the pointwise
//   LSTM backward in the epilogue; dG ([B,4096] fp16, loss-scaled) is written once and reused by the wgrad/dgrad GEMMs.
//   lstm_bwd_flat_kernel is the same computation without clusters (partial sums exchanged through L2) for the layer
//   pipeline's chunks, whose two concurrent launches do not fit on an H100 as 4-CTA clusters.
//
// Every kernel here takes at most 32 batch rows per launch (one 32-row wgmma tile); larger batches are split by the caller.
//
// Warp roles: warps 0-3 form one warpgroup that issues the wgmma of a step and runs the cell epilogue on the
// accumulator; warp 4 is the TMA producer.  Loads are issued as few multi-chunk 3-D boxes: issuing 16 2-D loads
// serially from one thread puts the issue time on the recurrence's critical path.
#include <type_traits>

#include "ptx.cuh"
#include "ft_internal.h"

namespace ft {

#define FT_TRACE(p, t, slot) do { if ((p).trace && blockIdx.x == 0) (p).trace[(t) * 16 + (slot)] = clock64(); } while (0)
static long long* g_lstm_trace = nullptr;      // set through ft_debug_set_lstm_trace
void set_lstm_trace(long long* p) { g_lstm_trace = p; }

constexpr int LH = 1024;
constexpr int LG = 4 * LH;
constexpr int KCH = 64;                        // K elements per 128-byte chunk (16-bit operands)
constexpr int LSTM_THREADS = 160;              // warps 0-3: one warpgroup (wgmma + cell epilogue), warp 4: TMA producer
constexpr int EPI_THREADS = 128;
constexpr int PRODUCER_WARP = 4;

__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}
__device__ __forceinline__ void epi_bar() { asm volatile("bar.sync 1, 128;" ::: "memory"); }   // the 4 warps of the warpgroup
__device__ __forceinline__ void st_dsmem_f2(uint32_t cluster_addr, float a, float b) {
    asm volatile("st.shared::cluster.v2.f32 [%0], {%1, %2};" ::"r"(cluster_addr), "f"(a), "f"(b) : "memory");
}

// `nch` K chunks (64 elements each, SWIZZLE_128B K-major) of D[64 x N] += A * B^T on the warpgroup; the first instruction
// overwrites the accumulator when `zero` is set.
template <int N>
__device__ __forceinline__ void mma_chunks(float* acc, uint64_t da, uint64_t db, int nch, uint64_t a_chunk, uint64_t b_chunk, bool zero) {
    for (int c = 0; c < nch; ++c) {
#pragma unroll
        for (int k = 0; k < KCH / 16; ++k) wgmma_k<N, FMT_F16, 0, 0>(acc, da + 2 * k, db + 2 * k, (zero && c == 0 && k == 0) ? 0u : 1u);
        da += a_chunk;
        db += b_chunk;
    }
}

// ------------------------------------------------------------------------------------------- forward
constexpr int FWD_NCH = LH / KCH;                  // 16 chunks / step
constexpr int FWD_GS = 8;                          // K chunks per TMA group: 2 groups per step
// FWD_UNITS hidden units per CTA: 8 -> 128 CTAs (whole GPU, lowest latency), 16 -> 64 CTAs (two such launches on two
// streams -- the layer pipeline's two layers, or two half batches -- run concurrently and hide each other's exchange latency)

struct LstmFwdParams {
    int T, B, Bbox;
    const float* xproj;        // [T*B, 4096] input projection + both biases (null when the projection is folded in)
    const float* b_ih; const float* b_hh;   // folded-projection form only: the two bias vectors [4096]
    const int* lens;           // [B] or null
    __half* hseq; long long ldh;   // [T*B, ldh] output (fp16), also the recurrent exchange buffer
    __half* gates;             // [T*B, 4096] post-activation i,f,g,o (fp16) or null
    float* cstate;             // [T*B, 1024] or null
    float* h32; long long ldh32;   // optional fp32 copy of h (or null)
    int* flags;                // [T * 16], zeroed by the launcher
    int* status;
    long long* trace;          // optional [T][8] clock64 stamps of CTA 0 (debug/profiling), or null
};

// ------------------------------------------------------------------------------------------- backward, split-K cluster
// 64 CTAs in 16 clusters of 4.  Cluster c owns hidden units [64c, 64c+64); rank r reduces over gate r's quarter of
// the contraction (K = 1024 of 4096):  partial_r[b, u] = sum_{k in gate r} dG_{t+1}[b, k] W_hh[k, u].
//   * the rank's W_hh^T block [64 units x 1024] (fp16, 128 KB) is resident; per step it streams only ITS quarter of
//     dG_{t+1} (B x 1024 fp16 = 64 KB at B=32 instead of all 256 KB broadcast to every CTA);
//   * partial sums (fp32 [B, 64]) go to shared memory; a cluster-scope mbarrier (4 remote arrives) publishes them;
//     each rank then finishes 16 of the 64 units, reading the 3 other partials over DSMEM;
//   * then the pointwise LSTM backward, the dG_t stores and one release flag per 64-column chunk of dG_t.
constexpr int BWD_NCH = LG / KCH;                                                                  // 64 dG chunks / step
constexpr int B4_CTAS = 64, B4_CLUSTER = 4, B4_UNITS = 64, B4_OWN = 16, B4_NCH = LH / KCH;     // 16 chunks / step / rank
constexpr int B4_W_BYTES = B4_NCH * B4_UNITS * 128;                                               // 128 KB
constexpr int B4_UP = 36;                                                                          // received-slice row pitch (floats): 32 batch columns, 16-byte aligned rows
constexpr int B4_XCHG_FLOATS = 2 * 4 * 16 * B4_UP;                                                 // [2 parities][4 source ranks][16 units][B4_UP]

// The kernel runs steps [t0, t1) of the sequence, highest step first: the whole sequence in one launch (t0 = 0, t1 = T), or
// one chunk of the layer pipeline (ar_step.cu), resuming dc*f from `dc_carry` ([B,1024] fp32, written by the chunk above) and
// dG_{t1} from the dG tensor.  Flags are indexed relative to t0, mbarrier phases are counted over the steps that have a
// recurrent term.
struct LstmBwdChunkParams {
    int T, B, Bbox;
    const float* dh_ext; long long ldd;   // [T*B, ldd] gradient w.r.t. the layer outputs (fp32, loss-scaled)
    const __half* gates;       // [T*B, 4096] saved i,f,g,o
    const float* cstate;       // [T*B, 1024] saved c_t
    const int* lens;
    __half* dG;                // [T*B, 4096] out: (loss-scaled) gradient w.r.t. gate pre-activations (fp16, saturating)
    int* flags;
    int* status;
    long long* trace;
    int t0, t1;                // steps [t0, t1); flags: [(t1 - t0) * 64] ints (flat kernel: [(t1 - t0) * 128]), zeroed by the launcher
    float* dc_carry;           // [B, 1024]
    float* xchg;               // flat kernel: partial-sum ring [2 parities][16 groups][4 ranks][B][64] fp32
};

// ------------------------------------------------------------------------------------------- backward, split-K flat
// lstm_bwd_flat_kernel: the same work split with no cluster -- CTA 4g + r plays rank r of group g.  A plain cooperative launch
// of 64 CTAs places them on any 64 SMs, so the layer pipeline's two BPTT chunks fit side by side; 4-CTA clusters must each fit
// in one GPC, and 32 of them (two chunks) do not reliably fit on an H100 (DESIGN §4.2).  The DSMEM exchange becomes an L2 one:
// each rank stores its whole fp32 partial [B, 64] to the ring `xchg` and releases one flag per (step, group, rank) (flags
// [(t1 - t0) * 64, (t1 - t0) * 128)); the rank that finishes units [64g + 16r, +16) acquires the other three ranks' flags and
// reads its slice of all four partials from L2, summing them in the cluster kernel's order (bit-identical results).
template <bool kFlat>
__device__ __forceinline__ void lstm_bwd_body(const CUtensorMap& tmWT, const CUtensorMap& tmG, const LstmBwdChunkParams& p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const int slot_bytes = p.Bbox * 128;
    uint8_t* sA = smem;                                          // [16 chunks][Bbox rows][128 B]
    uint8_t* sW = smem + B4_NCH * slot_bytes;                    // [16 chunks][64 rows][128 B]
    float* sPart = reinterpret_cast<float*>(sW + B4_W_BYTES);    // received partial sums: [2 parities][4 source ranks][16 units][B4_UP]
    uint64_t* bars = reinterpret_cast<uint64_t*>(sPart + (kFlat ? 0 : B4_XCHG_FLOATS));
    uint64_t* full = bars;                       // [2]
    uint64_t* wbar = bars + 2;
    uint64_t* part_bar = bars + 4;               // [2] : 4 cluster-scope arrivals each

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int rank = kFlat ? static_cast<int>(blockIdx.x % B4_CLUSTER) : static_cast<int>(cluster_ctarank());
    const int cl = blockIdx.x / B4_CLUSTER;
    constexpr int GS = 8, NG = B4_NCH / GS;
    const bool top = p.t1 == p.T;                                // the chunk that holds the last time step
    const int t_hi = top ? p.T - 2 : p.t1 - 1;                   // highest step that has a recurrent term (dG_{t+1} exists)

    if (warp == PRODUCER_WARP && lane == 0) {
        tma_prefetch_desc(&tmWT);
        tma_prefetch_desc(&tmG);
        mbar_init(&full[0], 1); mbar_init(&full[1], 1);
        mbar_init(wbar, 1);
        if (!kFlat) { mbar_init(&part_bar[0], B4_CLUSTER); mbar_init(&part_bar[1], B4_CLUSTER); }
        fence_mbar_init();
    }
    if (kFlat) __syncthreads();
    else cluster_sync_all();                                     // every rank's barriers exist before any remote arrive

    if (warp == PRODUCER_WARP) {
        if (lane == 0) {
            mbar_expect_tx(wbar, B4_W_BYTES);
            for (int kc = 0; kc < B4_NCH; ++kc)                  // W_hh^T rows [64c, 64c+64), columns of gate `rank`
                tma_load_2d(sW + kc * (B4_UNITS * 128), &tmWT, wbar, rank * LH + kc * KCH, B4_UNITS * cl);
        }
        for (int t = t_hi; t >= p.t0; --t) {
            // gate `rank` of dG_{t+1}: 16 chunks, each released by the 4 ranks of one cluster.  dG_{t1} (first step of a
            // lower chunk) was written by the previous launch on this stream: nothing to wait for.
            if (t + 1 < p.t1 && lane < B4_NCH)
                wait_flag_ge(&p.flags[(t + 1 - p.t0) * BWD_NCH + rank * B4_NCH + lane], 4, p.status, 232);
            __syncwarp();
            if (elect_one()) {
                FT_TRACE(p, t, 0);
                fence_proxy_async_global();
#pragma unroll
                for (int g = 0; g < NG; ++g) {
                    mbar_expect_tx(&full[g], GS * slot_bytes);
                    tma_load_3d(sA + g * GS * slot_bytes, &tmG, &full[g], 0, (t + 1) * p.B, rank * B4_NCH + g * GS);
                }
            }
            __syncwarp();
        }
    } else {
        const int q = warp;
        const int et = threadIdx.x;
        // swapped operands (see lstm_fwd_kernel): A = resident W_hh^T block (M = 64 units), B = dG_{t+1} quarter (N = 32 >= Bbox
        // batch rows; the rows beyond Bbox are read from the next chunk and never used)
        const uint64_t da_base = wgmma_desc(smem_u32(sW), 16, 1024), db_base = wgmma_desc(smem_u32(sA), 16, 1024);
        const uint64_t a_chunk = (B4_UNITS * 128) >> 4, b_chunk = static_cast<uint64_t>(slot_bytes >> 4);
        mbar_wait(wbar, 0, p.status, 233);
        const int n_items = p.B * 4;                              // (batch row, quad of units) over this rank's 16 final units
        const int u0 = B4_UNITS * cl + B4_OWN * rank;
        const int item = et;
        const bool has_item = item < n_items;
        const int ib = item >> 2, uq = item & 3;
        float dcs[4] = {0.f, 0.f, 0.f, 0.f};
        const int len = (has_item && p.lens) ? p.lens[ib] : p.T;
        if (!top && has_item) {                                   // resume dc * f carried out of the chunk above
            const float4 cv = *reinterpret_cast<const float4*>(p.dc_carry + static_cast<long long>(ib) * LH + B4_UNITS * cl + B4_OWN * rank + 4 * uq);
            dcs[0] = cv.x; dcs[1] = cv.y; dcs[2] = cv.z; dcs[3] = cv.w;
        }
        int step = 0;
        for (int t = p.t1 - 1; t >= p.t0; --t, ++step) {
            const int rs = top ? step - 1 : step;                 // index of this step among the steps with a recurrent term
            float dh[4], ct[4], cp[4];
            __half2 gt[4][2];
            const bool valid = has_item && (t < len);
            const long long r = static_cast<long long>(t) * p.B + ib;
            const int uo = u0 + 4 * uq;
            if (valid) {
                const float4 v = __ldg(reinterpret_cast<const float4*>(p.dh_ext + r * p.ldd + uo));
                dh[0] = v.x; dh[1] = v.y; dh[2] = v.z; dh[3] = v.w;
                const float4 cc = __ldg(reinterpret_cast<const float4*>(p.cstate + r * LH + uo));
                ct[0] = cc.x; ct[1] = cc.y; ct[2] = cc.z; ct[3] = cc.w;
                float4 pp = make_float4(0.f, 0.f, 0.f, 0.f);
                if (t > 0) pp = __ldg(reinterpret_cast<const float4*>(p.cstate + (r - p.B) * LH + uo));
                cp[0] = pp.x; cp[1] = pp.y; cp[2] = pp.z; cp[3] = pp.w;
#pragma unroll
                for (int g = 0; g < 4; ++g) {
                    const uint2 pk = __ldg(reinterpret_cast<const uint2*>(p.gates + r * LG + g * LH + uo));
                    *reinterpret_cast<uint2*>(&gt[g][0]) = pk;
                }
            }
            float rec[4] = {0.f, 0.f, 0.f, 0.f};                 // recurrent part of dh_t: sum over the 4 ranks' partials
            if (rs >= 0) {
                const int par = rs & 1;
                // Accumulator rows = the cluster block's 64 units: quadrant q (= this warp) holds units [16q, 16q+16), exactly the
                // units rank q finishes.  PUSH: each warp sends its 16 x Bbox partial sums straight into rank q's shared memory
                // (slot of THIS source rank, [unit][batch] rows of 32 floats), then one release-arrive per rank publishes them
                // and every rank sums four LOCAL slices -- one DSMEM hop on the critical path (r1 pulled: arrive, then a remote
                // load round trip), and all four epilogue warps move data instead of one.
                {
                    float acc[16];
#pragma unroll
                    for (int g = 0; g < NG; ++g) {
                        mbar_wait(&full[g], rs & 1, p.status, 234);
                        if (g == 0 && et == 0) FT_TRACE(p, t, 2);
                        wgmma_fence_acc<16>(acc);
                        wgmma_fence();
                        mma_chunks<32>(acc, da_base + g * GS * a_chunk, db_base + g * GS * b_chunk, GS, a_chunk, b_chunk, g == 0);
                        wgmma_commit();
                    }
                    wgmma_wait<0>();
                    wgmma_fence_acc<16>(acc);
                    if (et == 0) FT_TRACE(p, t, 4);
                    // fragment rows 16 q + lane / 4 (+ 8) = units of rank q, columns = batch rows 8 j + 2 (lane % 4) (+ 1)
                    const int u = lane >> 2, b = 2 * (lane & 3);
                    if (kFlat) {                                  // the whole partial [B][64] to this rank's ring slot
                        float* dst = p.xchg + static_cast<long long>((par * 16 + cl) * 4 + rank) * p.B * B4_UNITS + 16 * q + u;
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            const int bj = 8 * j + b;
                            if (bj < p.B) { dst[bj * B4_UNITS] = acc[4 * j]; dst[bj * B4_UNITS + 8] = acc[4 * j + 2]; }
                            if (bj + 1 < p.B) { dst[(bj + 1) * B4_UNITS] = acc[4 * j + 1]; dst[(bj + 1) * B4_UNITS + 8] = acc[4 * j + 3]; }
                        }
                    } else {
                        const uint32_t dst = mapa_shared(smem_u32(sPart) + static_cast<uint32_t>((((par * 4 + rank) * 16 + u) * B4_UP + b) * 4), q);
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            st_dsmem_f2(dst + 32 * j, acc[4 * j], acc[4 * j + 1]);
                            st_dsmem_f2(dst + (8 * B4_UP + 8 * j) * 4, acc[4 * j + 2], acc[4 * j + 3]);
                        }
                    }
                }
                if (et == 64) FT_TRACE(p, t, 6);
                epi_bar();
                if (kFlat) {
                    // publish this rank's partial (gpu-scope release, cumulative over the CTA's stores ordered by the barrier),
                    // then acquire the three other ranks' flags in parallel; the ring is read from L2 (ld.cg) below
                    int* xf = p.flags + static_cast<long long>(p.t1 - p.t0 + t - p.t0) * BWD_NCH + cl * B4_CLUSTER;
                    if (et == 0) red_release_add(&xf[rank], 1);
                    if (et < B4_CLUSTER && et != rank) wait_flag_ge(&xf[et], 1, p.status, 237);
                    epi_bar();
                } else {
                    // publish: one release-arrive on every rank's barrier, issued by 4 different threads so the four
                    // cluster-scope releases overlap (issued serially by one thread they would queue behind each other)
                    if (et < B4_CLUSTER) mbar_arrive_cluster(mapa_shared(smem_u32(&part_bar[par]), et));
                    mbar_wait_cluster(&part_bar[par], (rs >> 1) & 1, p.status, 236);
                }
                if (et == 0) FT_TRACE(p, t, 1);               // all partials visible
                if (has_item) {
#pragma unroll
                    for (int rr = 0; rr < B4_CLUSTER; ++rr) {
                        if (kFlat) {
                            const float4 v = __ldcg(reinterpret_cast<const float4*>(
                                p.xchg + (static_cast<long long>((par * 16 + cl) * 4 + rr) * p.B + ib) * B4_UNITS + B4_OWN * rank + 4 * uq));
                            rec[0] += v.x; rec[1] += v.y; rec[2] += v.z; rec[3] += v.w;
                        } else {
                            const float* src = sPart + ((par * 4 + rr) * 16 + 4 * uq) * B4_UP + ib;
#pragma unroll
                            for (int j = 0; j < 4; ++j) rec[j] += src[j * B4_UP];
                        }
                    }
                }
            }
            if (has_item) {
                __half2 out[4][2];
                if (valid) {
#pragma unroll
                    for (int j2 = 0; j2 < 2; ++j2) {
                        float da[4][2];
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int j = 2 * j2 + e;
                            const float gi = e ? __high2float(gt[0][j2]) : __low2float(gt[0][j2]);
                            const float gf = e ? __high2float(gt[1][j2]) : __low2float(gt[1][j2]);
                            const float gg = e ? __high2float(gt[2][j2]) : __low2float(gt[2][j2]);
                            const float go = e ? __high2float(gt[3][j2]) : __low2float(gt[3][j2]);
                            const float dht = dh[j] + rec[j];
                            const float tc = tanh_f(ct[j]);
                            const float dc = dcs[j] + dht * go * (1.f - tc * tc);
                            da[3][e] = dht * tc * go * (1.f - go);
                            da[0][e] = dc * gg * gi * (1.f - gi);
                            da[2][e] = dc * gi * (1.f - gg * gg);
                            da[1][e] = dc * cp[j] * gf * (1.f - gf);
                            dcs[j] = dc * gf;
                        }
#pragma unroll
                        for (int g = 0; g < 4; ++g)
                            out[g][j2] = __floats2half2_rn(fminf(fmaxf(da[g][0], -65504.f), 65504.f),
                                                           fminf(fmaxf(da[g][1], -65504.f), 65504.f));
                    }
                } else {
#pragma unroll
                    for (int g = 0; g < 4; ++g) { out[g][0] = __floats2half2_rn(0.f, 0.f); out[g][1] = out[g][0]; }
#pragma unroll
                    for (int j = 0; j < 4; ++j) dcs[j] = 0.f;
                }
#pragma unroll
                for (int g = 0; g < 4; ++g)
                    *reinterpret_cast<uint2*>(p.dG + r * LG + g * LH + uo) = *reinterpret_cast<uint2*>(&out[g][0]);
            }
            epi_bar();                                            // every dG_t store of this CTA precedes the releases
            if (et == 0) FT_TRACE(p, t, 5);
            if (et < 4) red_release_add(&p.flags[(t - p.t0) * BWD_NCH + et * 16 + cl], 1);     // chunk (gate et, units 64cl..) : 4 ranks
            if (et == 0) FT_TRACE(p, t, 7);
        }
        if (p.t0 > 0 && has_item)                                 // hand dc * f to the chunk below
            *reinterpret_cast<float4*>(p.dc_carry + static_cast<long long>(ib) * LH + B4_UNITS * cl + B4_OWN * rank + 4 * uq) =
                make_float4(dcs[0], dcs[1], dcs[2], dcs[3]);
    }
    if (!kFlat) cluster_sync_all();                              // nobody exits while a peer may still read its partials
}

__global__ void __launch_bounds__(LSTM_THREADS, 1)
lstm_bwd4_kernel(const __grid_constant__ CUtensorMap tmWT, const __grid_constant__ CUtensorMap tmG, LstmBwdChunkParams p) {
    lstm_bwd_body<false>(tmWT, tmG, p);
}

__global__ void __launch_bounds__(LSTM_THREADS, 1)
lstm_bwd_flat_kernel(const __grid_constant__ CUtensorMap tmWT, const __grid_constant__ CUtensorMap tmG, LstmBwdChunkParams p) {
    lstm_bwd_body<true>(tmWT, tmG, p);
}


// ------------------------------------------------------------------------------------------- forward kernel
// Steps [t0, t1) of the recurrence: the whole sequence in one launch (t0 = 0, t1 = T), or one chunk of the layer pipeline
// (ar_step.cu: two layers run as two 64-CTA kernels on two streams, chunk by chunk, one chunk apart), resuming h from the
// output tensor (row t0-1) and c from the saved cell states.  Flags are indexed relative to t0, mbarrier phases relative to
// the first step that has a recurrent term.
struct LstmFwdChunkParams : LstmFwdParams {
    int t0, t1;                // steps [t0, t1); flags: [(t1 - t0) * 16] ints, zeroed by the launcher
};

// kXIn: the layer's INPUT projection is folded into the recurrent contraction (narrow inputs: the attention LSTM's 80 mel
// channels).  The step's input row block x_t ([B, <=128] fp16, zero-filled by TMA beyond the real width) is loaded next to
// h_{t-1} as XCH more K chunks, W_ih's slice sits next to W_hh's in shared memory, and b_ih + b_hh are added in the epilogue:
// no [T*B, 4096] fp32 projection tensor is written (one GEMM + 524 MB write + 524 MB read per flow at B=32, T=1000).
// Requires x_0 == 0 (the teacher-forcing shift guarantees it): step 0 has no contraction at all.
constexpr int XCH = 2;                                           // extra K chunks (128 input channels max)

template <int FWD_UNITS, bool kXIn>
__global__ void __launch_bounds__(LSTM_THREADS, 1)
lstm_fwd_kernel(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmH, const __grid_constant__ CUtensorMap tmWx,
                const __grid_constant__ CUtensorMap tmX, LstmFwdChunkParams p) {
    constexpr int FWD_NG = FWD_NCH / FWD_GS;                     // TMA groups per step
    constexpr int NCHT = FWD_NCH + (kXIn ? XCH : 0);             // K chunks per step: h (16) [+ x (2)]
    constexpr int A_SLOTS = FWD_NCH + (kXIn ? 2 * XCH : 0);      // x_t is double-buffered: it is prefetched one step ahead
    constexpr int FWD_N = 4 * FWD_UNITS, FWD_W_BYTES = NCHT * FWD_N * 128, FWD_PROD = KCH / FWD_UNITS;
    constexpr int AP = FWD_N + 1;                                // accumulator staging pitch
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const int slot_bytes = p.Bbox * 128;
    uint8_t* sA = smem;                                          // [16 (+2x2) chunks][Bbox rows][128 B]: h chunks, then two x buffers
    uint8_t* sW = smem + A_SLOTS * slot_bytes;
    float* sAcc = reinterpret_cast<float*>(sW + FWD_W_BYTES);    // [32 rows][AP]
    uint64_t* bars = reinterpret_cast<uint64_t*>(sAcc + ((32 * AP + 1) & ~1));
    uint64_t* full = bars;                       // [FWD_NG] (<= 16)
    uint64_t* wbar = bars + 16;
    uint64_t* xfull = bars + 18;                 // [2] (kXIn)

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int cta = blockIdx.x;
    const int tm0 = p.t0 > 1 ? p.t0 : 1;                         // first step with a recurrent term

    if (warp == PRODUCER_WARP && lane == 0) {
        tma_prefetch_desc(&tmW);
        tma_prefetch_desc(&tmH);
        if (kXIn) { tma_prefetch_desc(&tmWx); tma_prefetch_desc(&tmX); }
        for (int g = 0; g < FWD_NG; ++g) mbar_init(&full[g], 1);
        mbar_init(wbar, 1);
        mbar_init(&xfull[0], 1); mbar_init(&xfull[1], 1);
        fence_mbar_init();
    }
    __syncthreads();

    if (warp == PRODUCER_WARP) {
        if (lane == 0) {
            // resident W_hh slice: chunk kc, gate g -> FWD_UNITS rows x 128 B
            mbar_expect_tx(wbar, FWD_W_BYTES);
            for (int kc = 0; kc < FWD_NCH; ++kc)
                for (int g = 0; g < 4; ++g)
                    tma_load_2d(sW + kc * (FWD_N * 128) + g * (FWD_UNITS * 128), &tmW, wbar, kc * KCH, g * LH + FWD_UNITS * cta);
            if (kXIn)                                          // W_ih slice behind it: chunks 16, 17 (columns beyond the input width: 0)
                for (int kc = 0; kc < XCH; ++kc)
                    for (int g = 0; g < 4; ++g)
                        tma_load_2d(sW + (FWD_NCH + kc) * (FWD_N * 128) + g * (FWD_UNITS * 128), &tmWx, wbar, kc * KCH, g * LH + FWD_UNITS * cta);
        }
        if (kXIn && tm0 < p.t1 && elect_one()) {               // x of the first contraction step: no dependency, load it now
            mbar_expect_tx(&xfull[0], XCH * slot_bytes);
#pragma unroll
            for (int kc = 0; kc < XCH; ++kc) tma_load_2d(sA + (FWD_NCH + kc) * slot_bytes, &tmX, &xfull[0], kc * KCH, tm0 * p.B);
        }
        __syncwarp();
        for (int t = tm0; t < p.t1; ++t) {
            // the first step of a chunk has nothing to wait for: h_{t0-1} was written by the previous launch on this stream
            // (kernel boundary) and the A buffer is untouched
            if (t > p.t0 && lane < FWD_NCH) wait_flag_ge(&p.flags[(t - 1 - p.t0) * FWD_NCH + lane], FWD_PROD, p.status, 212);
            __syncwarp();
            if (elect_one()) {
                FT_TRACE(p, t, 0);
                fence_proxy_async_global();        // generic-proxy writes of other SMs -> async-proxy (TMA) reads
                FT_TRACE(p, t, 6);
#pragma unroll
                for (int g = 0; g < FWD_NG; ++g) {
                    mbar_expect_tx(&full[g], FWD_GS * slot_bytes);
                    tma_load_3d(sA + g * FWD_GS * slot_bytes, &tmH, &full[g], 0, (t - 1) * p.B, g * FWD_GS);
                }
                if (kXIn && t + 1 < p.t1) {
                    // x_{t+1} does not depend on the recurrence: prefetch it one step ahead (it comes from HBM, not from L2
                    // like h: riding on this step's barrier would put its latency on the critical path).  Its buffer was last read by step t-1's MMAs,
                    // which have retired (all flags of step t-1, ours included, were seen above).
                    const int xs = (t + 1 - tm0) & 1;
                    mbar_expect_tx(&xfull[xs], XCH * slot_bytes);
#pragma unroll
                    for (int kc = 0; kc < XCH; ++kc)
                        tma_load_2d(sA + (FWD_NCH + xs * XCH + kc) * slot_bytes, &tmX, &xfull[xs], kc * KCH, (t + 1) * p.B);
                }
                FT_TRACE(p, t, 1);
            }
            __syncwarp();
        }
    } else {
        // ---------------------------------------------------------------- warpgroup: recurrent contraction + cell, 128 threads
        const int et = threadIdx.x;                           // 0..127
        // SWAPPED operands: A = the resident W slice (M = 64 accumulator rows: the CTA's 4*UNITS gate rows, plus -- for
        // UNITS = 8 -- 32 don't-care rows read from the next chunk), B = h_{t-1} (N = Bbox batch rows rounded up to 16 / 32;
        // rows beyond Bbox are read from the next chunk and never used).  A = h padded to 64 rows would make every
        // instruction read mostly padding from shared memory.
        const uint64_t da_base = wgmma_desc(smem_u32(sW), 16, 1024), db_base = wgmma_desc(smem_u32(sA), 16, 1024);
        const uint64_t a_chunk = (FWD_N * 128) >> 4, b_chunk = static_cast<uint64_t>(slot_bytes >> 4);
        const bool n16 = p.Bbox <= 16;
        // one step's contraction: [x_t chunks (kXIn)] + the 16 h_{t-1} chunks as they arrive, accumulator -> sAcc[batch][row]
        auto contract = [&](auto nb, int t) {
            constexpr int N = decltype(nb)::value;
            float acc[N / 2];
            const int xs = (t - tm0) & 1;
            // every operand chunk has landed before the first wgmma: a wait (a divergent polling loop) between wgmma
            // instructions would make ptxas serialize them
            if (kXIn) mbar_wait(&xfull[xs], ((t - tm0) >> 1) & 1, p.status, 216);
#pragma unroll
            for (int g = 0; g < FWD_NG; ++g) {
                mbar_wait(&full[g], (t - tm0) & 1, p.status, 214);
                if (et == 0 && g == 0) FT_TRACE(p, t, 2);
            }
            if (et == 0) FT_TRACE(p, t, 5);
            wgmma_fence_acc<N / 2>(acc);
            wgmma_fence();
            if (kXIn)                                         // the (prefetched) input chunks open the accumulation
                mma_chunks<N>(acc, da_base + FWD_NCH * a_chunk, db_base + (FWD_NCH + xs * XCH) * b_chunk, XCH, a_chunk, b_chunk, true);
            mma_chunks<N>(acc, da_base, db_base, FWD_NCH, a_chunk, b_chunk, !kXIn);
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_fence_acc<N / 2>(acc);
            if (et == 0) FT_TRACE(p, t, 4);
            const int r0 = 16 * warp + (lane >> 2), b0 = 2 * (lane & 3);
#pragma unroll
            for (int j = 0; j < N / 8; ++j) {
                const int b = 8 * j + b0;
                if (r0 < FWD_N) { sAcc[b * AP + r0] = acc[4 * j]; sAcc[(b + 1) * AP + r0] = acc[4 * j + 1]; }
                if (r0 + 8 < FWD_N) { sAcc[b * AP + r0 + 8] = acc[4 * j + 2]; sAcc[(b + 1) * AP + r0 + 8] = acc[4 * j + 3]; }
            }
        };
        mbar_wait(wbar, 0, p.status, 213);
        // work items: (batch row b, unit pair up) -> item = b * UP + up ; thread handles items et, et + 128
        constexpr int UP = FWD_UNITS / 2;
        const int n_items = p.B * UP;
        float c[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
        int len_i[2];
#pragma unroll
        for (int s = 0; s < 2; ++s) {
            const int item = et + s * EPI_THREADS;
            len_i[s] = (item < n_items && p.lens) ? p.lens[item / UP] : p.T;
        }
        const int u0 = FWD_UNITS * cta;
        if (p.t0 > 0) {                                       // resume the cell state saved by the previous chunk
#pragma unroll
            for (int s = 0; s < 2; ++s) {
                const int item = et + s * EPI_THREADS;
                if (item < n_items) {
                    const int b = item / UP, up = item % UP;
                    const float2 cv = *reinterpret_cast<const float2*>(p.cstate + (static_cast<long long>(p.t0 - 1) * p.B + b) * LH + u0 + 2 * up);
                    c[s][0] = cv.x; c[s][1] = cv.y;
                }
            }
        }
        float bias[2][8];                                     // kXIn: b_ih + b_hh of this thread's (gate, unit) pairs
        if (kXIn) {
#pragma unroll
            for (int s = 0; s < 2; ++s) {
                const int item = et + s * EPI_THREADS;
#pragma unroll
                for (int j = 0; j < 8; ++j) bias[s][j] = 0.f;
                if (item < n_items) {
                    const int up = item % UP;
#pragma unroll
                    for (int g = 0; g < 4; ++g) {
                        const int r = g * LH + u0 + 2 * up;
                        bias[s][2 * g] = p.b_ih[r] + p.b_hh[r];
                        bias[s][2 * g + 1] = p.b_ih[r + 1] + p.b_hh[r + 1];
                    }
                }
            }
        }
        for (int t = p.t0; t < p.t1; ++t) {
            float x[2][8];                                    // [item][gate*2 + e]
#pragma unroll
            for (int s = 0; s < 2; ++s) {
                const int item = et + s * EPI_THREADS;
                if (kXIn) {
#pragma unroll
                    for (int j = 0; j < 8; ++j) x[s][j] = bias[s][j];
                } else if (item < n_items) {
                    const int b = item / UP, up = item % UP;
                    const float* src = p.xproj + (static_cast<long long>(t) * p.B + b) * LG + u0 + 2 * up;
#pragma unroll
                    for (int g = 0; g < 4; ++g) {
                        const float2 v = __ldg(reinterpret_cast<const float2*>(src + g * LH));
                        x[s][2 * g] = v.x; x[s][2 * g + 1] = v.y;
                    }
                }
            }
            if (t > 0) {
                if (n16) contract(std::integral_constant<int, 16>(), t);
                else contract(std::integral_constant<int, 32>(), t);
                epi_bar();
                if (et == 0) FT_TRACE(p, t, 8);               // accumulator transposed into shared memory
#pragma unroll
                for (int s = 0; s < 2; ++s) {
                    const int item = et + s * EPI_THREADS;
                    if (item < n_items) {
                        const int b = item / UP, up = item % UP;
                        const float* a = sAcc + b * AP + 2 * up;
#pragma unroll
                        for (int g = 0; g < 4; ++g) { x[s][2 * g] += a[g * FWD_UNITS]; x[s][2 * g + 1] += a[g * FWD_UNITS + 1]; }
                    }
                }
            }
            float gi[2][2], gf[2][2], gg[2][2], go[2][2], hv[2][2];
#pragma unroll
            for (int s = 0; s < 2; ++s) {
                const int item = et + s * EPI_THREADS;
                if (item < n_items) {
                    const int b = item / UP, up = item % UP;
                    const bool valid = t < len_i[s];
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        gi[s][e] = sigmoid_f(x[s][0 + e]);
                        gf[s][e] = sigmoid_f(x[s][2 + e]);
                        gg[s][e] = tanh_f(x[s][4 + e]);
                        go[s][e] = sigmoid_f(x[s][6 + e]);
                        c[s][e] = gf[s][e] * c[s][e] + gi[s][e] * gg[s][e];
                        hv[s][e] = valid ? go[s][e] * tanh_f(c[s][e]) : 0.f;
                    }
                    const long long r = static_cast<long long>(t) * p.B + b;
                    const __half2 h2 = __floats2half2_rn(hv[s][0], hv[s][1]);
                    *reinterpret_cast<__half2*>(p.hseq + r * p.ldh + u0 + 2 * up) = h2;     // critical path: h_t first
                }
            }
            if (et == 0) FT_TRACE(p, t, 9);                   // cell computed, h_t stores issued
            epi_bar();                                        // all h_t stores of this CTA precede the release
            if (et == 0) {
                FT_TRACE(p, t, 10);
                red_release_add(&p.flags[(t - p.t0) * FWD_NCH + cta / FWD_PROD], 1);      // cumulative release (gpu scope)
                FT_TRACE(p, t, 7);
            }
            // off the critical path: tensors only the backward pass reads
#pragma unroll
            for (int s = 0; s < 2; ++s) {
                const int item = et + s * EPI_THREADS;
                if (item < n_items) {
                    const int b = item / UP, up = item % UP;
                    const long long r = static_cast<long long>(t) * p.B + b;
                    if (p.h32) *reinterpret_cast<float2*>(p.h32 + r * p.ldh32 + u0 + 2 * up) = make_float2(hv[s][0], hv[s][1]);
                    if (p.gates) {
                        __half* gp = p.gates + r * LG + u0 + 2 * up;
                        *reinterpret_cast<__half2*>(gp) = __floats2half2_rn(gi[s][0], gi[s][1]);
                        *reinterpret_cast<__half2*>(gp + LH) = __floats2half2_rn(gf[s][0], gf[s][1]);
                        *reinterpret_cast<__half2*>(gp + 2 * LH) = __floats2half2_rn(gg[s][0], gg[s][1]);
                        *reinterpret_cast<__half2*>(gp + 3 * LH) = __floats2half2_rn(go[s][0], go[s][1]);
                    }
                    if (p.cstate) *reinterpret_cast<float2*>(p.cstate + r * LH + u0 + 2 * up) = make_float2(c[s][0], c[s][1]);
                }
            }
        }
    }
}


// ------------------------------------------------------------------------------------------- host
static int smem_optin() {
    static int v = -1;
    if (v < 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&v, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    }
    return v;
}

PFN_encodeTiled get_tma_encoder();     // gemm.cu

// 3-D view of a row-major [rows, 64*nchunks] 16-bit tensor as {64 elems, rows, chunks}; box {64, box_rows, box_chunks}.
// The shared-memory image of one box is chunk-major: [chunk][row][128 B], SWIZZLE_128B -- i.e. `box_chunks`
// consecutive K-major wgmma tiles.
static int make_tmap_chunks(CUtensorMap* out, const void* ptr, long long rows, int nchunks, long long ld, int box_rows,
                            int box_chunks) {
    PFN_encodeTiled enc = get_tma_encoder();
    if (!enc) return -1;
    if ((reinterpret_cast<uintptr_t>(ptr) & 15) || ((ld * 2) & 15)) return ft_set_error("TMA operand must be 16-byte aligned with a 16-byte-multiple row pitch");
    cuuint64_t dims[3] = {64, static_cast<cuuint64_t>(rows), static_cast<cuuint64_t>(nchunks)};
    cuuint64_t strides[2] = {static_cast<cuuint64_t>(ld * 2), 128};
    cuuint32_t box[3] = {64, static_cast<cuuint32_t>(box_rows), static_cast<cuuint32_t>(box_chunks)};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(ptr), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return ft_set_error("cuTensorMapEncodeTiled (3-D chunk view) failed");
    return 0;
}

// Steps [t0, t1) of one layer's forward recurrence on 1024 / UNITS CTAs.  `flags` needs (t1 - t0) * 16 ints.
// x16 != null: folded input projection (kXIn): x16 [T*B, kx] fp16 (row pitch ldx), wih16 [4096, kx] fp16, biases fp32.
template <int UNITS, bool kXIn>
static int launch_fwd_t(int T, int B, int t0, int t1, const float* xproj, const void* whh16, const int* lens, void* hseq16,
                        long long ldh, void* gates16, float* cstate, float* h32, long long ldh32, int* flags, cudaStream_t st,
                        const void* x16 = nullptr, long long ldx = 0, int kx = 0, const void* wih16 = nullptr,
                        const float* b_ih = nullptr, const float* b_hh = nullptr) {
    constexpr int NCHT = FWD_NCH + (kXIn ? XCH : 0);
    constexpr int N = 4 * UNITS, W_BYTES = NCHT * N * 128, CTAS = LH / UNITS;
    LstmFwdChunkParams p;
    p.T = T; p.B = B; p.Bbox = (B + 7) & ~7; p.t0 = t0; p.t1 = t1;
    p.xproj = xproj; p.b_ih = b_ih; p.b_hh = b_hh; p.lens = lens; p.hseq = static_cast<__half*>(hseq16); p.ldh = ldh;
    p.gates = static_cast<__half*>(gates16); p.cstate = cstate; p.h32 = h32; p.ldh32 = ldh32;
    p.flags = flags; p.status = ft_status_word(); p.trace = (t0 == 0 && t1 == T) ? g_lstm_trace : nullptr;
    const int slot = p.Bbox * 128;
    const int smem = (FWD_NCH + (kXIn ? 2 * XCH : 0)) * slot + W_BYTES + 32 * (N + 1) * 4 + 8 + 256 + 1024;
    if (smem > smem_optin()) return ft_set_error("lstm_fwd: not enough shared memory");
    CUtensorMap tmW, tmH, tmWx, tmX;
    if (make_tmap_2d(&tmW, whh16, FMT_F16, LG, LH, LH, KCH, UNITS)) return -1;
    if (make_tmap_chunks(&tmH, hseq16, static_cast<long long>(T) * B, FWD_NCH, ldh, p.Bbox, FWD_GS)) return -1;
    if (kXIn) {
        if (kx <= 0 || kx > XCH * KCH) return ft_set_error("lstm_fwd: folded input width must be in (0, 128]");
        if (make_tmap_2d(&tmWx, wih16, FMT_F16, LG, kx, kx, KCH, UNITS)) return -1;
        if (make_tmap_2d(&tmX, x16, FMT_F16, static_cast<long long>(T) * B, kx, ldx, KCH, p.Bbox)) return -1;
    } else {
        tmWx = tmW; tmX = tmH;                                   // unused
    }
    FT_CU(cudaMemsetAsync(flags, 0, sizeof(int) * (t1 - t0) * FWD_NCH, st), "lstm_fwd");
    void* fn = reinterpret_cast<void*>(lstm_fwd_kernel<UNITS, kXIn>);
    cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    TimeScope ts("lstm_fwd", t1 - t0, B, 0, st);
    void* args[] = {&tmW, &tmH, &tmWx, &tmX, &p};
    cudaError_t e = cudaLaunchCooperativeKernel(fn, dim3(CTAS), dim3(LSTM_THREADS), args, smem, st);
    if (e != cudaSuccess) return ft_set_error(cudaGetErrorString(e));
    ft_count_launch(1);
    return ft_check_launch("lstm_fwd_kernel");
}

// Whole sequence on 64 CTAs: the kernel of launch_lstm_fwd_chunk over [0, T).
int launch_lstm_fwd(int T, int B, const float* xproj, const void* whh16, const int* lens, void* hseq16, long long ldh,
                    void* gates16, float* cstate, float* h32, long long ldh32, int* flags, cudaStream_t st) {
    if (T <= 0 || B <= 0) return 0;
    if (B > 32) return ft_set_error("lstm_fwd: batch > 32 per call not supported (split the batch)");
    return launch_fwd_t<16, false>(T, B, 0, T, xproj, whh16, lens, hseq16, ldh, gates16, cstate, h32, ldh32, flags, st);
}

// Whole sequence with the input projection folded in (narrow inputs, kx <= 128; x16 row 0..B-1 must be zero: step 0 skips the
// contraction).  128 CTAs.
int launch_lstm_fwd_xin(int T, int B, const void* x16, long long ldx, int kx, const void* wih16, const float* b_ih, const float* b_hh,
                        const void* whh16, const int* lens, void* hseq16, long long ldh, void* gates16, float* cstate, float* h32,
                        long long ldh32, int* flags, cudaStream_t st) {
    if (T <= 0 || B <= 0) return 0;
    if (B > 32) return ft_set_error("lstm_fwd: batch > 32 per call not supported (split the batch)");
    if (!x16 || !wih16 || !b_ih || !b_hh) return ft_set_error("lstm_fwd_xin: NULL argument");
    return launch_fwd_t<8, true>(T, B, 0, T, nullptr, whh16, lens, hseq16, ldh, gates16, cstate, h32, ldh32, flags, st, x16, ldx, kx, wih16, b_ih, b_hh);
}

// Steps [t0, t1) of a layer on 64 CTAs (layer pipeline, ar_step.cu).  `flags` needs (t1 - t0) * 16 ints.
int launch_lstm_fwd_chunk(int T, int B, int t0, int t1, const float* xproj, const void* whh16, const int* lens, void* hseq16,
                          long long ldh, void* gates16, float* cstate, int* flags, cudaStream_t st, float* h32, long long ldh32) {
    if (T <= 0 || B <= 0 || t1 <= t0) return 0;
    if (B > 32 || t0 < 0 || t1 > T) return ft_set_error("lstm_fwd_chunk: bad batch or step range");
    if (t0 > 0 && !cstate) return ft_set_error("lstm_fwd_chunk: resuming a chunk needs the saved cell states");
    return launch_fwd_t<16, false>(T, B, t0, t1, xproj, whh16, lens, hseq16, ldh, gates16, cstate, h32, ldh32, flags, st);
}

// Steps [t0, t1) of a layer's BPTT.  Cluster kernel (xchg == null): `flags` needs (t1 - t0) * 64 ints.  Flat kernel: `flags`
// needs (t1 - t0) * 128 ints and `xchg` 2 * 16 * 4 * B * 64 floats.  `dc_carry` ([B,1024] fp32) is only touched when the
// range is a proper chunk.
static int launch_bwd(int T, int B, int t0, int t1, const float* dh_ext, long long ldd, const void* whhT16, const void* gates16,
                      const float* cstate, const int* lens, void* dG16, float* dc_carry, int* flags, float* xchg, cudaStream_t st) {
    const bool flat = xchg != nullptr;
    LstmBwdChunkParams p;
    p.T = T; p.B = B; p.Bbox = (B + 7) & ~7; p.t0 = t0; p.t1 = t1; p.dc_carry = dc_carry; p.xchg = xchg;
    const int slot = p.Bbox * 128;
    p.dh_ext = dh_ext; p.ldd = ldd; p.gates = static_cast<const __half*>(gates16); p.cstate = cstate; p.lens = lens;
    p.dG = static_cast<__half*>(dG16); p.flags = flags; p.status = ft_status_word();
    p.trace = (t0 == 0 && t1 == T) ? g_lstm_trace : nullptr;
    CUtensorMap tmWT, tmG;
    if (make_tmap_2d(&tmWT, whhT16, FMT_F16, LH, LG, LG, KCH, B4_UNITS)) return -1;
    if (make_tmap_chunks(&tmG, dG16, static_cast<long long>(T) * B, BWD_NCH, LG, p.Bbox, 8)) return -1;
    FT_CU(cudaMemsetAsync(flags, 0, sizeof(int) * (t1 - t0) * BWD_NCH * (flat ? 2 : 1), st), "lstm_bwd");
    if (flat) {
        const int smem = B4_NCH * slot + B4_W_BYTES + 256 + 1024;
        cudaFuncSetAttribute(lstm_bwd_flat_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        TimeScope ts("lstm_bwd", t1 - t0, B, 0, st);
        void* args[] = {&tmWT, &tmG, &p};
        cudaError_t e = cudaLaunchCooperativeKernel(reinterpret_cast<void*>(lstm_bwd_flat_kernel), dim3(B4_CTAS), dim3(LSTM_THREADS),
                                                    args, smem, st);
        if (e != cudaSuccess) return ft_set_error(cudaGetErrorString(e));
        ft_count_launch(1);
        return ft_check_launch("lstm_bwd_flat_kernel");
    }
    const int smem = B4_NCH * slot + B4_W_BYTES + B4_XCHG_FLOATS * 4 + 256 + 1024;
    cudaFuncSetAttribute(lstm_bwd4_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(B4_CTAS); cfg.blockDim = dim3(LSTM_THREADS); cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attrs[2];
    attrs[0].id = cudaLaunchAttributeClusterDimension;
    attrs[0].val.clusterDim.x = B4_CLUSTER; attrs[0].val.clusterDim.y = 1; attrs[0].val.clusterDim.z = 1;
    attrs[1].id = cudaLaunchAttributeCooperative;
    attrs[1].val.cooperative = 1;
    cfg.attrs = attrs; cfg.numAttrs = 2;
    TimeScope ts("lstm_bwd", t1 - t0, B, 0, st);
    cudaError_t e = cudaLaunchKernelEx(&cfg, lstm_bwd4_kernel, tmWT, tmG, p);
    if (e != cudaSuccess) {                                  // co-residency is implied by 64 CTAs <= SMs; retry without the attribute
        cudaGetLastError();
        cfg.numAttrs = 1;
        e = cudaLaunchKernelEx(&cfg, lstm_bwd4_kernel, tmWT, tmG, p);
    }
    if (e != cudaSuccess) return ft_set_error(cudaGetErrorString(e));
    ft_count_launch(1);
    return ft_check_launch("lstm_bwd4_kernel");
}

int lstm_bwd_max_clusters(int B) {
    const int smem = B4_NCH * (((B + 7) & ~7) * 128) + B4_W_BYTES + B4_XCHG_FLOATS * 4 + 256 + 1024;
    if (cudaFuncSetAttribute(lstm_bwd4_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess) return -1;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(B4_CTAS); cfg.blockDim = dim3(LSTM_THREADS); cfg.dynamicSmemBytes = smem;
    cudaLaunchAttribute attr;
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = B4_CLUSTER; attr.val.clusterDim.y = 1; attr.val.clusterDim.z = 1;
    cfg.attrs = &attr; cfg.numAttrs = 1;
    int n = -1;
    if (cudaOccupancyMaxActiveClusters(&n, lstm_bwd4_kernel, &cfg) != cudaSuccess) return -1;
    return n;
}

// Steps [t0, t1) of a layer's BPTT (layer pipeline, ar_step.cu).  `xchg` non-null: the flat kernel, whose 64 CTAs fit next
// to the other layer's chunk; null: the cluster kernel.  See launch_bwd for the sizes of `flags` and `xchg`.
int launch_lstm_bwd_chunk(int T, int B, int t0, int t1, const float* dh_ext, long long ldd, const void* whhT16, const void* gates16,
                          const float* cstate, const int* lens, void* dG16, float* dc_carry, int* flags, float* xchg, cudaStream_t st) {
    if (T <= 0 || B <= 0 || t1 <= t0) return 0;
    if (B > 32 || t0 < 0 || t1 > T || !dc_carry) return ft_set_error("lstm_bwd_chunk: bad batch, step range or carry buffer");
    return launch_bwd(T, B, t0, t1, dh_ext, ldd, whhT16, gates16, cstate, lens, dG16, dc_carry, flags, xchg, st);
}

// Whole sequence (the attention LSTM's BPTT, which runs alone) on the cluster kernel: alone, its DSMEM exchange is the
// faster one -- 3.96 us/step against the flat kernel's 4.27 (T = 1000, B = 32, H100 80GB HBM3, tools/bptt_overlap.py).
int launch_lstm_bwd(int T, int B, const float* dh_ext, long long ldd, const void* whhT16, const void* gates16,
                    const float* cstate, const int* lens, void* dG16, int* flags, cudaStream_t st) {
    if (T <= 0 || B <= 0) return 0;
    if (B > 32) return ft_set_error("lstm_bwd: batch > 32 per call not supported (split the batch)");
    return launch_bwd(T, B, 0, T, dh_ext, ldd, whhT16, gates16, cstate, lens, dG16, nullptr, flags, nullptr, st);
}

}  // namespace ft
