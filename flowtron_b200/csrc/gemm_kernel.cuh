// wgmma + TMA GEMM for sm_90a:  C[M,N] = act(alpha * A[M,K] * B[N,K]^T + bias (+bias2)) (+ C if beta)
//
//  * operands 16-bit (f16 / bf16, K = 16 per wgmma) or tf32 (fp32 storage, K = 8 per wgmma), fp32 accumulation in registers;
//    a 16-bit operand may be K-major (row-major [rows, K]) or MN-major (row-major [K, rows], i.e. the transposed view of a
//    natural activation / gradient tensor) -- this is what lets dW = dY^T X and dX = dY W run on the tensors exactly as the
//    forward pass left them (no transposes anywhere);
//  * persistent: one CTA per SM walks a static list of 128 x BN output tiles (BN = 256, or 128 for narrow outputs) through a
//    4-stage (BN = 256: 48 KB per stage) / 6-stage (BN = 128: 32 KB) TMA ring in SWIZZLE_128B layout, optional split-K;
//  * warpgroup roles: WG0 = TMA producer (one elected thread), WG1 / WG2 = consumers.  Cooperative schedule: each consumer
//    owns 64 rows of the tile with a 64 x BN fp32 accumulator in registers (128 registers per thread at BN = 256;
//    setmaxnreg moves registers from the producer to the consumers).  Ping-pong schedule (PP, launch_gemm picks it by
//    shape): each consumer owns whole 128 x 128 tiles, alternating with the other, so one's epilogue runs under the
//    other's main loop.  While a consumer runs its epilogue the producer already fills the ring for its next tile;
//  * epilogue through shared memory: each consumer stages its 64 x BN result in 64 x 32 chunks (two 8 KB slots, SWIZZLE_128B
//    for fp32 / SWIZZLE_64B for 16-bit outputs; ping-pong: each warp its own 16 x 32 chunks in two 2 KB slots) and writes
//    them with TMA stores (reduce-add for split-K partial tiles and for beta = 1 without a 16-bit output), so it returns to
//    its next tile's wgmmas while the stores drain.
//
// Used for every non-recurrent contraction on the Flowtron hot path (LSTM input projections flowtron.py:654-655, attention
// Q/K/V projections :568-571, DenseLayer :461-464, 1x1 conv :768, and all their dgrad/wgrad counterparts).
#pragma once
#include "ptx.cuh"
#include "ft_internal.h"

namespace ft {

constexpr int BM = 128;
constexpr int TILE_BYTES = BM * 128;               // A tile of one stage: 128 rows x 128 B (one SW128 row per matrix row)

struct GemmParams {
    int M, N, K;
    const float* bias;         // [N] or null
    const float* bias2;        // [N] or null
    int act;                   // 0 none, 1 tanh, 2 multiply by (1 - aux^2)  (tanh backward; aux = saved tanh output)
    const __half* aux16; long long ldaux;
    int beta;                  // 1: C32 += result (C32 read-modify-write)
    float alpha;               // scale on the accumulator before bias
    const float* alpha_ptr;    // optional device scalar multiplied into alpha (loss-scale undo)
    float* C32; long long ldc32;
    void* C16; long long ldc16; int c16_fmt;   // 0 f16, 1 bf16
    int* status;
    int splitk = 1;            // K is cut into `splitk` ranges, partial tiles are added into a zeroed C32
    int tma_c = 0;             // 1: staged epilogue with TMA stores (aligned outputs, even N); 0: fragment stores (epi_pair)
    int c32_add = 0;           // tma_c: C32 += tile by TMA reduce-add (split-K, or beta without C16)
};

constexpr int G2_THREADS = 384;                                 // WG0 producer, WG1 + WG2 consumers
constexpr int G2_CONSUMER_WARPS = 8;
// NCTA = 2 (BN = 256 only): a 2-CTA cluster owns a 256 x 256 tile.  Each CTA stages its own 128 rows of A and fetches HALF of
// B's 256 rows, multicasting it into both CTAs' rings: B is read from L2 once per 256 output rows instead of once per 128.
constexpr int EPI_SLOT = 64 * 128;                       // one staged 64 x 32 fp32 chunk (a 16-bit chunk uses half)
constexpr int EPI_BYTES = 2 * 2 * EPI_SLOT;              // two slots per consumer warpgroup
template <int BN_, int NCTA = 1> struct G2Cfg {
    static constexpr int STAGE_BYTES = (BM + BN_) * 128;
    static constexpr int STAGES = BN_ == 256 ? 4 : 6;
    static constexpr int SMEM = STAGES * STAGE_BYTES + EPI_BYTES + 256 + 1024;
};

// One output pair (columns n, n + 1 of row m) through alpha / bias / activation / beta into C32 and / or C16.
__device__ __forceinline__ void epi_pair(const GemmParams& p, long long m, int n, float v0, float v1, float alpha, bool vec2) {
    if (m >= p.M || n >= p.N) return;
    if (vec2) {                                                   // N even, every operand 8 / 4-byte aligned: n + 1 < N
        float2 b = make_float2(0.f, 0.f);
        if (p.bias) b = __ldg(reinterpret_cast<const float2*>(p.bias + n));
        if (p.bias2) { const float2 t = __ldg(reinterpret_cast<const float2*>(p.bias2 + n)); b.x += t.x; b.y += t.y; }
        float x0 = fmaf(v0, alpha, b.x), x1 = fmaf(v1, alpha, b.y);
        if (p.act == 1) { x0 = tanh_f(x0); x1 = tanh_f(x1); }
        else if (p.act == 2) {
            const float2 y = __half22float2(*reinterpret_cast<const __half2*>(p.aux16 + m * p.ldaux + n));
            x0 *= (1.f - y.x * y.x); x1 *= (1.f - y.y * y.y);
        }
        if (p.C32) {
            float2* dst = reinterpret_cast<float2*>(p.C32 + m * p.ldc32 + n);
            if (p.splitk > 1) { atomicAdd(dst, make_float2(x0, x1)); return; }
            if (p.beta) { const float2 o = *dst; x0 += o.x; x1 += o.y; }
            *dst = make_float2(x0, x1);
        }
        if (p.C16) {
            if (p.c16_fmt == 0)      // fp16: saturate instead of overflowing to inf
                *reinterpret_cast<__half2*>(reinterpret_cast<__half*>(p.C16) + m * p.ldc16 + n) =
                    __floats2half2_rn(fminf(fmaxf(x0, -65504.f), 65504.f), fminf(fmaxf(x1, -65504.f), 65504.f));
            else
                *reinterpret_cast<__nv_bfloat162*>(reinterpret_cast<__nv_bfloat16*>(p.C16) + m * p.ldc16 + n) = __floats2bfloat162_rn(x0, x1);
        }
        return;
    }
    // unaligned / odd-N outputs: element by element (no shape on the hot path)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
        const int c = n + e;
        if (c >= p.N) break;
        float x = fmaf(e ? v1 : v0, alpha, (p.bias ? __ldg(p.bias + c) : 0.f) + (p.bias2 ? __ldg(p.bias2 + c) : 0.f));
        if (p.act == 1) x = tanh_f(x);
        else if (p.act == 2) { const float y = __half2float(p.aux16[m * p.ldaux + c]); x *= (1.f - y * y); }
        if (p.C32) {
            float* dst = p.C32 + m * p.ldc32 + c;
            if (p.splitk > 1) { atomicAdd(dst, x); continue; }
            if (p.beta) x += *dst;
            *dst = x;
        }
        if (p.C16) {
            if (p.c16_fmt == 0) reinterpret_cast<__half*>(p.C16)[m * p.ldc16 + c] = __float2half_rn(fminf(fmaxf(x, -65504.f), 65504.f));
            else reinterpret_cast<__nv_bfloat16*>(p.C16)[m * p.ldc16 + c] = __float2bfloat16_rn(x);
        }
    }
}

// Staged epilogue of one consumer warpgroup's 64 x BN accumulator (rows m_base.., columns n_base..): 64 x 32 chunks into
// the warpgroup's two shared-memory slots (chunk q in slot q & 1), each written by one TMA store (or reduce-add) issued by
// the warpgroup's first thread, which therefore owns every bulk group of the warpgroup.  A slot is refilled once the store
// issued from it two chunks earlier has read it; the first chunk of a tile waits for all of the previous tile's stores to
// have read shared memory (long done: a whole main loop ran since), and with both C32 and C16 the two slots hold one
// chunk's two tiles, so each chunk waits for the previous one.  Per element the values are those of epi_pair.
template <int BN_>
__device__ __forceinline__ void epi_staged(const GemmParams& p, const CUtensorMap* tmC32, const CUtensorMap* tmC16,
                                           const float* acc, float alpha, uint32_t stg, int c, int m_base, int n_base) {
    const int t = threadIdx.x & 127, lane = t & 31;
    const bool dual = p.C32 && p.C16;
    const int r0 = (t >> 5) * 16 + (lane >> 2);              // rows r0 and r0 + 8 of the 64-row sub-tile
    const int sw = lane >> 2;                                // (r0 + 8 h) & 7
#pragma unroll
    for (int q = 0; q < BN_ / 32; ++q) {
        const int nq = n_base + 32 * q;
        if (nq >= p.N) break;
        if (t == 0) {
            if (q == 0 || dual) bulk_wait_read<0>();
            else bulk_wait_read<1>();
        }
        named_bar_sync(1 + c, 128);                          // the slot(s) about to be written have been read
        const uint32_t s32 = stg + (dual ? 0 : q & 1) * EPI_SLOT;     // shared-memory addresses
        const uint32_t s16 = stg + (dual ? 1 : q & 1) * EPI_SLOT;
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
            const int j = 4 * q + jj;
            const int cl = 8 * jj + 2 * (lane & 3);          // column pair within the chunk
            const int n = nq + cl;
            const bool nin = n < p.N;                        // N even: n + 1 < N as well
            float2 b = make_float2(0.f, 0.f);
            if (nin && p.bias) b = __ldg(reinterpret_cast<const float2*>(p.bias + n));
            if (nin && p.bias2) { const float2 u2 = __ldg(reinterpret_cast<const float2*>(p.bias2 + n)); b.x += u2.x; b.y += u2.y; }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = r0 + 8 * h;
                const int m = m_base + r;
                const bool in = nin && m < p.M;
                float x0 = fmaf(acc[4 * j + 2 * h], alpha, b.x), x1 = fmaf(acc[4 * j + 2 * h + 1], alpha, b.y);
                if (p.act == 1) { x0 = tanh_f(x0); x1 = tanh_f(x1); }
                else if (p.act == 2 && in) {
                    const float2 y = __half22float2(*reinterpret_cast<const __half2*>(p.aux16 + static_cast<long long>(m) * p.ldaux + n));
                    x0 *= (1.f - y.x * y.x); x1 *= (1.f - y.y * y.y);
                }
                if (p.C32) {
                    if (p.beta && !p.c32_add && in) {        // beta with a 16-bit output: C16 gets the sum too
                        const float2 o = *reinterpret_cast<const float2*>(p.C32 + static_cast<long long>(m) * p.ldc32 + n);
                        x0 += o.x; x1 += o.y;
                    }
                    const int u = cl >> 2;                   // SWIZZLE_128B: 16-byte unit u of row r sits at u ^ (r & 7)
                    st_shared_f2(s32 + r * 128 + ((u ^ sw) << 4) + (cl & 2) * 4, x0, x1);
                }
                if (p.C16) {
                    const int u = cl >> 3;                   // SWIZZLE_64B, 64-byte rows: unit u of row r sits at u ^ ((r >> 1) & 3)
                    const uint32_t d = s16 + r * 64 + ((u ^ ((r >> 1) & 3)) << 4) + (cl & 6) * 2;
                    if (p.c16_fmt == 0) {    // fp16: saturate instead of overflowing to inf
                        const __half2 h2 = __floats2half2_rn(fminf(fmaxf(x0, -65504.f), 65504.f), fminf(fmaxf(x1, -65504.f), 65504.f));
                        st_shared_b32(d, *reinterpret_cast<const uint32_t*>(&h2));
                    } else {
                        const __nv_bfloat162 h2 = __floats2bfloat162_rn(x0, x1);
                        st_shared_b32(d, *reinterpret_cast<const uint32_t*>(&h2));
                    }
                }
            }
        }
        fence_proxy_async_smem();                            // the staged chunk is visible to the TMA unit
        named_bar_sync(1 + c, 128);
        if (t == 0) {
            if (p.C32) {
                if (p.c32_add) tma_reduce_add_2d(tmC32, s32, nq, m_base);
                else tma_store_2d(tmC32, s32, nq, m_base);
            }
            if (p.C16) tma_store_2d(tmC16, s16, nq, m_base);
            bulk_commit();
        }
    }
}

// Ping-pong epilogue of one warp: its 16 rows of each 64-row half of the warpgroup's 128 x 128 tile (acc[64 h + ..], the
// m64n128 fragment layout; rows m_w + 64 h + ..), in 16 x 32 chunks staged in the warp's own two 2 KB slots at `stg` (the
// n-th chunk of the tile in slot n & 1; with both C32 and C16 one chunk fills both slots) and written by a TMA store, or
// reduce-add for beta = 1 without a 16-bit output, that the warp's lane 0 issues.  So the warp needs only __syncwarp, not a
// warpgroup barrier, and lane 0 owns the warp's bulk groups.  No global loads but bias / bias2: launch_gemm keeps act = 2
// (aux reads) and beta with a 16-bit output (C32 reads) on the cooperative schedule, where per-element loads fit the
// register budget.  Per element the values are those of epi_pair.
__device__ __forceinline__ void epi_warp(const GemmParams& p, const CUtensorMap* tmC32, const CUtensorMap* tmC16,
                                         const float* acc, float alpha, uint32_t stg, int m_w, int n_base) {
    const int lane = threadIdx.x & 31;
    const bool dual = p.C32 && p.C16;
    const int sw = lane >> 2;                                // (r + 8 hh) & 7 for row r = lane / 4 + 8 hh of the chunk
    const int nqc = min(4, (p.N - n_base + 31) / 32);        // column chunks of the tile inside N (>= 1)
    const int nh = m_w + 64 < p.M ? 2 : 1;                   // halves with rows inside M (the TMA store would clip the rest)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        if (h >= nh) break;
        const int mh = m_w + 64 * h;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            if (q >= nqc) break;
            const int nq = n_base + 32 * q;
            float2 b[4];
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) {
                const int n = nq + 8 * jj + 2 * (lane & 3);
                b[jj] = make_float2(0.f, 0.f);
                if (n < p.N && p.bias) b[jj] = __ldg(reinterpret_cast<const float2*>(p.bias + n));
                if (n < p.N && p.bias2) { const float2 u2 = __ldg(reinterpret_cast<const float2*>(p.bias2 + n)); b[jj].x += u2.x; b[jj].y += u2.y; }
            }
            const int nc = nqc * h + q;                       // chunks of this tile so far
            if (lane == 0) {
                if (nc == 0 || dual) bulk_wait_read<0>();
                else bulk_wait_read<1>();                    // the store issued from this slot two chunks ago has read it
            }
            __syncwarp();
            const uint32_t s32 = stg + (dual ? 0 : nc & 1) * 2048;
            const uint32_t s16 = stg + (dual ? 1 : nc & 1) * 2048;
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) {
                const int j = 4 * q + jj;
                const int cl = 8 * jj + 2 * (lane & 3);      // column pair within the chunk
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
                    const int r = (lane >> 2) + 8 * hh;
                    float x0 = fmaf(acc[64 * h + 4 * j + 2 * hh], alpha, b[jj].x), x1 = fmaf(acc[64 * h + 4 * j + 2 * hh + 1], alpha, b[jj].y);
                    if (p.act == 1) { x0 = tanh_f(x0); x1 = tanh_f(x1); }
                    if (p.C32) {
                        const int u = cl >> 2;               // SWIZZLE_128B: 16-byte unit u of row r sits at u ^ (r & 7)
                        st_shared_f2(s32 + r * 128 + ((u ^ sw) << 4) + (cl & 2) * 4, x0, x1);
                    }
                    if (p.C16) {
                        const int u = cl >> 3;               // SWIZZLE_64B, 64-byte rows: unit u of row r sits at u ^ ((r >> 1) & 3)
                        const uint32_t d = s16 + r * 64 + ((u ^ ((r >> 1) & 3)) << 4) + (cl & 6) * 2;
                        if (p.c16_fmt == 0) {    // fp16: saturate instead of overflowing to inf
                            const __half2 h2 = __floats2half2_rn(fminf(fmaxf(x0, -65504.f), 65504.f), fminf(fmaxf(x1, -65504.f), 65504.f));
                            st_shared_b32(d, *reinterpret_cast<const uint32_t*>(&h2));
                        } else {
                            const __nv_bfloat162 h2 = __floats2bfloat162_rn(x0, x1);
                            st_shared_b32(d, *reinterpret_cast<const uint32_t*>(&h2));
                        }
                    }
                }
            }
            fence_proxy_async_smem();                        // the staged chunk is visible to the TMA unit
            __syncwarp();
            if (lane == 0) {
                if (p.C32) {
                    if (p.c32_add) tma_reduce_add_2d(tmC32, s32, nq, mh);
                    else tma_store_2d(tmC32, s32, nq, mh);
                }
                if (p.C16) tma_store_2d(tmC16, s16, nq, mh);
                bulk_commit();
            }
        }
    }
}

// PP = false: cooperative schedule, both consumer warpgroups on one 128 x BN tile (64 rows each; CTA pairs, split-K).
// PP = true (BN_ = 128, NCTA = 1, no split-K, staged epilogue without act = 2 or a C32 read): ping-pong schedule, each consumer warpgroup owns whole
// 128 x 128 tiles (two m64n128 wgmmas per K step, 128 accumulator registers as in the cooperative tile) and the two take
// alternate tiles of the CTA's list; named barriers 3 and 4 hand the tensor cores from one warpgroup's main loop to the
// other's, so each warpgroup's epilogue runs under the other's main loop.
template <int FMT, int BN_, int NCTA, int TA, int TB, bool PP = false>
__global__ void __launch_bounds__(G2_THREADS, 1)
gemm2_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
             const __grid_constant__ CUtensorMap tmC32, const __grid_constant__ CUtensorMap tmC16, GemmParams p, int tiles_n,
             int n_tiles) {
    static_assert(!PP || (BN_ == 128 && NCTA == 1), "ping-pong tiles are 128 x 128, single CTA");
    using C = G2Cfg<BN_, NCTA>;
    constexpr int TM = BM * NCTA;                   // rows of a work item's tile
    const int rank = NCTA == 2 ? static_cast<int>(cluster_ctarank()) : 0;
    const int wid0 = NCTA == 2 ? static_cast<int>(blockIdx.x >> 1) : static_cast<int>(blockIdx.x);
    const int wstep = NCTA == 2 ? static_cast<int>(gridDim.x >> 1) : static_cast<int>(gridDim.x);
    constexpr int ST = C::STAGES;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* epi = smem + ST * C::STAGE_BYTES;      // [2 consumer warpgroups][2 slots] staged output chunks
    uint64_t* bars = reinterpret_cast<uint64_t*>(epi + EPI_BYTES);
    uint64_t* full = bars;                 // [ST]
    uint64_t* empty = bars + ST;           // [ST]: one arrival per consumer warp of every CTA that writes into this stage

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7;
    constexpr int ELT = FMT == FMT_TF32 ? 4 : 2;
    constexpr int BK = 128 / ELT;
    constexpr int UK = 32 / ELT;
    const int num_kb_all = (p.K + BK - 1) / BK;
    const int kb_per_split = (num_kb_all + p.splitk - 1) / p.splitk;     // work item w = split * n_tiles + tile
    const int n_work = n_tiles * p.splitk;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        if (p.tma_c && p.C32) tma_prefetch_desc(&tmC32);
        if (p.tma_c && p.C16) tma_prefetch_desc(&tmC16);
        // empty: every consumer warp of the CTA(s) reading the stage, i.e. of one warpgroup under ping-pong
        for (int s = 0; s < ST; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], PP ? 4 : G2_CONSUMER_WARPS * NCTA); }
        fence_mbar_init();
    }
    if (NCTA == 2) cluster_sync_all();              // the peer's barriers exist before anything can arrive on them
    else __syncthreads();

    if (wg == 0) {
        setmaxnreg_dec40();
        if (warp == 0) {
            // ------------------------------------------------ TMA producer (warp-uniform loop, one elected lane issues)
            constexpr int BNC = BN_ / NCTA;         // B rows this CTA fetches
            int it = 0;
            auto ldb = [&](void* dst, int c0, int c1) {
                if (NCTA == 2) tma_load_2d_mc(dst, &tmB, &full[it % ST], c0, c1, 0x3);
                else tma_load_2d(dst, &tmB, &full[it % ST], c0, c1);
            };
            for (int w = wid0; w < n_work; w += wstep) {
                const int split = w / n_tiles, tile = w - split * n_tiles;
                const int tile_m = tile / tiles_n, tile_n = tile - tile_m * tiles_n;
                const int kb0 = split * kb_per_split, kb1 = min(num_kb_all, kb0 + kb_per_split);
                const int am = tile_m * TM + rank * BM, bn = tile_n * BN_ + rank * BNC;
                for (int kb = kb0; kb < kb1; ++kb, ++it) {
                    const int s = it % ST, ph = (it / ST) & 1;
                    if (NCTA == 2) mbar_wait_cluster(&empty[s], ph ^ 1, p.status, 111);
                    else mbar_wait(&empty[s], ph ^ 1, p.status, 111);
                    uint8_t* a = smem + s * C::STAGE_BYTES;
                    uint8_t* b = a + TILE_BYTES + rank * (BNC * 128);
                    if (elect_one()) {
                        mbar_expect_tx(&full[s], C::STAGE_BYTES);     // own A + all of B (the peer multicasts its half)
                        if (!TA) {
                            tma_load_2d(a, &tmA, &full[s], kb * BK, am);
                        } else {
#pragma unroll
                            for (int j = 0; j < BM / BK; ++j) tma_load_2d(a + j * (BK * 128), &tmA, &full[s], am + j * BK, kb * BK);
                        }
                        if (!TB) {
                            ldb(b, kb * BK, bn);
                        } else {
#pragma unroll
                            for (int j = 0; j < BNC / BK; ++j) ldb(b + j * (BK * 128), bn + j * BK, kb * BK);
                        }
                    }
                    __syncwarp();
                }
            }
        }
    } else if constexpr (PP) {
        setmaxnreg_inc232();
        // ------------------------------------------------ ping-pong consumers: warpgroup c owns items j = c, c + 2, .. of
        // the CTA's list; warp wq stores rows [16 wq, 16 wq + 16) of each 64-row half of the tile
        const int c = wg - 1, wq = warp & 3;
        const float alpha = p.alpha_ptr ? p.alpha * __ldg(p.alpha_ptr) : p.alpha;
        constexpr uint64_t KA = TA ? (UK * 128) >> 4 : 2, KB = TB ? (UK * 128) >> 4 : 2;   // descriptor advance per wgmma K step
        constexpr uint64_t AH = (64 * 128) >> 4;                                            // A rows 64..127 of the tile
        const uint64_t da0 = wgmma_desc(smem_u32(smem), BK * 128, 1024);
        const uint64_t db0 = wgmma_desc(smem_u32(smem + TILE_BYTES), BK * 128, 1024);
        const uint32_t stg = smem_u32(epi) + (4 * c + wq) * (2 * 2048);
        float acc[128];
        int j = c;                                           // list item
        for (int w = wid0 + c * wstep; w < n_work; w += 2 * wstep, j += 2) {
            const int it = j * num_kb_all;                   // ring position of its first stage
            const int tile_m = w / tiles_n, tile_n = w - tile_m * tiles_n;
            const int n_base = tile_n * BN_;
            if (j > 0) named_bar_sync(3 + c, 256);           // the other warpgroup has issued item j - 1's main loop
            for (int kb = 0; kb < num_kb_all; ++kb) {
                const int i = it + kb, s = i % ST, ph = (i / ST) & 1;
                mbar_wait(&full[s], ph, p.status, 113);
                const uint64_t so = static_cast<uint64_t>(s) * (C::STAGE_BYTES >> 4);
                wgmma_fence_acc<128>(acc);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < BK / UK; ++k) {
                    wgmma_k<128, FMT, TA, TB>(acc, da0 + so + k * KA, db0 + so + k * KB, (kb > 0 || k > 0) ? 1u : 0u);
                    wgmma_k<128, FMT, TA, TB>(acc + 64, da0 + AH + so + k * KA, db0 + so + k * KB, (kb > 0 || k > 0) ? 1u : 0u);
                }
                wgmma_commit();
                wgmma_wait<1>();                             // the previous stage's wgmmas have read their operands
                wgmma_fence_acc<128>(acc);
                if (kb > 0 && lane == 0) mbar_arrive(&empty[(i - 1) % ST]);
            }
            if (w + wstep < n_work) named_bar_arrive(3 + (c ^ 1), 256);   // item j + 1 may take the tensor cores
            wgmma_wait<0>();
            wgmma_fence_acc<128>(acc);
            if (lane == 0) mbar_arrive(&empty[(it + num_kb_all - 1) % ST]);
#ifndef FT_GEMM_NO_STORE
            epi_warp(p, &tmC32, &tmC16, acc, alpha, stg, tile_m * BM + 16 * wq, n_base);
#endif
        }
        if (lane == 0) bulk_wait_all();                      // staged chunks stay in shared memory until stored
    } else {
        setmaxnreg_inc232();
        // ------------------------------------------------ consumers: rows [64 c, 64 c + 64) of the CTA's 128-row tile
        const int c = wg - 1, wq = warp & 3;
        const float alpha = p.alpha_ptr ? p.alpha * __ldg(p.alpha_ptr) : p.alpha;
        const bool vec2 = (p.N % 2 == 0) &&
                          (!p.C32 || (((reinterpret_cast<uintptr_t>(p.C32) & 7) == 0) && (p.ldc32 % 2 == 0))) &&
                          (!p.C16 || (((reinterpret_cast<uintptr_t>(p.C16) & 3) == 0) && (p.ldc16 % 2 == 0))) &&
                          (p.act != 2 || (((reinterpret_cast<uintptr_t>(p.aux16) & 3) == 0) && (p.ldaux % 2 == 0))) &&
                          (!p.bias || (reinterpret_cast<uintptr_t>(p.bias) & 7) == 0) && (!p.bias2 || (reinterpret_cast<uintptr_t>(p.bias2) & 7) == 0);
        constexpr uint64_t KA = TA ? (UK * 128) >> 4 : 2, KB = TB ? (UK * 128) >> 4 : 2;   // descriptor advance per wgmma K step
        const uint64_t da0 = wgmma_desc(smem_u32(smem + c * (64 * 128)), BK * 128, 1024);
        const uint64_t db0 = wgmma_desc(smem_u32(smem + TILE_BYTES), BK * 128, 1024);
        auto release = [&](int s) {
            if (lane == 0) {
                if (NCTA == 2) {
#pragma unroll
                    for (int r = 0; r < 2; ++r) mbar_arrive_cluster(mapa_shared(smem_u32(&empty[s]), r));
                } else {
                    mbar_arrive(&empty[s]);
                }
            }
        };
        float acc[BN_ / 2];
        int it = 0;
        for (int w = wid0; w < n_work; w += wstep) {
            const int split = w / n_tiles, tile = w - split * n_tiles;
            const int tile_m = tile / tiles_n, tile_n = tile - tile_m * tiles_n;
            const int kb0 = split * kb_per_split, kb1 = min(num_kb_all, kb0 + kb_per_split);
            if (kb1 <= kb0) continue;                                 // empty split-K range: nothing to add
            for (int kb = kb0; kb < kb1; ++kb, ++it) {
                const int s = it % ST, ph = (it / ST) & 1;
                mbar_wait(&full[s], ph, p.status, 113);
                const uint64_t so = static_cast<uint64_t>(s) * (C::STAGE_BYTES >> 4);
                wgmma_fence_acc<BN_ / 2>(acc);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < BK / UK; ++k)
                    wgmma_k<BN_, FMT, TA, TB>(acc, da0 + so + k * KA, db0 + so + k * KB, (kb > kb0 || k > 0) ? 1u : 0u);
                wgmma_commit();
                wgmma_wait<1>();                                      // the previous stage's wgmmas have read their operands
                wgmma_fence_acc<BN_ / 2>(acc);
                if (kb > kb0) release((it - 1) % ST);
            }
            wgmma_wait<0>();
            wgmma_fence_acc<BN_ / 2>(acc);
            release((it - 1) % ST);
#ifndef FT_GEMM_NO_STORE                            // tools/gemm_shapes.py --mainloop: the main loop alone
            const int mb = tile_m * TM + rank * BM + c * 64;             // < M, an int
            if (p.tma_c) {
                epi_staged<BN_>(p, &tmC32, &tmC16, acc, alpha, smem_u32(epi) + c * (2 * EPI_SLOT), c, mb, tile_n * BN_);
            } else {
                const long long m0 = static_cast<long long>(mb) + wq * 16 + (lane >> 2);
                const int n0 = tile_n * BN_ + 2 * (lane & 3);
#pragma unroll
                for (int j = 0; j < BN_ / 8; ++j) {
                    epi_pair(p, m0, n0 + 8 * j, acc[4 * j], acc[4 * j + 1], alpha, vec2);
                    epi_pair(p, m0 + 8, n0 + 8 * j, acc[4 * j + 2], acc[4 * j + 3], alpha, vec2);
                }
            }
#endif
        }
        if (p.tma_c && (threadIdx.x & 127) == 0) bulk_wait_all();   // staged chunks stay in shared memory until stored
    }
    if (NCTA == 2) cluster_sync_all();              // no CTA exits while its peer may still arrive on its barriers
}

template <int FMT, int BN_, int NCTA, int TA, bool PP = false>
const void* gemm_kernel_tb(int tb) {
    if constexpr (FMT == FMT_TF32) return reinterpret_cast<const void*>(gemm2_kernel<FMT, BN_, NCTA, TA, 0, PP>);   // K-major only
    else return tb ? reinterpret_cast<const void*>(gemm2_kernel<FMT, BN_, NCTA, TA, 1, PP>) : reinterpret_cast<const void*>(gemm2_kernel<FMT, BN_, NCTA, TA, 0, PP>);
}

// The launchable instantiations of one operand format and A layout (explicitly instantiated in gemm_inst_*.cu, one
// translation unit each, so the build compiles them in parallel).
template <int FMT, int TA>
const void* gemm_kernel_ptr(int bn, int ncta, int tb, int pp) {
    if (pp) return gemm_kernel_tb<FMT, 128, 1, TA, true>(tb);
    if (ncta == 2) return gemm_kernel_tb<FMT, 256, 2, TA>(tb);
    return bn == 256 ? gemm_kernel_tb<FMT, 256, 1, TA>(tb) : gemm_kernel_tb<FMT, 128, 1, TA>(tb);
}

}  // namespace ft
