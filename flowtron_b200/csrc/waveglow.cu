// WaveGlow.infer (tacotron2/waveglow/glow.py:251-293 of the reference) for the shipped configuration: 80 mel channels,
// n_group 8, WN with 256 channels and kernel 3.  See DESIGN.md §4.13.
//
// Layout: every activation lives time-major in one packed row grid.  One row is one group of 8 audio samples; the rows
// of an utterance are contiguous and utterances are separated by WG_GUARD (= the largest dilation, 2^7) rows that no
// kernel ever writes and whose fp16 hidden state is zero.  The dilated k=3 convolution of WN layer i is then ONE GEMM
// whose A operand runs over four K segments -- the hidden state shifted by -d, 0, +d rows and the upsampled spectrogram
// row -- and the guard rows supply the convolution's zero padding, for any batch and any lengths.
//
// Kernels:
//   wg_prep_kernel     mel [B,80,F] fp32 -> time-major fp16 frame grid (3 zero rows ahead of each utterance) and the row maps
//   wg_gemm_kernel     mma.sync m16n8k16 fp16 GEMM, fp32 accumulate, multi-segment A, three epilogues:
//                        UP    ConvTranspose1d upsample: bias, fp16 store of 32 grid rows per mel frame
//                        GATE  in_layer + cond_layer: columns (2c, 2c+1) hold (tanh, sigmoid) inputs of channel c,
//                              writes fp16 tanh(x0) * sigmoid(x1) to column c
//                        RES   res_skip_layer: h32 += first C columns (and refreshes the fp16 shadow h16), skip32 (+)= rest
//   wg_tail_kernel     per flow, one warp per row: end conv from the fp32 skip sum, affine inverse, inverse 1x1 conv,
//                      noise injection and the next flow's start conv (or the audio store after the last flow)
// fp16 tensor-core operands; hidden residual, skip sum, flow state, affine step and the 1x1 inverse stay fp32.
#include <cuda_fp16.h>

#include <algorithm>

#include "ptx.cuh"
#include "ft_internal.h"
#include "../../include/flowtron_b200.h"

namespace ft {

constexpr int WG_C = 256;             // WN n_channels
constexpr int WG_SPECT = 640;         // n_mel * n_group: conditioning channels per group row
constexpr int WG_MEL = 80;
constexpr int WG_MEL_LD = 96;         // frame-grid row: 80 mel channels zero-padded to the GEMM's K block
constexpr int WG_UP_N = 32 * WG_SPECT;   // upsample GEMM columns: 256 samples x 80 channels of one frame
constexpr int WG_GUARD = 128;
constexpr int WG_MAX_B = 128;

// ------------------------------------------------------------------------------------------------ GEMM
constexpr int GB_M = 128, GB_N = 128, GB_K = 32, G_STAGES = 4, G_THREADS = 256;
constexpr int G_LDS = GB_K + 8;                         // smem row pitch (halves): 80 B, ldmatrix conflict-free
constexpr int G_STAGE_HALVES = (GB_M + GB_N) * G_LDS;
constexpr int G_SMEM = G_STAGES * G_STAGE_HALVES * 2;

enum { WG_EPI_UP = 0, WG_EPI_GATE = 1, WG_EPI_RES = 2, WG_EPI_GATE_BWD = 3 };

struct WgSeg {
    const __half* base;   // row-major [rows, ld]
    long long rows, ld;
    int shift;            // A row m reads base row m + shift (out of range: zeros)
    int k;                // columns taken from this segment (multiple of GB_K)
};

struct WgGemmParams {
    int M, N, K, nseg;
    WgSeg seg[4];
    const __half* W;      // [N, K] fp16 (K contiguous)
    const float* bias;    // [N]
    const int* rowmap;    // [M]: < 0 = row m is not written; UP: the destination row of frame row m
    const int* m_live;    // optional device row count <= M (the infer plan's totals): rows and tiles past it are skipped
    int mode;
    __half* out16; long long ld16;            // UP, GATE
    float* h32; __half* h16; float* skip32;   // RES ([rows, C] each)
    int res_cols;                             // RES: columns [0, res_cols) update the hidden state, the rest the skip sum
    int skip_store;                           // RES: 1 = skip32 = x (first layer), 0 = skip32 += x
    __half* pre16;                            // GATE: optional store of the pre-activations [rows, 2C] (training forward);
                                              // GATE_BWD: the saved pre-activations it reads
};

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool pred) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(pred ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}

__device__ __forceinline__ __half sat_half(float x) { return __float2half_rn(fminf(fmaxf(x, -65504.f), 65504.f)); }

__device__ __forceinline__ void wg_epi_pair(const WgGemmParams& p, int M, int m, int n, float v0, float v1) {
    if (m >= M) return;
    const int info = __ldg(p.rowmap + m);
    if (info < 0) return;                                     // guard / padding rows are never written
    const int row = p.mode == WG_EPI_UP ? info : m;           // UP: a frame row lands on its first group row
    if (p.mode == WG_EPI_GATE_BWD) {
        // v0, v1 = d acts of channels n, n+1 -> d pre-activations (interleaved like the forward's columns) and acts
        const long long o = static_cast<long long>(row) * 2 * WG_C + 2 * n;
        const uint2 raw = *reinterpret_cast<const uint2*>(p.pre16 + o);
        const __half2 q0 = *reinterpret_cast<const __half2*>(&raw.x), q1 = *reinterpret_cast<const __half2*>(&raw.y);
        const float t0 = tanh_f(__low2float(q0)), s0 = sigmoid_f(__high2float(q0));
        const float t1 = tanh_f(__low2float(q1)), s1 = sigmoid_f(__high2float(q1));
        const __half2 d0 = __halves2half2(sat_half(v0 * s0 * (1.f - t0 * t0)), sat_half(v0 * t0 * s0 * (1.f - s0)));
        const __half2 d1 = __halves2half2(sat_half(v1 * s1 * (1.f - t1 * t1)), sat_half(v1 * t1 * s1 * (1.f - s1)));
        uint2 outv;
        outv.x = *reinterpret_cast<const uint32_t*>(&d0); outv.y = *reinterpret_cast<const uint32_t*>(&d1);
        *reinterpret_cast<uint2*>(p.out16 + o) = outv;
        *reinterpret_cast<__half2*>(p.h16 + static_cast<long long>(row) * WG_C + n) = __halves2half2(sat_half(t0 * s0), sat_half(t1 * s1));
        return;
    }
    const float2 b = __ldg(reinterpret_cast<const float2*>(p.bias + n));
    const float x0 = v0 + b.x, x1 = v1 + b.y;
    if (p.mode == WG_EPI_GATE) {
        p.out16[static_cast<long long>(row) * p.ld16 + (n >> 1)] = sat_half(tanh_f(x0) * sigmoid_f(x1));
        if (p.pre16)
            *reinterpret_cast<__half2*>(p.pre16 + static_cast<long long>(row) * 2 * WG_C + n) = __halves2half2(sat_half(x0), sat_half(x1));
    } else if (p.mode == WG_EPI_UP) {
        *reinterpret_cast<__half2*>(p.out16 + static_cast<long long>(row) * p.ld16 + n) = __halves2half2(sat_half(x0), sat_half(x1));
    } else if (n < p.res_cols) {
        const long long o = static_cast<long long>(row) * WG_C + n;
        float2* h = reinterpret_cast<float2*>(p.h32 + o);
        float2 v = *h;
        v.x += x0; v.y += x1;
        *h = v;
        *reinterpret_cast<__half2*>(p.h16 + o) = __halves2half2(sat_half(v.x), sat_half(v.y));
    } else {
        float2* s = reinterpret_cast<float2*>(p.skip32 + static_cast<long long>(row) * WG_C + (n - p.res_cols));
        if (p.skip_store) {
            *s = make_float2(x0, x1);
        } else {
            float2 v = *s;
            v.x += x0; v.y += x1;
            *s = v;
        }
    }
}

__global__ void __launch_bounds__(G_THREADS, 2) wg_gemm_kernel(const __grid_constant__ WgGemmParams p) {
    extern __shared__ __align__(16) __half g_smem[];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int wm = warp & 1, wn = warp >> 1;                  // warp tile: 64 rows x 32 columns
    const int n0 = blockIdx.x * GB_N;
    const int m0 = blockIdx.y * GB_M;
    const int M = p.m_live ? min(__ldg(p.m_live), p.M) : p.M;
    if (m0 >= M) return;                                      // block-uniform: a tile wholly past the live rows
    const int nkb = p.K / GB_K;

    auto load_stage = [&](int stage, int kb) {
        __half* sa = g_smem + stage * G_STAGE_HALVES;
        __half* sb = sa + GB_M * G_LDS;
        // which A segment holds this K block (segment widths are multiples of GB_K)
        int kk = kb * GB_K;
        const __half* base = p.seg[0].base;
        long long rows = p.seg[0].rows, ld = p.seg[0].ld;
        int shift = p.seg[0].shift, seg_k = p.seg[0].k;
#pragma unroll
        for (int s = 1; s < 4; ++s) {
            if (s < p.nseg && kk >= seg_k) {
                kk -= seg_k;
                base = p.seg[s].base; rows = p.seg[s].rows; ld = p.seg[s].ld; shift = p.seg[s].shift; seg_k = p.seg[s].k;
            }
        }
#pragma unroll
        for (int i = 0; i < 2; ++i) {                         // 128 rows x 4 chunks of 16 B, A and B
            const int c = tid + i * G_THREADS;
            const int r = c >> 2, q = c & 3;
            const long long ar = static_cast<long long>(m0 + r) + shift;
            const bool ok = (m0 + r < M) && ar >= 0 && ar < rows;
            const __half* src = ok ? base + ar * ld + kk + q * 8 : base;
            cp_async16(smem_u32(sa + r * G_LDS + q * 8), src, ok);
            const __half* wsrc = p.W + static_cast<long long>(n0 + r) * p.K + kb * GB_K + q * 8;
            cp_async16(smem_u32(sb + r * G_LDS + q * 8), wsrc, true);
        }
    };

    float acc[4][4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[i][j][e] = 0.f;

#pragma unroll
    for (int s = 0; s < G_STAGES - 1; ++s) {
        if (s < nkb) load_stage(s, s);
        cp_async_commit();
    }
    for (int kb = 0; kb < nkb; ++kb) {
        cp_async_wait<G_STAGES - 2>();
        __syncthreads();                                      // stage kb landed; stage kb-1 is no longer read
        const int nxt = kb + G_STAGES - 1;
        if (nxt < nkb) load_stage(nxt % G_STAGES, nxt);
        cp_async_commit();
        const __half* sa = g_smem + (kb % G_STAGES) * G_STAGE_HALVES;
        const __half* sb = sa + GB_M * G_LDS;
#pragma unroll
        for (int k16 = 0; k16 < GB_K; k16 += 16) {
            uint32_t af[4][4], bf[4][2];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int r = wm * 64 + i * 16 + (lane & 15);
                ldsm_x4(smem_u32(sa + r * G_LDS + k16 + (lane >> 4) * 8), af[i][0], af[i][1], af[i][2], af[i][3]);
            }
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                const int r = wn * 32 + j * 16 + (lane & 7) + ((lane >> 4) << 3);
                ldsm_x4(smem_u32(sb + r * G_LDS + k16 + ((lane >> 3) & 1) * 8), bf[2 * j][0], bf[2 * j][1], bf[2 * j + 1][0],
                        bf[2 * j + 1][1]);
            }
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) mma16816(acc[i][j], af[i][0], af[i][1], af[i][2], af[i][3], bf[j][0], bf[j][1]);
        }
    }
    cp_async_wait<0>();

#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int m = m0 + wm * 64 + i * 16 + (lane >> 2);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int n = n0 + wn * 32 + j * 8 + 2 * (lane & 3);
            wg_epi_pair(p, M, m, n, acc[i][j][0], acc[i][j][1]);
            wg_epi_pair(p, M, m + 8, n, acc[i][j][2], acc[i][j][3]);
        }
    }
}

static int launch_wg_gemm(const WgGemmParams& p, cudaStream_t st) {
    if (p.N % GB_N || p.K % GB_K) return ft_set_error("waveglow gemm: N must be a multiple of 128 and K of 32");
    static bool attr = false;
    if (!attr) {
        if (cudaFuncSetAttribute(wg_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, G_SMEM) != cudaSuccess)
            return ft_set_error("waveglow gemm: shared-memory opt-in failed");
        attr = true;
    }
    const dim3 grid(p.N / GB_N, (p.M + GB_M - 1) / GB_M);
    static const char* const names[] = {"wg_upsample", "wg_in_layer", "wg_res_skip", "wg_gate_bwd"};
    TimeScope ts(names[p.mode], p.M, p.N, p.K, st);
    wg_gemm_kernel<<<grid, G_THREADS, G_SMEM, st>>>(p);
    ft_count_launch(1);
    return ft_check_launch("wg_gemm_kernel");
}

// ------------------------------------------------------------------------------------------------ plan and prep
// The packed row layout of a batch.  It lives in device memory, written by wg_plan_kernel from the frame counts, so the
// counts may themselves be device data (a CUDA graph replays with new lengths); the host only sizes grids and scratch
// for the largest layout the counts can give.
struct WgBatch {
    int B, Tg_max;
    int mrows, grows;            // frame-grid rows (= mbase[B]); group-grid rows (gbase[B] + the trailing guard)
    int frames[WG_MAX_B];        // clamped to 1..F_max
    int mbase[WG_MAX_B + 1];     // first frame-grid row of utterance b (its 3 zero rows come first); mbase[B] = rows
    int gbase[WG_MAX_B + 1];     // first group-grid row of utterance b; gbase[B] = end of the last utterance
};

struct WgFrames { int f[WG_MAX_B]; };   // host frame counts, passed by value

constexpr int WG_PLAN_THREADS = WG_MAX_B + 32;

// One CTA: thread b <= B sums the rows of the utterances before b.  Counts come from `dev` (int32 [B] in device memory)
// or, when it is null, from `host`; every count is clamped to 1..F_max so no length can address past the grids.
__global__ void __launch_bounds__(WG_PLAN_THREADS) wg_plan_kernel(const __grid_constant__ WgFrames host, const int* __restrict__ dev,
                                                                  int B, int F_max, int Tg_max, WgBatch* __restrict__ bt) {
    __shared__ int s_f[WG_MAX_B];
    const int t = threadIdx.x;
    if (t < B) s_f[t] = min(max(dev ? __ldg(dev + t) : host.f[t], 1), F_max);
    __syncthreads();
    if (t > B) return;
    int m = 0, g = WG_GUARD;
    for (int j = 0; j < t; ++j) {
        m += s_f[j] + 3;
        g += 32 * s_f[j] + WG_GUARD;
    }
    if (t < B) {
        bt->frames[t] = s_f[t];
        bt->mbase[t] = m;
        bt->gbase[t] = g;
    } else {
        bt->B = B; bt->Tg_max = Tg_max;
        bt->mbase[B] = m; bt->gbase[B] = g - WG_GUARD;
        bt->mrows = m; bt->grows = g;
    }
}

__device__ __forceinline__ int find_utt(const int* base, int B, int r) {   // largest b with base[b] <= r
    int lo = 0, hi = B - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (base[mid] <= r) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// mel [B, 80, F_max] fp32 -> mel16 [mrows, 96]; up_rowmap [mrows]; rowinfo [grows] = b * Tg_max + g, or -1 for guard rows.
// The grid is sized for the host's bound on the layout; the loop runs over the plan's rows.
__global__ void wg_prep_kernel(const WgBatch* __restrict__ plan, const float* __restrict__ mel, int F_max, __half* __restrict__ mel16,
                               int* __restrict__ up_rowmap, int* __restrict__ rowinfo) {
    __shared__ WgBatch bt;
    for (int i = threadIdx.x; i < static_cast<int>(sizeof(WgBatch) / 4); i += blockDim.x)
        reinterpret_cast<int*>(&bt)[i] = __ldg(reinterpret_cast<const int*>(plan) + i);
    __syncthreads();
    const int mrows = bt.mrows, grows = bt.grows;
    const long long n_mel = static_cast<long long>(mrows) * WG_MEL_LD;
    const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n_mel + mrows + grows; i += stride) {
        if (i < n_mel) {
            const int r = static_cast<int>(i / WG_MEL_LD), c = static_cast<int>(i % WG_MEL_LD);
            const int b = find_utt(bt.mbase, bt.B, r);
            const int f = r - bt.mbase[b] - 3;
            float v = 0.f;
            if (f >= 0 && c < WG_MEL) v = __ldg(mel + (static_cast<long long>(b) * WG_MEL + c) * F_max + f);
            mel16[i] = __float2half_rn(v);
        } else if (i < n_mel + mrows) {
            const int r = static_cast<int>(i - n_mel);
            const int b = find_utt(bt.mbase, bt.B, r);
            const int f = r - bt.mbase[b] - 3;
            up_rowmap[r] = f >= 0 ? bt.gbase[b] + 32 * f : -1;
        } else {
            const int r = static_cast<int>(i - n_mel - mrows);
            int info = -1;
            if (r >= bt.gbase[0] && r < bt.gbase[bt.B]) {
                const int b = find_utt(bt.gbase, bt.B, r);
                const int g = r - bt.gbase[b];
                if (g < 32 * bt.frames[b] && g < bt.Tg_max) info = b * bt.Tg_max + g;   // training: Tg_max = N / 8
            }
            rowinfo[r] = info;
        }
    }
}

// ------------------------------------------------------------------------------------------------ flow tail
constexpr int T_THREADS = 256, T_ROWS_PER_WARP = 8;

struct WgTailParams {
    int R;                          // grid rows: the host's bound
    const int* live_rows;           // device: the plan's grid rows (<= R); rows past it are skipped
    const int* rowinfo;             // [R]
    float* state;                   // [R, 8] fp32 flow state; the c live channels of a flow sit at positions [8 - c, 8)
    // the flow being finished (cur = 0 for the head launch, which only draws the initial noise)
    int cur, o, nh;                 // o = 8 - c: first live position; nh = n_half
    const float* skip32;            // [R, C]
    const float* end_w;             // [2 nh, C]
    const float* end_b;             // [2 nh]
    const float* inv_w;             // [c, c] inverse of the flow's 1x1 conv
    // noise: positions [inj_lo, inj_hi) = sigma * noise[b, pos, g]
    int inj_lo, inj_hi;
    const float* noise; int Tg_max; float sigma;
    // next flow's start conv from positions [o_next, o_next + nh_next), or the audio store
    int next, o_next, nh_next;
    const float* start_w;           // [C, nh_next]
    const float* start_b;           // [C]
    float* h32; __half* h16;        // [R, C]
    float* audio;                   // [B, Tg_max * 8] (next == 0)
};

__global__ void __launch_bounds__(T_THREADS) wg_tail_kernel(const __grid_constant__ WgTailParams p) {
    __shared__ float s_end[8 * WG_C];
    __shared__ float s_start[WG_C * 4];
    __shared__ float s_misc[64 + 8 + WG_C];    // inv_w, end_b, start_b
    float* s_inv = s_misc;
    float* s_endb = s_misc + 64;
    float* s_startb = s_misc + 72;
    const int c = 8 - p.o;
    const int R = min(p.R, __ldg(p.live_rows));
    if (static_cast<int>(blockIdx.x) * (T_THREADS / 32) * T_ROWS_PER_WARP >= R) return;   // block-uniform
    if (p.cur) {
        for (int i = threadIdx.x; i < 2 * p.nh * WG_C; i += T_THREADS) s_end[i] = p.end_w[i];
        for (int i = threadIdx.x; i < c * c; i += T_THREADS) s_inv[i] = p.inv_w[i];
        if (threadIdx.x < 2 * p.nh) s_endb[threadIdx.x] = p.end_b[threadIdx.x];
    }
    if (p.next) {
        for (int i = threadIdx.x; i < WG_C * p.nh_next; i += T_THREADS) s_start[i] = p.start_w[i];
        for (int i = threadIdx.x; i < WG_C; i += T_THREADS) s_startb[i] = p.start_b[i];
    }
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    __shared__ float s_x[T_THREADS / 32][8], s_y[T_THREADS / 32][8], s_out[T_THREADS / 32][8];
    float* xs = s_x[warp];
    float* ys = s_y[warp];
    float* so = s_out[warp];
    const int r0 = (blockIdx.x * (T_THREADS / 32) + warp) * T_ROWS_PER_WARP;
    for (int r = r0; r < r0 + T_ROWS_PER_WARP && r < R; ++r) {
        const int info = __ldg(p.rowinfo + r);
        if (info < 0) continue;                                   // warp-uniform
        const int b = info / p.Tg_max, g = info - b * p.Tg_max;
        // lanes 0..7 own the 8 state positions; the warp shares them through shared memory
        if (lane < 8) xs[lane] = p.state[static_cast<long long>(r) * 8 + lane];
        if (p.cur) {
            // end conv: lane owns channels [8 lane, 8 lane + 8) of the skip sum
            const float4* skp = reinterpret_cast<const float4*>(p.skip32 + static_cast<long long>(r) * WG_C + lane * 8);
            const float4 s0 = skp[0], s1 = skp[1];
            const float sk[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                if (j < 2 * p.nh) {
                    float a = 0.f;
#pragma unroll
                    for (int e = 0; e < 8; ++e) a = fmaf(s_end[j * WG_C + lane * 8 + e], sk[e], a);
#pragma unroll
                    for (int off = 16; off; off >>= 1) a += __shfl_xor_sync(0xffffffffu, a, off);
                    if (lane == j) so[j] = a + s_endb[j];
                }
            }
            __syncwarp();
            // affine coupling inverse on audio_1 = positions [o + nh, 8): (audio_1 - b) / exp(log_s)
            if (lane < 8) {
                float v = xs[lane];
                const int i = lane - p.o - p.nh;
                if (i >= 0) v = (v - so[i]) * __expf(-so[p.nh + i]);
                ys[lane] = v;
            }
            __syncwarp();
            // inverse 1x1 conv over the c live positions [o, 8)
            if (lane < 8) {
                float v = ys[lane];
                if (lane >= p.o) {
                    v = 0.f;
                    for (int j = 0; j < c; ++j) v = fmaf(s_inv[(lane - p.o) * c + j], ys[p.o + j], v);
                }
                xs[lane] = v;
            }
        }
        if (lane >= p.inj_lo && lane < p.inj_hi)
            xs[lane] = p.sigma * __ldg(p.noise + (static_cast<long long>(b) * 8 + lane) * p.Tg_max + g);
        __syncwarp();
        if (p.next) {
            float h[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const int ch = lane * 8 + e;
                float a = s_startb[ch];
#pragma unroll
                for (int i = 0; i < 4; ++i)
                    if (i < p.nh_next) a = fmaf(s_start[ch * p.nh_next + i], xs[p.o_next + i], a);
                h[e] = a;
            }
            const long long o = static_cast<long long>(r) * WG_C + lane * 8;
            float4* hp = reinterpret_cast<float4*>(p.h32 + o);
            hp[0] = make_float4(h[0], h[1], h[2], h[3]);
            hp[1] = make_float4(h[4], h[5], h[6], h[7]);
            const __half2 q0 = __halves2half2(sat_half(h[0]), sat_half(h[1])), q1 = __halves2half2(sat_half(h[2]), sat_half(h[3]));
            const __half2 q2 = __halves2half2(sat_half(h[4]), sat_half(h[5])), q3 = __halves2half2(sat_half(h[6]), sat_half(h[7]));
            uint4 pk;
            pk.x = *reinterpret_cast<const uint32_t*>(&q0); pk.y = *reinterpret_cast<const uint32_t*>(&q1);
            pk.z = *reinterpret_cast<const uint32_t*>(&q2); pk.w = *reinterpret_cast<const uint32_t*>(&q3);
            *reinterpret_cast<uint4*>(p.h16 + o) = pk;
            if (lane < 8) p.state[static_cast<long long>(r) * 8 + lane] = xs[lane];
        } else if (lane < 8) {
            p.audio[(static_cast<long long>(b) * p.Tg_max + g) * 8 + lane] = xs[lane];
        }
        __syncwarp();                                             // xs is reused by the next row
    }
}

static int launch_wg_tail(const WgTailParams& p, cudaStream_t st) {
    const int rows_per_block = (T_THREADS / 32) * T_ROWS_PER_WARP;
    const int grid = (p.R + rows_per_block - 1) / rows_per_block;
    TimeScope ts("wg_tail", p.R, p.cur, p.next, st);
    wg_tail_kernel<<<grid, T_THREADS, 0, st>>>(p);
    ft_count_launch(1);
    return ft_check_launch("wg_tail_kernel");
}

// ------------------------------------------------------------------------------------------------ driver
// Host side of a batch, for infer and training alike: the flows' channel schedule and the bound on the row layout (the
// exact layout for host frame counts; every utterance at F_max when the counts are device data) that sizes grids and
// workspaces, with the host counts for wg_plan_kernel.  Tg_max is the group rows of an utterance in noise / audio (infer:
// 32 F_max) or in z (training: N / 8, and the rows after it are padding).
struct WgGrid {
    int B, F_max, Tg_max, nf, nl, mrows, grows;
    int c[FT_WG_MAX_FLOWS];      // live channels of flow k (its 1x1 conv is c x c), n_half = c / 2
    WgFrames fr;
};

// d->frames == NULL: the counts arrive in device memory, and the layout is bounded by F_max for every utterance.
static int wg_grid(const FtWaveGlowDesc* d, int Tg_max, WgGrid* G) {
    if (d->n_mel != WG_MEL || d->n_group != 8 || d->n_channels != WG_C || d->kernel_size != 3)
        return ft_set_error("waveglow: only n_mel 80, n_group 8, n_channels 256, kernel_size 3 are built");
    if (d->n_flows < 1 || d->n_flows > FT_WG_MAX_FLOWS || d->n_layers < 1 || d->n_layers > FT_WG_MAX_LAYERS)
        return ft_set_error("waveglow: n_flows must be 1..16 and n_layers 1..8");
    if (d->n_early_every < 1 || d->n_early_size < 0 || d->n_early_size % 2)
        return ft_set_error("waveglow: n_early_every >= 1 and an even n_early_size >= 0 required");
    const int n_early = (d->n_flows - 1) / d->n_early_every;
    if (8 - n_early * d->n_early_size < 2) return ft_set_error("waveglow: early outputs leave fewer than 2 channels");
    if (d->B < 1 || d->B > WG_MAX_B) return ft_set_error("waveglow: batch must be 1..128");
    G->B = d->B; G->F_max = d->F_max; G->Tg_max = Tg_max; G->nf = d->n_flows; G->nl = d->n_layers;
    for (int k = 0, c = 8; k < G->nf; ++k) {
        if (k > 0 && k % d->n_early_every == 0) c -= d->n_early_size;
        G->c[k] = c;
    }
    long long m = 0, g = WG_GUARD;
    for (int b = 0; b < d->B; ++b) {
        const int f = d->frames ? d->frames[b] : d->F_max;
        if (f < 1 || f > d->F_max) return ft_set_error("waveglow: frames[b] must be in 1..F_max");
        G->fr.f[b] = f;
        m += f + 3;
        g += 32LL * f + WG_GUARD;
        if (g > (1LL << 30)) return ft_set_error("waveglow: batch too long");
    }
    G->mrows = static_cast<int>(m);
    G->grows = static_cast<int>(g);
    return 0;
}

static int wg_infer_grid(const FtWaveGlowDesc* d, WgGrid* G) {
    return d ? wg_grid(d, 32 * d->F_max, G) : ft_set_error("waveglow: null descriptor");
}

// The prep's outputs, the first regions of the infer scratch and of the training `saved`: the planned layout, the fp16
// frame grid, the two row maps and the upsampled spectrogram.
struct WgPrep {
    WgBatch* batch; __half* mel16; int* uprow; int* rowinfo; __half* spect;
    void plan(Workspace& ws, const WgGrid& g) {
        const size_t R = g.grows;
        batch = ws.get<WgBatch>(1);
        mel16 = ws.get<__half>(static_cast<size_t>(g.mrows) * WG_MEL_LD);
        uprow = ws.get<int>(g.mrows);
        rowinfo = ws.get<int>(R);
        spect = ws.get<__half>(R * WG_SPECT);
    }
};

struct WgInferScratch {
    WgPrep in;
    float* h32; __half* h16; __half* acts; float* skip; float* state;
    void plan(Workspace& ws, const WgGrid& g) {
        const size_t R = g.grows;
        in.plan(ws, g);
        h32 = ws.get<float>(R * WG_C);
        h16 = ws.get<__half>(R * WG_C);
        acts = ws.get<__half>(R * WG_C);
        skip = ws.get<float>(R * WG_C);
        state = ws.get<float>(R * 8);
    }
};

// Plan P of the workspace at `base`; wg_bytes: its size.
template <typename P> static P wg_carve(const void* base, const WgGrid& g) {
    Workspace ws;
    ws.base = static_cast<uint8_t*>(const_cast<void*>(base));
    P p;
    p.plan(ws, g);
    return p;
}
template <typename P> static size_t wg_bytes(const WgGrid& g) {
    Workspace ws;
    P p;
    p.plan(ws, g);
    return ws.off;
}

// The plan (frames_dev: int32 [B] device counts, or null for the grid's host counts), then the prep over it.
static int launch_wg_plan_prep(const WgGrid& g, const WgPrep& in, const int* frames_dev, const float* mel, cudaStream_t st) {
    {
        TimeScope ts("wg_plan", g.B, g.F_max, frames_dev != nullptr, st);
        wg_plan_kernel<<<1, WG_PLAN_THREADS, 0, st>>>(g.fr, frames_dev, g.B, g.F_max, g.Tg_max, in.batch);
        ft_count_launch(1);
        if (ft_check_launch("wg_plan_kernel")) return -1;
    }
    const long long work = static_cast<long long>(g.mrows) * (WG_MEL_LD + 1) + g.grows;
    const int grid = static_cast<int>(std::min<long long>((work + 255) / 256, 4096));
    TimeScope ts("wg_prep", g.mrows, g.grows, 0, st);
    wg_prep_kernel<<<grid, 256, 0, st>>>(in.batch, mel, g.F_max, in.mel16, in.uprow, in.rowinfo);
    ft_count_launch(1);
    return ft_check_launch("wg_prep_kernel");
}

// The WN forward GEMMs, shared by infer and the training forward (W: FtWaveGlowWeights or FtWaveGlowTrainWeights).
// m_live: the plan's live row count, or null to run every row of the bound.
// Upsample: frame row f = frames f-3..f (A segments shifted 0..-3) -> 32 group rows of 640 channels.
template <typename W>
static int wg_upsample(const WgGrid& g, const WgPrep& in, const W* w, const int* m_live, cudaStream_t st) {
    WgGemmParams p = {};
    p.M = g.mrows; p.N = WG_UP_N; p.K = 4 * WG_MEL_LD; p.nseg = 4;
    for (int j = 0; j < 4; ++j) p.seg[j] = WgSeg{in.mel16, g.mrows, WG_MEL_LD, -j, WG_MEL_LD};
    p.W = static_cast<const __half*>(w->up_w); p.bias = w->up_b; p.rowmap = in.uprow; p.m_live = m_live; p.mode = WG_EPI_UP;
    p.out16 = in.spect; p.ld16 = WG_SPECT;
    return launch_wg_gemm(p, st);
}

// Flow k's WN layers, each a GATE GEMM (in_layer + cond_layer) and a RES GEMM (res_skip_layer).  Layer i reads its fp16
// input at h16 + i h_step and its RES writes layer i + 1's there (h_step 0: infer's one buffer; training keeps every
// layer's input).  pre: null, or where GATE stores layer i's pre-activations, at pre + i R 2C.
template <typename W>
static int wg_flow_wn(const WgGrid& g, const WgPrep& in, const W* w, int k, __half* h16, long long h_step, __half* pre,
                      __half* acts, float* h32, float* skip, const int* m_live, cudaStream_t st) {
    const long long R = g.grows;
    for (int i = 0; i < g.nl; ++i) {
        const int dil = 1 << i;
        const bool last = i == g.nl - 1;
        __half* hin = h16 + i * h_step;
        WgGemmParams p = {};
        p.M = static_cast<int>(R); p.N = 2 * WG_C; p.K = 3 * WG_C + WG_SPECT; p.nseg = 4;
        p.seg[0] = WgSeg{hin, R, WG_C, -dil, WG_C};
        p.seg[1] = WgSeg{hin, R, WG_C, 0, WG_C};
        p.seg[2] = WgSeg{hin, R, WG_C, dil, WG_C};
        p.seg[3] = WgSeg{in.spect, R, WG_SPECT, 0, WG_SPECT};
        p.W = static_cast<const __half*>(w->in_w[k][i]); p.bias = w->in_b[k][i]; p.rowmap = in.rowinfo; p.m_live = m_live;
        p.mode = WG_EPI_GATE; p.out16 = acts; p.ld16 = WG_C; p.pre16 = pre ? pre + i * R * 2 * WG_C : nullptr;
        if (launch_wg_gemm(p, st)) return -1;
        WgGemmParams q = {};
        q.M = static_cast<int>(R); q.N = last ? WG_C : 2 * WG_C; q.K = WG_C; q.nseg = 1;
        q.seg[0] = WgSeg{acts, R, WG_C, 0, WG_C};
        q.W = static_cast<const __half*>(w->rs_w[k][i]); q.bias = w->rs_b[k][i]; q.rowmap = in.rowinfo; q.m_live = m_live;
        q.mode = WG_EPI_RES; q.h32 = h32; q.h16 = last ? hin : hin + h_step; q.skip32 = skip; q.res_cols = last ? 0 : WG_C;
        q.skip_store = i == 0;
        if (launch_wg_gemm(q, st)) return -1;
    }
    return 0;
}

// ------------------------------------------------------------------------------------------------ training
// WaveGlow.forward (glow.py:196-245, the z direction) with its saved activations, and its backward.  See DESIGN.md §4.21.
// The forward runs on the same grid, prep, upsample and GATE / RES GEMMs as infer; the GATE epilogue also stores the
// pre-activations, and each layer's RES epilogue writes the next layer's fp16 input into its own saved slot.
constexpr float WG_GRAD_TARGET = 64.f;   // per-flow loss scale: S * max|d skip| ~ 64 (headroom 2^10 below fp16's max)

// forward -> backward
struct WtSaved {
    WgPrep in;
    float* x;          // [nf][R, 8] flow inputs (before the 1x1 conv), fp32
    float* skip;       // [nf][R, C] WN skip sums, fp32
    __half* h16;       // [nf][nl][R, C] WN layer inputs, fp16, zero guard rows
    __half* pre;       // [nf][nl][R, 2C] gate pre-activations, fp16, interleaved like in_w's rows
    void plan(Workspace& ws, const WgGrid& g) {
        const size_t R = g.grows, nf = g.nf, nfl = nf * g.nl;
        in.plan(ws, g);
        x = ws.get<float>(nf * R * 8);
        skip = ws.get<float>(nf * R * WG_C);
        h16 = ws.get<__half>(nfl * R * WG_C);
        pre = ws.get<__half>(nfl * R * 2 * WG_C);
    }
};

struct WtScratch {
    float* h32; __half* acts; float* state; float* dstate; float* dout; float* dy; __half* dskip; __half* g16; float* g32;
    __half* dx; float* dsp32; __half* dsp16; __half* mela; float* zero; float* scale;
    void plan(Workspace& ws, const WgGrid& g) {
        const size_t R = g.grows;
        h32 = ws.get<float>(R * WG_C);
        acts = ws.get<__half>(R * WG_C);
        state = ws.get<float>(R * 8);
        dstate = ws.get<float>(R * 8);
        dout = ws.get<float>(R * 8);
        dy = ws.get<float>(R * 8);
        dskip = ws.get<__half>(R * WG_C);
        g16 = ws.get<__half>(R * WG_C);
        g32 = ws.get<float>(R * WG_C);
        dx = ws.get<__half>(R * 2 * WG_C);
        dsp32 = ws.get<float>(R * WG_SPECT);
        dsp16 = ws.get<__half>(R * WG_SPECT);
        mela = ws.get<__half>(R / 32 * 4 * WG_MEL_LD);
        zero = ws.get<float>(2 * WG_C);
        scale = ws.get<float>((static_cast<size_t>(g.nf) + 1) * 4);
    }
};

// The infer grid of B utterances of ceil(N / 256) frames each; the rows g >= N / 8 of an utterance are padding (rowinfo -1).
static int wt_grid(const FtWaveGlowTrainDesc* d, WgGrid* G) {
    if (!d) return ft_set_error("waveglow train: null descriptor");
    if (d->B < 1 || d->B > WG_MAX_B) return ft_set_error("waveglow train: batch must be 1..128");
    if (d->F < 1 || d->N < 8 || d->N % 8 || d->N > 256LL * d->F)
        return ft_set_error("waveglow train: N must be a positive multiple of 8 and at most 256 F");
    int frames[WG_MAX_B];
    const int fu = (d->N + 255) / 256;                 // frames whose upsampled samples reach sample N - 1
    for (int b = 0; b < d->B; ++b) frames[b] = fu;
    FtWaveGlowDesc gd = {d->n_mel, d->n_flows, d->n_group, d->n_early_every, d->n_early_size, d->n_layers, d->n_channels,
                         d->kernel_size, d->B, d->F, frames};
    return wg_grid(&gd, d->N / 8, G);
}

// One warp per grid row, for the flow boundary of the forward: finish flow `cur` (end conv from the skip sum, affine
// coupling audio_1 <- exp(log_s) audio_1 + b, log_s store), then start flow `next` (save its input, 1x1 conv over its live
// positions, start conv into h32 / the fp16 layer-0 input) or, after the last flow, store z.  The head launch loads audio.
struct WtTailParams {
    int R, Tn, N;
    const int* rowinfo;
    float* state;                   // [R, 8]: positions [0, o) hold early outputs, [o, 8) the c live channels
    const float* audio;             // head: [B, N]
    int cur, o, nh;
    const float* skip32; const float* end_w; const float* end_b;
    float* log_s;                   // [B, nh, Tn]
    int next, o_next, nh_next;
    const float* conv_w;            // [c, c] of flow `next`
    float* x_save;                  // [R, 8]
    const float* start_w; const float* start_b;
    float* h32; __half* h16;
    float* z;                       // [B, 8, Tn]
};

__global__ void __launch_bounds__(T_THREADS) wg_train_tail_kernel(const __grid_constant__ WtTailParams p) {
    __shared__ float s_end[8 * WG_C];
    __shared__ float s_start[WG_C * 4];
    __shared__ float s_misc[64 + 8 + WG_C];    // conv_w, end_b, start_b
    float* s_w = s_misc;
    float* s_endb = s_misc + 64;
    float* s_startb = s_misc + 72;
    const int cn = 8 - p.o_next;
    if (p.cur >= 0) {
        for (int i = threadIdx.x; i < 2 * p.nh * WG_C; i += T_THREADS) s_end[i] = p.end_w[i];
        if (threadIdx.x < 2 * p.nh) s_endb[threadIdx.x] = p.end_b[threadIdx.x];
    }
    if (p.next >= 0) {
        for (int i = threadIdx.x; i < WG_C * p.nh_next; i += T_THREADS) s_start[i] = p.start_w[i];
        for (int i = threadIdx.x; i < WG_C; i += T_THREADS) s_startb[i] = p.start_b[i];
        for (int i = threadIdx.x; i < cn * cn; i += T_THREADS) s_w[i] = p.conv_w[i];
    }
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    __shared__ float s_x[T_THREADS / 32][8], s_out[T_THREADS / 32][8];
    float* xs = s_x[warp];
    float* so = s_out[warp];
    const int r0 = (blockIdx.x * (T_THREADS / 32) + warp) * T_ROWS_PER_WARP;
    for (int r = r0; r < r0 + T_ROWS_PER_WARP && r < p.R; ++r) {
        const int info = __ldg(p.rowinfo + r);
        if (info < 0) continue;                                   // warp-uniform
        const int b = info / p.Tn, g = info - b * p.Tn;
        if (lane < 8) xs[lane] = p.audio ? __ldg(p.audio + static_cast<long long>(b) * p.N + 8 * g + lane)
                                         : p.state[static_cast<long long>(r) * 8 + lane];
        if (p.cur >= 0) {
            const float4* skp = reinterpret_cast<const float4*>(p.skip32 + static_cast<long long>(r) * WG_C + lane * 8);
            const float4 s0 = skp[0], s1 = skp[1];
            const float sk[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                if (j < 2 * p.nh) {
                    float a = 0.f;
#pragma unroll
                    for (int e = 0; e < 8; ++e) a = fmaf(s_end[j * WG_C + lane * 8 + e], sk[e], a);
#pragma unroll
                    for (int off = 16; off; off >>= 1) a += __shfl_xor_sync(0xffffffffu, a, off);
                    if (lane == j) so[j] = a + s_endb[j];
                }
            }
            __syncwarp();
            if (lane < p.nh) {                                    // audio_1 = positions [o + nh, 8)
                const int pos = p.o + p.nh + lane;
                const float ls = so[p.nh + lane];
                xs[pos] = expf(ls) * xs[pos] + so[lane];
                p.log_s[(static_cast<long long>(b) * p.nh + lane) * p.Tn + g] = ls;
            }
        }
        __syncwarp();
        if (p.next >= 0) {
            float v = 0.f;
            if (lane < 8) {
                v = xs[lane];
                p.x_save[static_cast<long long>(r) * 8 + lane] = v;
                if (lane >= p.o_next) {
                    v = 0.f;
                    for (int j = 0; j < cn; ++j) v = fmaf(s_w[(lane - p.o_next) * cn + j], xs[p.o_next + j], v);
                }
            }
            __syncwarp();
            if (lane < 8) xs[lane] = v;
            __syncwarp();
            float h[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const int ch = lane * 8 + e;
                float a = s_startb[ch];
#pragma unroll
                for (int i = 0; i < 4; ++i)
                    if (i < p.nh_next) a = fmaf(s_start[ch * p.nh_next + i], xs[p.o_next + i], a);
                h[e] = a;
            }
            const long long o = static_cast<long long>(r) * WG_C + lane * 8;
            float4* hp = reinterpret_cast<float4*>(p.h32 + o);
            hp[0] = make_float4(h[0], h[1], h[2], h[3]);
            hp[1] = make_float4(h[4], h[5], h[6], h[7]);
            const __half2 q0 = __halves2half2(sat_half(h[0]), sat_half(h[1])), q1 = __halves2half2(sat_half(h[2]), sat_half(h[3]));
            const __half2 q2 = __halves2half2(sat_half(h[4]), sat_half(h[5])), q3 = __halves2half2(sat_half(h[6]), sat_half(h[7]));
            uint4 pk;
            pk.x = *reinterpret_cast<const uint32_t*>(&q0); pk.y = *reinterpret_cast<const uint32_t*>(&q1);
            pk.z = *reinterpret_cast<const uint32_t*>(&q2); pk.w = *reinterpret_cast<const uint32_t*>(&q3);
            *reinterpret_cast<uint4*>(p.h16 + o) = pk;
            if (lane < 8) p.state[static_cast<long long>(r) * 8 + lane] = xs[lane];
        } else if (lane < 8) {
            p.z[(static_cast<long long>(b) * 8 + lane) * p.Tn + g] = xs[lane];
        }
        __syncwarp();
    }
}

static int launch_wt_tail(const WtTailParams& p, cudaStream_t st) {
    const int rows_per_block = (T_THREADS / 32) * T_ROWS_PER_WARP;
    TimeScope ts("wg_train_tail", p.R, p.cur, p.next, st);
    wg_train_tail_kernel<<<(p.R + rows_per_block - 1) / rows_per_block, T_THREADS, 0, st>>>(p);
    ft_count_launch(1);
    return ft_check_launch("wg_train_tail_kernel");
}

// Backward of one flow's boundary, in three grid-stride launches (one warp per row, per-block partial sums of the small
// weight gradients, then one atomicAdd per entry and block):
//   out   d_out = (d b, d log_s) from the incoming d audio_1 and d_log_s; d audio_1 before the coupling into dy; d end_w /
//         d end_b; max |d skip| for the flow's loss scale
//   skip  S from that maximum; d skip = end_w^T d_out * S (fp16, the WN backward's operand); G32 = 0
//   in    d a0 = start_w^T G / S + the pass-through gradient; d x = W^T dy into dstate; d start_w / d start_b / d W
struct WtBwdParams {
    int R, Tn;
    const int* rowinfo;
    int o, nh;
    const float* x_save; const float* conv_w; const float* skip32; const float* end_w; const float* end_b;
    const float* start_w;
    const float* dz;                // d_z [B, 8, Tn] (last flow only; NULL = zero): dstate starts from it
    const float* dlog_s;            // [B, nh, Tn] or NULL
    float* dstate; float* dout; float* dy;
    float* scale;                   // [S, 1/S, max |d skip| bits]
    __half* dskip16; float* g32;
    float* g_end_w; float* g_end_b; float* g_start_w; float* g_start_b; float* g_conv_w;
};

constexpr int WT_BLOCKS = 264;

__device__ __forceinline__ float wt_scale(const float* scale) {
    const float m = __uint_as_float(reinterpret_cast<const unsigned int*>(scale)[2]);
    if (!(m > 0.f) || !isfinite(m)) return 1.f;
    int e = static_cast<int>(floorf(log2f(WG_GRAD_TARGET / m)));
    e = e < -60 ? -60 : (e > 60 ? 60 : e);
    return exp2f(static_cast<float>(e));
}

__device__ __forceinline__ void wt_flush(float* red, int n, float* out) {
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += T_THREADS) atomicAdd(out + i, red[i]);
}

__global__ void __launch_bounds__(T_THREADS) wg_train_bwd_out_kernel(const __grid_constant__ WtBwdParams p) {
    __shared__ float s_end[8 * WG_C];
    __shared__ float s_red[8 * WG_C + 8];
    __shared__ float s_w[64], s_endb[8];
    __shared__ float s_x[T_THREADS / 32][8], s_d[T_THREADS / 32][8];
    const int c = 8 - p.o, nh = p.nh;
    for (int i = threadIdx.x; i < 2 * nh * WG_C; i += T_THREADS) s_end[i] = p.end_w[i];
    for (int i = threadIdx.x; i < 8 * WG_C + 8; i += T_THREADS) s_red[i] = 0.f;
    if (threadIdx.x < c * c) s_w[threadIdx.x] = p.conv_w[threadIdx.x];
    if (threadIdx.x < 2 * nh) s_endb[threadIdx.x] = p.end_b[threadIdx.x];
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float* xs = s_x[warp];
    float* ds = s_d[warp];
    float acc[8][8], accb[8], mx = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        accb[j] = 0.f;
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[j][e] = 0.f;
    }
    const int nw = gridDim.x * (T_THREADS / 32);
    for (int r = blockIdx.x * (T_THREADS / 32) + warp; r < p.R; r += nw) {
        const int info = __ldg(p.rowinfo + r);
        if (info < 0) continue;
        const int b = info / p.Tn, g = info - b * p.Tn;
        if (lane < 8) {
            xs[lane] = p.x_save[static_cast<long long>(r) * 8 + lane];
            ds[lane] = p.dz ? __ldg(p.dz + (static_cast<long long>(b) * 8 + lane) * p.Tn + g)
                            : p.dstate[static_cast<long long>(r) * 8 + lane];
        }
        __syncwarp();
        if (p.dz && lane < 8) p.dstate[static_cast<long long>(r) * 8 + lane] = ds[lane];
        const float4* skp = reinterpret_cast<const float4*>(p.skip32 + static_cast<long long>(r) * WG_C + lane * 8);
        const float4 s0 = skp[0], s1 = skp[1];
        const float sk[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
        float d[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            if (i < nh) {
                float a = 0.f;                                    // log_s_i, recomputed exactly as the forward did
#pragma unroll
                for (int e = 0; e < 8; ++e) a = fmaf(s_end[(nh + i) * WG_C + lane * 8 + e], sk[e], a);
#pragma unroll
                for (int off = 16; off; off >>= 1) a += __shfl_xor_sync(0xffffffffu, a, off);
                const float ls = a + s_endb[nh + i];
                float a1 = 0.f;                                   // audio_1 before the coupling: (W x)[nh + i]
                for (int j = 0; j < c; ++j) a1 = fmaf(s_w[(nh + i) * c + j], xs[p.o + j], a1);
                const float dap = ds[p.o + nh + i], ex = expf(ls);
                const float dls = p.dlog_s ? __ldg(p.dlog_s + (static_cast<long long>(b) * nh + i) * p.Tn + g) : 0.f;
                d[i] = dap;
                d[nh + i] = dap * ex * a1 + dls;
                if (lane == 0) p.dy[static_cast<long long>(r) * 8 + nh + i] = ex * dap;
            }
        }
        if (lane < 2 * nh) {
            float v = 0.f;
#pragma unroll
            for (int j = 0; j < 8; ++j) if (j == lane) v = d[j];
            p.dout[static_cast<long long>(r) * 8 + lane] = v;
        }
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            float dsk = 0.f;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                if (j < 2 * nh) {
                    acc[j][e] = fmaf(d[j], sk[e], acc[j][e]);
                    dsk = fmaf(s_end[j * WG_C + lane * 8 + e], d[j], dsk);
                }
            }
            mx = fmaxf(mx, fabsf(dsk));
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) if (j < 2 * nh) accb[j] += d[j];
        __syncwarp();
    }
#pragma unroll
    for (int off = 16; off; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
    if (lane == 0) atomicMax(reinterpret_cast<unsigned int*>(p.scale) + 2, __float_as_uint(mx));
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        if (j < 2 * nh) {
#pragma unroll
            for (int e = 0; e < 8; ++e) atomicAdd(&s_red[j * WG_C + lane * 8 + e], acc[j][e]);
            if (lane == 0) atomicAdd(&s_red[8 * WG_C + j], accb[j]);
        }
    }
    wt_flush(s_red, 2 * nh * WG_C, p.g_end_w);
    if (threadIdx.x < 2 * nh) atomicAdd(p.g_end_b + threadIdx.x, s_red[8 * WG_C + threadIdx.x]);
}

__global__ void __launch_bounds__(T_THREADS) wg_train_bwd_skip_kernel(const __grid_constant__ WtBwdParams p) {
    __shared__ float s_end[8 * WG_C];
    const int nh = p.nh;
    for (int i = threadIdx.x; i < 2 * nh * WG_C; i += T_THREADS) s_end[i] = p.end_w[i];
    __syncthreads();
    const float S = wt_scale(p.scale);
    if (blockIdx.x == 0 && threadIdx.x == 0) { p.scale[0] = S; p.scale[1] = 1.f / S; }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nw = gridDim.x * (T_THREADS / 32);
    for (int r = blockIdx.x * (T_THREADS / 32) + warp; r < p.R; r += nw) {
        if (__ldg(p.rowinfo + r) < 0) continue;
        float d[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) d[j] = j < 2 * nh ? p.dout[static_cast<long long>(r) * 8 + j] : 0.f;
        float v[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            float a = 0.f;
#pragma unroll
            for (int j = 0; j < 8; ++j) if (j < 2 * nh) a = fmaf(s_end[j * WG_C + lane * 8 + e], d[j], a);
            v[e] = a * S;
        }
        const long long o = static_cast<long long>(r) * WG_C + lane * 8;
        const __half2 q0 = __halves2half2(sat_half(v[0]), sat_half(v[1])), q1 = __halves2half2(sat_half(v[2]), sat_half(v[3]));
        const __half2 q2 = __halves2half2(sat_half(v[4]), sat_half(v[5])), q3 = __halves2half2(sat_half(v[6]), sat_half(v[7]));
        uint4 pk;
        pk.x = *reinterpret_cast<const uint32_t*>(&q0); pk.y = *reinterpret_cast<const uint32_t*>(&q1);
        pk.z = *reinterpret_cast<const uint32_t*>(&q2); pk.w = *reinterpret_cast<const uint32_t*>(&q3);
        *reinterpret_cast<uint4*>(p.dskip16 + o) = pk;
        float4* gp = reinterpret_cast<float4*>(p.g32 + o);
        gp[0] = make_float4(0.f, 0.f, 0.f, 0.f);
        gp[1] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
}

__global__ void __launch_bounds__(T_THREADS) wg_train_bwd_in_kernel(const __grid_constant__ WtBwdParams p) {
    __shared__ float s_start[WG_C * 4];
    __shared__ float s_red[WG_C * 4 + WG_C + 64];
    __shared__ float s_w[64];
    __shared__ float s_x[T_THREADS / 32][8], s_y[T_THREADS / 32][8], s_dy[T_THREADS / 32][8];
    const int c = 8 - p.o, nh = p.nh;
    for (int i = threadIdx.x; i < WG_C * nh; i += T_THREADS) s_start[i] = p.start_w[i];
    for (int i = threadIdx.x; i < WG_C * 5 + 64; i += T_THREADS) s_red[i] = 0.f;
    if (threadIdx.x < c * c) s_w[threadIdx.x] = p.conv_w[threadIdx.x];
    __syncthreads();
    const float iS = p.scale[1];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float* xs = s_x[warp];
    float* ys = s_y[warp];
    float* dys = s_dy[warp];
    float acc[8][4], accb[8], accw[2] = {0.f, 0.f};
#pragma unroll
    for (int e = 0; e < 8; ++e) {
        accb[e] = 0.f;
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[e][i] = 0.f;
    }
    const int nw = gridDim.x * (T_THREADS / 32);
    for (int r = blockIdx.x * (T_THREADS / 32) + warp; r < p.R; r += nw) {
        if (__ldg(p.rowinfo + r) < 0) continue;
        const long long r8 = static_cast<long long>(r) * 8;
        if (lane < 8) xs[lane] = p.x_save[r8 + lane];
        __syncwarp();
        if (lane < c) {
            float a = 0.f;
            for (int j = 0; j < c; ++j) a = fmaf(s_w[lane * c + j], xs[p.o + j], a);
            ys[lane] = a;                                         // y = W x over the live positions (relative index)
        }
        const float4* gp = reinterpret_cast<const float4*>(p.g32 + static_cast<long long>(r) * WG_C + lane * 8);
        const float4 g0 = gp[0], g1 = gp[1];
        float gv[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
#pragma unroll
        for (int e = 0; e < 8; ++e) gv[e] *= iS;
        __syncwarp();
        float da0[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            da0[i] = 0.f;
            if (i < nh) {
                float a = 0.f;
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                    a = fmaf(s_start[(lane * 8 + e) * nh + i], gv[e], a);
                    acc[e][i] = fmaf(gv[e], ys[i], acc[e][i]);
                }
#pragma unroll
                for (int off = 16; off; off >>= 1) a += __shfl_xor_sync(0xffffffffu, a, off);
                da0[i] = a;
            }
        }
#pragma unroll
        for (int e = 0; e < 8; ++e) accb[e] += gv[e];
        if (lane < c) {
            float v;
            if (lane < nh) {
                v = p.dstate[r8 + p.o + lane];                     // audio_0 passes through the coupling unchanged
#pragma unroll
                for (int i = 0; i < 4; ++i) if (i == lane) v += da0[i];
            } else {
                v = p.dy[r8 + lane];
            }
            dys[lane] = v;
        }
        __syncwarp();
#pragma unroll
        for (int q = 0; q < 2; ++q) {                             // d W[i][j] += dy_i x_j, entry i * c + j = lane + 32 q
            const int ij = lane + 32 * q;
            if (ij < c * c) accw[q] = fmaf(dys[ij / c], xs[p.o + ij % c], accw[q]);
        }
        if (lane < c) {
            float a = 0.f;
            for (int i = 0; i < c; ++i) a = fmaf(s_w[i * c + lane], dys[i], a);
            p.dstate[r8 + p.o + lane] = a;
        }
        __syncwarp();
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) {
#pragma unroll
        for (int i = 0; i < 4; ++i) if (i < nh) atomicAdd(&s_red[(lane * 8 + e) * nh + i], acc[e][i]);
        atomicAdd(&s_red[4 * WG_C + lane * 8 + e], accb[e]);
    }
#pragma unroll
    for (int q = 0; q < 2; ++q) if (lane + 32 * q < c * c) atomicAdd(&s_red[5 * WG_C + lane + 32 * q], accw[q]);
    wt_flush(s_red, WG_C * nh, p.g_start_w);
    for (int i = threadIdx.x; i < WG_C; i += T_THREADS) atomicAdd(p.g_start_b + i, s_red[4 * WG_C + i]);
    if (threadIdx.x < c * c) atomicAdd(p.g_conv_w + threadIdx.x, s_red[5 * WG_C + threadIdx.x]);
}

// d spect (fp32, accumulated over every flow and layer) -> fp16 * S for the upsample's weight gradient
__global__ void wg_scale_cast_kernel(const float* __restrict__ src, long long n, const float* __restrict__ scale2,
                                     __half* __restrict__ dst) {
    const float S = scale2[0];
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
         i += static_cast<long long>(gridDim.x) * blockDim.x)
        dst[i] = sat_half(src[i] * S);
}

// The upsample GEMM's A operand, one row per 32 grid rows (one mel frame): mela[fr] = mel frames f, f-1, f-2, f-3 of the
// utterance whose frame f starts at grid row 32 fr, zero rows between utterances; d up_w = d spect^T mela over frames.
__global__ void wg_mela_kernel(const WgBatch* __restrict__ plan, const int* __restrict__ rowinfo, const __half* __restrict__ mel16,
                               int n_fr, __half* __restrict__ mela) {
    const WgBatch& bt = *plan;
    const long long n = static_cast<long long>(n_fr) * 4 * WG_MEL_LD;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int fr = static_cast<int>(i / (4 * WG_MEL_LD)), col = static_cast<int>(i % (4 * WG_MEL_LD));
        const int info = __ldg(rowinfo + 32 * fr);
        __half v = __float2half_rn(0.f);
        if (info >= 0) {
            const int b = info / bt.Tg_max, f = (info - b * bt.Tg_max) / 32, j = col / WG_MEL_LD;
            v = mel16[static_cast<long long>(bt.mbase[b] + 3 + f - j) * WG_MEL_LD + col % WG_MEL_LD];
        }
        mela[i] = v;
    }
}

static int wt_launch(const void* fn, const WtBwdParams& p, cudaStream_t st, const char* name) {
    TimeScope ts(name, p.R, p.nh, 0, st);
    void* args[] = {const_cast<WtBwdParams*>(&p)};
    if (cudaLaunchKernel(fn, dim3(WT_BLOCKS), dim3(T_THREADS), args, 0, st) != cudaSuccess) return ft_set_error(name);
    ft_count_launch(1);
    return ft_check_launch(name);
}

// frames_dev: null for d->frames (host counts), else the device counts (d->frames must then be null).  Every kernel after
// the plan reads the layout and the live row counts from the planned WgBatch; grids and GEMM M come from G, the bound.
static int wg_infer(const FtWaveGlowDesc* d, const FtWaveGlowWeights* w, const float* mel, const float* noise, float sigma,
                    const int* frames_dev, float* audio, void* scratch, void* stream) {
    WgGrid G;
    if (wg_infer_grid(d, &G)) return -1;
    if (!w || !mel || !noise || !audio || !scratch) return ft_set_error("waveglow: null pointer argument");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const WgInferScratch s = wg_carve<WgInferScratch>(scratch, G);
    const int* live = &s.in.batch->grows;
    const int R = G.grows, nf = G.nf;

    // zero hidden-state guard rows (the dilated taps read them) and the audio padding after each utterance
    FT_CU(cudaMemsetAsync(s.h16, 0, static_cast<size_t>(R) * WG_C * 2, st), "waveglow");
    FT_CU(cudaMemsetAsync(audio, 0, sizeof(float) * static_cast<size_t>(G.B) * G.Tg_max * 8, st), "waveglow");
    if (launch_wg_plan_prep(G, s.in, frames_dev, mel, st)) return -1;
    if (wg_upsample(G, s.in, w, &s.in.batch->mrows, st)) return -1;
    // head: initial noise on the last flow's live positions and that flow's start conv
    {
        const int c = G.c[nf - 1];
        WgTailParams t = {};
        t.R = R; t.live_rows = live; t.rowinfo = s.in.rowinfo; t.state = s.state;
        t.cur = 0; t.o = 8 - c; t.nh = c / 2;
        t.inj_lo = 8 - c; t.inj_hi = 8; t.noise = noise; t.Tg_max = G.Tg_max; t.sigma = sigma;
        t.next = 1; t.o_next = 8 - c; t.nh_next = c / 2; t.start_w = w->start_w[nf - 1]; t.start_b = w->start_b[nf - 1];
        t.h32 = s.h32; t.h16 = s.h16;
        if (launch_wg_tail(t, st)) return -1;
    }
    for (int k = nf - 1; k >= 0; --k) {
        if (wg_flow_wn(G, s.in, w, k, s.h16, 0, nullptr, s.acts, s.h32, s.skip, live, st)) return -1;
        const int c = G.c[k];
        WgTailParams t = {};
        t.R = R; t.live_rows = live; t.rowinfo = s.in.rowinfo; t.state = s.state;
        t.cur = 1; t.o = 8 - c; t.nh = c / 2;
        t.skip32 = s.skip; t.end_w = w->end_w[k]; t.end_b = w->end_b[k]; t.inv_w = w->inv_w[k];
        const bool inject = k > 0 && k % d->n_early_every == 0 && d->n_early_size > 0;
        t.inj_lo = inject ? 8 - c - d->n_early_size : 0; t.inj_hi = inject ? 8 - c : 0;
        t.noise = noise; t.Tg_max = G.Tg_max; t.sigma = sigma;
        if (k > 0) {
            const int cn = G.c[k - 1];
            t.next = 1; t.o_next = 8 - cn; t.nh_next = cn / 2; t.start_w = w->start_w[k - 1]; t.start_b = w->start_b[k - 1];
            t.h32 = s.h32; t.h16 = s.h16;
        } else {
            t.next = 0; t.audio = audio;
        }
        if (launch_wg_tail(t, st)) return -1;
    }
    return 0;
}

}  // namespace ft

extern "C" {

size_t ft_waveglow_scratch_bytes(const FtWaveGlowDesc* d) {
    ft::WgGrid G;
    return ft::wg_infer_grid(d, &G) ? 0 : ft::wg_bytes<ft::WgInferScratch>(G);
}

int ft_waveglow_infer(const FtWaveGlowDesc* d, const FtWaveGlowWeights* w, const float* mel, const float* noise, float sigma,
                      float* audio, void* scratch, void* stream) {
    if (d && !d->frames) return ft::ft_set_error("waveglow: frames (host array) required; ft_waveglow_infer_dev takes device frames");
    return ft::wg_infer(d, w, mel, noise, sigma, nullptr, audio, scratch, stream);
}

int ft_waveglow_infer_dev(const FtWaveGlowDesc* d, const FtWaveGlowWeights* w, const float* mel, const float* noise, float sigma,
                          const int* frames_dev, float* audio, void* scratch, void* stream) {
    if (d && d->frames) return ft::ft_set_error("waveglow: ft_waveglow_infer_dev takes desc->frames == NULL");
    if (!frames_dev) return ft::ft_set_error("waveglow: null frames_dev");
    return ft::wg_infer(d, w, mel, noise, sigma, frames_dev, audio, scratch, stream);
}

size_t ft_waveglow_train_saved_bytes(const FtWaveGlowTrainDesc* d) {
    ft::WgGrid G;
    return ft::wt_grid(d, &G) ? 0 : ft::wg_bytes<ft::WtSaved>(G);
}

size_t ft_waveglow_train_scratch_bytes(const FtWaveGlowTrainDesc* d) {
    ft::WgGrid G;
    return ft::wt_grid(d, &G) ? 0 : ft::wg_bytes<ft::WtScratch>(G);
}

int ft_waveglow_train_fwd(const FtWaveGlowTrainDesc* d, const FtWaveGlowTrainWeights* w, const float* mel, const float* audio,
                          float* z, float* const* log_s, void* saved, void* scratch, void* stream) {
    using namespace ft;
    WgGrid G;
    if (wt_grid(d, &G)) return -1;
    if (!w || !mel || !audio || !z || !log_s || !saved || !scratch) return ft_set_error("waveglow train: null pointer argument");
    for (int k = 0; k < G.nf; ++k) if (!log_s[k]) return ft_set_error("waveglow train: null log_s pointer");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const WtSaved s = wg_carve<WtSaved>(saved, G);
    const WtScratch c = wg_carve<WtScratch>(scratch, G);
    const long long R = G.grows, flow_h16 = G.nl * R * WG_C;   // one flow's saved layer inputs

    // guard and padding rows of every layer input and of the upsampled spectrogram are zero: the dilated taps and the
    // row-reduced weight gradients read them
    FT_CU(cudaMemsetAsync(s.h16, 0, static_cast<size_t>(G.nf) * flow_h16 * 2, st), "waveglow train");
    FT_CU(cudaMemsetAsync(s.in.spect, 0, static_cast<size_t>(R) * WG_SPECT * 2, st), "waveglow train");
    if (launch_wg_plan_prep(G, s.in, nullptr, mel, st)) return -1;
    if (wg_upsample(G, s.in, w, nullptr, st)) return -1;
    WtTailParams t = {};
    t.R = static_cast<int>(R); t.Tn = G.Tg_max; t.N = d->N; t.rowinfo = s.in.rowinfo; t.state = c.state; t.h32 = c.h32;
    t.audio = audio; t.cur = -1;
    for (int k = 0; k <= G.nf; ++k) {
        if (k < G.nf) {
            t.next = k; t.o_next = 8 - G.c[k]; t.nh_next = G.c[k] / 2;
            t.conv_w = w->conv_w[k]; t.x_save = s.x + k * R * 8;
            t.start_w = w->start_w[k]; t.start_b = w->start_b[k]; t.h16 = s.h16 + k * flow_h16;
        } else {
            t.next = -1; t.z = z;
        }
        if (launch_wt_tail(t, st)) return -1;
        if (k == G.nf) break;
        float* skip_k = s.skip + k * R * WG_C;
        if (wg_flow_wn(G, s.in, w, k, s.h16 + k * flow_h16, R * WG_C, s.pre + 2 * k * flow_h16, c.acts, c.h32, skip_k, nullptr, st))
            return -1;
        t.audio = nullptr;
        t.cur = k; t.o = 8 - G.c[k]; t.nh = G.c[k] / 2;
        t.skip32 = skip_k; t.end_w = w->end_w[k]; t.end_b = w->end_b[k]; t.log_s = log_s[k];
    }
    return 0;
}

int ft_waveglow_train_bwd(const FtWaveGlowTrainDesc* d, const FtWaveGlowTrainWeights* w, const float* d_z,
                          const float* const* d_log_s, const void* saved, const FtWaveGlowTrainGrads* gr, void* scratch,
                          void* stream) {
    using namespace ft;
    WgGrid G;
    if (wt_grid(d, &G)) return -1;
    if (!w || !saved || !gr || !scratch) return ft_set_error("waveglow train: null pointer argument");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const WtSaved s = wg_carve<WtSaved>(saved, G);
    const WtScratch c = wg_carve<WtScratch>(scratch, G);
    const long long R = G.grows, C = WG_C;
    const long long W0 = WG_GUARD, RW = R - 2 * WG_GUARD;   // row window of the shifted-tap weight gradients

    auto z0 = [&](void* p, size_t n) { FT_CU(cudaMemsetAsync(p, 0, n, st), "waveglow train"); return 0; };
    // rows no kernel writes (guards, padding) stay zero in every fp16 gradient operand: the shifted taps and the
    // row-reduced weight gradients and column sums read them
    if (z0(c.acts, R * C * 2) || z0(c.dskip, R * C * 2) || z0(c.g16, R * C * 2) || z0(c.dx, R * 2 * C * 2) ||
        z0(c.dsp32, R * WG_SPECT * 4) || z0(c.zero, 2 * C * 4) || z0(c.scale, (G.nf + 1) * 16))
        return -1;
    for (int k = 0; k < G.nf; ++k) {
        const int ck = G.c[k], nh = ck / 2;
        if (z0(gr->end_w[k], 2 * nh * C * 4) || z0(gr->end_b[k], 2 * nh * 4) || z0(gr->start_w[k], C * nh * 4) ||
            z0(gr->start_b[k], C * 4) || z0(gr->conv_w[k], ck * ck * 4))
            return -1;
    }
    for (int k = G.nf - 1; k >= 0; --k) {
        const int ck = G.c[k], nh = ck / 2;
        WtBwdParams b = {};
        b.R = static_cast<int>(R); b.Tn = G.Tg_max; b.rowinfo = s.in.rowinfo; b.o = 8 - ck; b.nh = nh;
        b.x_save = s.x + k * R * 8; b.conv_w = w->conv_w[k];
        b.skip32 = s.skip + k * R * C; b.end_w = w->end_w[k]; b.end_b = w->end_b[k]; b.start_w = w->start_w[k];
        b.dz = k == G.nf - 1 ? d_z : nullptr;
        b.dlog_s = d_log_s ? d_log_s[k] : nullptr;
        b.dstate = c.dstate; b.dout = c.dout; b.dy = c.dy; b.scale = c.scale + 4 * k; b.dskip16 = c.dskip; b.g32 = c.g32;
        b.g_end_w = gr->end_w[k]; b.g_end_b = gr->end_b[k]; b.g_start_w = gr->start_w[k]; b.g_start_b = gr->start_b[k];
        b.g_conv_w = gr->conv_w[k];
        if (k == G.nf - 1 && !d_z && z0(c.dstate, R * 8 * 4)) return -1;
        if (wt_launch(reinterpret_cast<const void*>(wg_train_bwd_out_kernel), b, st, "wg_train_bwd_out")) return -1;
        if (wt_launch(reinterpret_cast<const void*>(wg_train_bwd_skip_kernel), b, st, "wg_train_bwd_skip")) return -1;
        const float* iS = c.scale + 4 * k + 1;
        for (int i = G.nl - 1; i >= 0; --i) {
            const int dil = 1 << i;
            const bool last = i == G.nl - 1;
            const long long layer = static_cast<long long>(k) * G.nl + i;
            const __half* hin = s.h16 + layer * R * C;
            // d acts = rs_w^T [G; d skip] -> d pre-activations (dx) and the recomputed acts
            WgGemmParams p = {};
            p.M = static_cast<int>(R); p.N = WG_C; p.nseg = last ? 1 : 2; p.K = p.nseg * WG_C;
            if (last) {
                p.seg[0] = WgSeg{c.dskip, R, WG_C, 0, WG_C};
            } else {
                p.seg[0] = WgSeg{c.g16, R, WG_C, 0, WG_C};
                p.seg[1] = WgSeg{c.dskip, R, WG_C, 0, WG_C};
            }
            p.W = static_cast<const __half*>(w->rs_wT[k][i]); p.rowmap = s.in.rowinfo; p.mode = WG_EPI_GATE_BWD;
            p.out16 = c.dx; p.ld16 = 2 * WG_C; p.h16 = c.acts; p.pre16 = s.pre + layer * R * 2 * C;
            if (launch_wg_gemm(p, st)) return -1;
            // res_skip_layer: rows [0, C) meet G (the residual), the rest d skip
            float* grs = gr->rs_w[k][i];
            if (!last) {
                if (gemm_wgrad(st, WG_C, WG_C, R, c.g16, C, c.acts, C, grs, WG_C, iS)) return -1;
                if (launch_colsum(c.g16, 0, C, R, WG_C, gr->rs_b[k][i], iS, st)) return -1;
            }
            const long long so = last ? 0 : C;
            if (gemm_wgrad(st, WG_C, WG_C, R, c.dskip, C, c.acts, C, grs + so * C, WG_C, iS)) return -1;
            if (launch_colsum(c.dskip, 0, C, R, WG_C, gr->rs_b[k][i] + so, iS, st)) return -1;
            // in_layer taps (h shifted by -d, 0, +d) and the cond_layer slice
            for (int tap = 0; tap < 3; ++tap)
                if (gemm_wgrad(st, 2 * WG_C, WG_C, RW, c.dx + W0 * 2 * C, 2 * C, hin + (W0 + (tap - 1) * dil) * C, C,
                               gr->in_w[k][i][tap], WG_C, iS))
                    return -1;
            if (gemm_wgrad(st, 2 * WG_C, WG_SPECT, R, c.dx, 2 * C, s.in.spect, WG_SPECT, gr->in_w[k][i][3], WG_SPECT, iS)) return -1;
            if (launch_colsum(c.dx, 0, 2 * C, R, 2 * WG_C, gr->in_b[k][i], iS, st)) return -1;
            // d spect += dx cond_w (fp32, unscaled on the way out)
            if (gemm_dgrad(st, R, WG_SPECT, 2 * WG_C, c.dx, 2 * C, static_cast<const __half*>(w->in_w[k][i]) + 3 * WG_C,
                           3 * WG_C + WG_SPECT, c.dsp32, WG_SPECT, nullptr, 0, 1, iS))
                return -1;
            // G += in_w^T dx over the transposed taps: dx shifted by +d, 0, -d (the guard rows keep padding out)
            WgGemmParams q = {};
            q.M = static_cast<int>(R); q.N = WG_C; q.K = 6 * WG_C; q.nseg = 3;
            for (int tap = 0; tap < 3; ++tap) q.seg[tap] = WgSeg{c.dx, R, 2 * WG_C, (1 - tap) * dil, 2 * WG_C};
            q.W = static_cast<const __half*>(w->in_wT[k][i]); q.bias = c.zero; q.rowmap = s.in.rowinfo; q.mode = WG_EPI_RES;
            q.h32 = c.g32; q.h16 = c.g16; q.res_cols = WG_C;
            if (launch_wg_gemm(q, st)) return -1;
        }
        if (wt_launch(reinterpret_cast<const void*>(wg_train_bwd_in_kernel), b, st, "wg_train_bwd_in")) return -1;
    }
    // upsample: d up_w = d spect^T mela over mel frames (32 grid rows each), d up_b = column sums of d spect
    float* sup = c.scale + 4 * G.nf;
    const long long nfr = R / 32, nsp = R * WG_SPECT;
    if (launch_grad_scale(c.dsp32, nsp, nullptr, 0, nullptr, 0, WG_GRAD_TARGET, sup, st)) return -1;
    {
        TimeScope ts("wg_train_up_prep", nfr, 0, 0, st);
        wg_scale_cast_kernel<<<static_cast<int>(std::min<long long>((nsp + 255) / 256, 4096)), 256, 0, st>>>(c.dsp32, nsp, sup, c.dsp16);
        wg_mela_kernel<<<static_cast<int>(std::min<long long>((nfr * 384 + 255) / 256, 4096)), 256, 0, st>>>(
            s.in.batch, s.in.rowinfo, s.in.mel16, static_cast<int>(nfr), c.mela);
        ft_count_launch(2);
        if (ft_check_launch("wg_train_up_prep")) return -1;
    }
    if (gemm_wgrad(st, WG_UP_N, 4 * WG_MEL_LD, nfr, c.dsp16, WG_UP_N, c.mela, 4 * WG_MEL_LD, gr->up_w, 4 * WG_MEL_LD, sup + 1)) return -1;
    if (launch_colsum(c.dsp32, 2, WG_UP_N, nfr, WG_UP_N, gr->up_b, nullptr, st)) return -1;
    return 0;
}

}  // extern "C"
