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

enum { WG_EPI_UP = 0, WG_EPI_GATE = 1, WG_EPI_RES = 2 };

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
    int mode;
    __half* out16; long long ld16;            // UP, GATE
    float* h32; __half* h16; float* skip32;   // RES ([rows, C] each)
    int res_cols;                             // RES: columns [0, res_cols) update the hidden state, the rest the skip sum
    int skip_store;                           // RES: 1 = skip32 = x (first layer), 0 = skip32 += x
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
__device__ __forceinline__ void mma16816(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ __half sat_half(float x) { return __float2half_rn(fminf(fmaxf(x, -65504.f), 65504.f)); }

__device__ __forceinline__ void wg_epi_pair(const WgGemmParams& p, int m, int n, float v0, float v1) {
    if (m >= p.M) return;
    const int info = __ldg(p.rowmap + m);
    if (info < 0) return;                                     // guard / padding rows are never written
    const int row = p.mode == WG_EPI_UP ? info : m;           // UP: a frame row lands on its first group row
    const float2 b = __ldg(reinterpret_cast<const float2*>(p.bias + n));
    const float x0 = v0 + b.x, x1 = v1 + b.y;
    if (p.mode == WG_EPI_GATE) {
        p.out16[static_cast<long long>(row) * p.ld16 + (n >> 1)] = sat_half(tanh_f(x0) * sigmoid_f(x1));
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
            const bool ok = (m0 + r < p.M) && ar >= 0 && ar < rows;
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
                for (int j = 0; j < 4; ++j) mma16816(acc[i][j], af[i], bf[j][0], bf[j][1]);
        }
    }
    cp_async_wait<0>();

#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int m = m0 + wm * 64 + i * 16 + (lane >> 2);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int n = n0 + wn * 32 + j * 8 + 2 * (lane & 3);
            wg_epi_pair(p, m, n, acc[i][j][0], acc[i][j][1]);
            wg_epi_pair(p, m + 8, n, acc[i][j][2], acc[i][j][3]);
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
    TimeScope ts(p.mode == WG_EPI_UP ? "wg_upsample" : (p.mode == WG_EPI_GATE ? "wg_in_layer" : "wg_res_skip"), p.M, p.N, p.K, st);
    wg_gemm_kernel<<<grid, G_THREADS, G_SMEM, st>>>(p);
    ft_count_launch(1);
    return ft_check_launch("wg_gemm_kernel");
}

// ------------------------------------------------------------------------------------------------ prep
struct WgBatch {
    int B, Tg_max;
    int frames[WG_MAX_B];
    int mbase[WG_MAX_B + 1];     // first frame-grid row of utterance b (its 3 zero rows come first); mbase[B] = rows
    int gbase[WG_MAX_B + 1];     // first group-grid row of utterance b; gbase[B] = end of the last utterance
};

__device__ __forceinline__ int find_utt(const int* base, int B, int r) {   // largest b with base[b] <= r
    int lo = 0, hi = B - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (base[mid] <= r) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// mel [B, 80, F_max] fp32 -> mel16 [mrows, 96]; up_rowmap [mrows]; rowinfo [grows] = b * Tg_max + g, or -1 for guard rows.
__global__ void wg_prep_kernel(const __grid_constant__ WgBatch bt, const float* __restrict__ mel, int F_max, __half* __restrict__ mel16,
                               int* __restrict__ up_rowmap, int* __restrict__ rowinfo, int grows) {
    const int mrows = bt.mbase[bt.B];
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
                if (g < 32 * bt.frames[b]) info = b * bt.Tg_max + g;
            }
            rowinfo[r] = info;
        }
    }
}

// ------------------------------------------------------------------------------------------------ flow tail
constexpr int T_THREADS = 256, T_ROWS_PER_WARP = 8;

struct WgTailParams {
    int R;                          // grid rows
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
    for (int r = r0; r < r0 + T_ROWS_PER_WARP && r < p.R; ++r) {
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
struct WgLayout {
    int B, Tg_max, mrows, grows;
    WgBatch bt;
    size_t off_mel16, off_uprow, off_rowinfo, off_spect, off_h32, off_h16, off_acts, off_skip, off_state, total;
};

static int wg_layout(const FtWaveGlowDesc* d, WgLayout* L) {
    if (!d) return ft_set_error("waveglow: null descriptor");
    if (d->n_mel != WG_MEL || d->n_group != 8 || d->n_channels != WG_C || d->kernel_size != 3)
        return ft_set_error("waveglow: only n_mel 80, n_group 8, n_channels 256, kernel_size 3 are built");
    if (d->n_flows < 1 || d->n_flows > FT_WG_MAX_FLOWS || d->n_layers < 1 || d->n_layers > FT_WG_MAX_LAYERS)
        return ft_set_error("waveglow: n_flows must be 1..16 and n_layers 1..8");
    if (d->n_early_every < 1 || d->n_early_size < 0 || d->n_early_size % 2)
        return ft_set_error("waveglow: n_early_every >= 1 and an even n_early_size >= 0 required");
    const int n_early = (d->n_flows - 1) / d->n_early_every;
    if (8 - n_early * d->n_early_size < 2) return ft_set_error("waveglow: early outputs leave fewer than 2 channels");
    if (d->B < 1 || d->B > WG_MAX_B) return ft_set_error("waveglow: batch must be 1..128");
    if (!d->frames) return ft_set_error("waveglow: frames (host array) required");
    L->B = d->B;
    L->Tg_max = 32 * d->F_max;
    L->bt.B = d->B;
    L->bt.Tg_max = L->Tg_max;
    long long m = 0, g = WG_GUARD;
    for (int b = 0; b < d->B; ++b) {
        const int f = d->frames[b];
        if (f < 1 || f > d->F_max) return ft_set_error("waveglow: frames[b] must be in 1..F_max");
        L->bt.frames[b] = f;
        L->bt.mbase[b] = static_cast<int>(m);
        L->bt.gbase[b] = static_cast<int>(g);
        m += f + 3;
        g += 32LL * f + WG_GUARD;
        if (g > (1LL << 30)) return ft_set_error("waveglow: batch too long");
    }
    L->bt.mbase[d->B] = static_cast<int>(m);
    L->bt.gbase[d->B] = static_cast<int>(g - WG_GUARD);
    L->mrows = static_cast<int>(m);
    L->grows = static_cast<int>(g);
    size_t off = 0;
    auto take = [&](size_t bytes) { const size_t o = off; off += (bytes + 255) & ~size_t(255); return o; };
    const size_t R = static_cast<size_t>(L->grows);
    L->off_mel16 = take(static_cast<size_t>(L->mrows) * WG_MEL_LD * 2);
    L->off_uprow = take(static_cast<size_t>(L->mrows) * 4);
    L->off_rowinfo = take(R * 4);
    L->off_spect = take(R * WG_SPECT * 2);
    L->off_h32 = take(R * WG_C * 4);
    L->off_h16 = take(R * WG_C * 2);
    L->off_acts = take(R * WG_C * 2);
    L->off_skip = take(R * WG_C * 4);
    L->off_state = take(R * 8 * 4);
    L->total = off;
    return 0;
}

// channel bookkeeping of the inverse pass: flow k has c_k live channels, n_half = c_k / 2
static int wg_channels(const FtWaveGlowDesc* d, int k) {
    int c = 8;
    for (int j = 1; j <= k; ++j)
        if (j % d->n_early_every == 0) c -= d->n_early_size;
    return c;
}

}  // namespace ft

extern "C" {

size_t ft_waveglow_scratch_bytes(const FtWaveGlowDesc* d) {
    ft::WgLayout L;
    if (ft::wg_layout(d, &L)) return 0;
    return L.total;
}

int ft_waveglow_infer(const FtWaveGlowDesc* d, const FtWaveGlowWeights* w, const float* mel, const float* noise, float sigma,
                      float* audio, void* scratch, void* stream) {
    using namespace ft;
    WgLayout L;
    if (wg_layout(d, &L)) return -1;
    if (!w || !mel || !noise || !audio || !scratch) return ft_set_error("waveglow: null pointer argument");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    uint8_t* base = static_cast<uint8_t*>(scratch);
    __half* mel16 = reinterpret_cast<__half*>(base + L.off_mel16);
    int* uprow = reinterpret_cast<int*>(base + L.off_uprow);
    int* rowinfo = reinterpret_cast<int*>(base + L.off_rowinfo);
    __half* spect = reinterpret_cast<__half*>(base + L.off_spect);
    float* h32 = reinterpret_cast<float*>(base + L.off_h32);
    __half* h16 = reinterpret_cast<__half*>(base + L.off_h16);
    __half* acts = reinterpret_cast<__half*>(base + L.off_acts);
    float* skip = reinterpret_cast<float*>(base + L.off_skip);
    float* state = reinterpret_cast<float*>(base + L.off_state);
    const long long R = L.grows;

    // zero hidden-state guard rows (the dilated taps read them) and the audio padding after each utterance
    if (cudaMemsetAsync(h16, 0, static_cast<size_t>(R) * WG_C * 2, st) != cudaSuccess ||
        cudaMemsetAsync(audio, 0, sizeof(float) * static_cast<size_t>(L.B) * L.Tg_max * 8, st) != cudaSuccess)
        return ft_set_error("waveglow: memset failed");
    {
        const long long work = static_cast<long long>(L.mrows) * (WG_MEL_LD + 1) + R;
        const int grid = static_cast<int>(std::min<long long>((work + 255) / 256, 4096));
        TimeScope ts("wg_prep", L.mrows, R, 0, st);
        wg_prep_kernel<<<grid, 256, 0, st>>>(L.bt, mel, d->F_max, mel16, uprow, rowinfo, static_cast<int>(R));
        ft_count_launch(1);
        if (ft_check_launch("wg_prep_kernel")) return -1;
    }
    {   // upsample: frame row f = frames f-3..f (A segments shifted 0..-3) -> 32 group rows of 640 channels
        WgGemmParams p = {};
        p.M = L.mrows; p.N = WG_UP_N; p.K = 4 * WG_MEL_LD; p.nseg = 4;
        for (int j = 0; j < 4; ++j) p.seg[j] = WgSeg{mel16, L.mrows, WG_MEL_LD, -j, WG_MEL_LD};
        p.W = static_cast<const __half*>(w->up_w); p.bias = w->up_b; p.rowmap = uprow; p.mode = WG_EPI_UP;
        p.out16 = spect; p.ld16 = WG_SPECT;
        if (launch_wg_gemm(p, st)) return -1;
    }
    const int nf = d->n_flows, nl = d->n_layers;
    // head: initial noise on the last flow's live positions and that flow's start conv
    {
        const int c = wg_channels(d, nf - 1);
        WgTailParams t = {};
        t.R = static_cast<int>(R); t.rowinfo = rowinfo; t.state = state;
        t.cur = 0; t.o = 8 - c; t.nh = c / 2;
        t.inj_lo = 8 - c; t.inj_hi = 8; t.noise = noise; t.Tg_max = L.Tg_max; t.sigma = sigma;
        t.next = 1; t.o_next = 8 - c; t.nh_next = c / 2; t.start_w = w->start_w[nf - 1]; t.start_b = w->start_b[nf - 1];
        t.h32 = h32; t.h16 = h16;
        if (launch_wg_tail(t, st)) return -1;
    }
    for (int k = nf - 1; k >= 0; --k) {
        for (int i = 0; i < nl; ++i) {
            const int dil = 1 << i;
            WgGemmParams p = {};
            p.M = static_cast<int>(R); p.N = 2 * WG_C; p.K = 3 * WG_C + WG_SPECT; p.nseg = 4;
            p.seg[0] = WgSeg{h16, R, WG_C, -dil, WG_C};
            p.seg[1] = WgSeg{h16, R, WG_C, 0, WG_C};
            p.seg[2] = WgSeg{h16, R, WG_C, dil, WG_C};
            p.seg[3] = WgSeg{spect, R, WG_SPECT, 0, WG_SPECT};
            p.W = static_cast<const __half*>(w->in_w[k][i]); p.bias = w->in_b[k][i]; p.rowmap = rowinfo; p.mode = WG_EPI_GATE;
            p.out16 = acts; p.ld16 = WG_C;
            if (launch_wg_gemm(p, st)) return -1;
            WgGemmParams q = {};
            const bool last = i == nl - 1;
            q.M = static_cast<int>(R); q.N = last ? WG_C : 2 * WG_C; q.K = WG_C; q.nseg = 1;
            q.seg[0] = WgSeg{acts, R, WG_C, 0, WG_C};
            q.W = static_cast<const __half*>(w->rs_w[k][i]); q.bias = w->rs_b[k][i]; q.rowmap = rowinfo; q.mode = WG_EPI_RES;
            q.h32 = h32; q.h16 = h16; q.skip32 = skip; q.res_cols = last ? 0 : WG_C; q.skip_store = i == 0;
            if (launch_wg_gemm(q, st)) return -1;
        }
        const int c = wg_channels(d, k);
        WgTailParams t = {};
        t.R = static_cast<int>(R); t.rowinfo = rowinfo; t.state = state;
        t.cur = 1; t.o = 8 - c; t.nh = c / 2;
        t.skip32 = skip; t.end_w = w->end_w[k]; t.end_b = w->end_b[k]; t.inv_w = w->inv_w[k];
        const bool inject = k > 0 && k % d->n_early_every == 0 && d->n_early_size > 0;
        t.inj_lo = inject ? 8 - c - d->n_early_size : 0; t.inj_hi = inject ? 8 - c : 0;
        t.noise = noise; t.Tg_max = L.Tg_max; t.sigma = sigma;
        if (k > 0) {
            const int cn = wg_channels(d, k - 1);
            t.next = 1; t.o_next = 8 - cn; t.nh_next = cn / 2; t.start_w = w->start_w[k - 1]; t.start_b = w->start_b[k - 1];
            t.h32 = h32; t.h16 = h16;
        } else {
            t.next = 0; t.audio = audio;
        }
        if (launch_wg_tail(t, st)) return -1;
    }
    return 0;
}

}  // extern "C"
