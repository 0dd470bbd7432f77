// Fused content attention for the Flowtron AR step (flowtron.py:559-592, 544-557), sm_90a.
//
//   e[b,t,l]  = (sum_a v_a tanh(Q[b,t,a] + K[b,l,a])) / temperature ;  -inf at padded keys
//   p         = softmax_l(e)
//   no prior : attn = p,                      attn_logprob = log(p + 1e-8)
//   prior    : lp = log(p+1e-20)+log(prior+1e-20), attn_logprob = lp, attn = softmax_l(mask(lp))
//   ctx[t,b]  = sum_l attn[b,t,l] V[b,l]
//
// The reference materialises the [B,T,L,A] tanh tensor (12 GB at B=32,T=1000,L=160); here it only ever
// exists as a 4x8 register tile per thread.  tanh(q+k) is evaluated as 1 - 2/(e^{2q} e^{2k} + 1): the
// exponentials are taken once per tile element when it is staged in shared memory, so the inner loop is
// 2 FMA + 1 MUFU.RCP per (t,l,a) -- the kernel is bound by the SFU pipe (16 rcp/clk/SM), not by HBM.
// The backward kernel recomputes the tile the same way and reduces dQ (shuffles), dK/dV (shared +
// global float atomics across t-tiles) and dv.
// Both kernels keep a 64-query tile's rows of scores (forward) / attention gradients (backward) in shared memory while
// they fit in a block's 227 KiB (L <= 672 at A = 640); longer texts run the kGlobalRows instantiations, which keep those
// rows in a caller-provided global area instead (attn_rows_floats) and are otherwise the same code (DESIGN.md 4.16).
#include "ptx.cuh"
#include "ft_internal.h"
#include "../../include/flowtron_b200.h"

namespace ft {

constexpr int AT_TT = 64;        // queries per CTA
constexpr int AT_LB = 128;       // keys per l-block
constexpr int AT_AC = 64;        // attention channels per chunk
constexpr int AT_THREADS = 256;
constexpr int SQ_LD = AT_TT + 4;     // 68: keeps float4 rows 16-byte aligned, spreads banks
constexpr int SK_LD = AT_LB + 4;     // 132

struct AttnFwdParams {
    int t_begin, t_end;                  // query rows [t_begin, t_end) of this launch (t_begin a multiple of the tile height)
    int T, B, L, A;
    const float* Q; long long ldq;       // [T*B, A] row = t*B + b
    const float* K; long long ldk;       // [L*B, A] row = l*B + b
    const float* V; long long ldv;       // [L*B, A]
    const float* v;                      // [A]
    const int* in_lens;                  // [B] valid keys (null: all)
    const int* out_lens;                 // [B] valid queries (null: all)
    const float* prior;                  // [B,T,L] or null
    int reversed;                        // prior row for flow-time t is r_b(t) (AR_Back_Step)
    float inv_temperature;
    float* attn; float* logprob;         // [B,T,L]
    float* p_save;                       // [B,T,L] first softmax (only when prior), or null
    __half* ctx16; long long ldc;        // ctx (fp16) written at ctx16[(t*B+b)*ldc + a]
    float* ctx32; long long ldc32;       // optional fp32 ctx (null ok)
    float* rows;                         // kGlobalRows: score rows [B][T rounded up to 64][Lr + 4]
};

__device__ __forceinline__ float exp2x_clamped(float x) {               // e^{2x}, x clamped to +-40
    float xc = fminf(fmaxf(x, -40.f), 40.f);
    return fast_ex2(2.8853900817779268f * xc);
}

// score accumulation for one staged (query, key, channel) chunk; NJ = key columns per thread actually needed.
// The MUFU (XU) pipe bounds this loop, so two reciprocals share one MUFU.RCP:
//   1/x0 = x1 * rcp(x0 x1),  1/x1 = x0 * rcp(x0 x1)      (x = e^{2q} e^{2k} + 1 >= 1)
// x is clamped to 2^60 so the product stays finite (1/x < 1e-18 there: far below fp32 resolution of tanh = 1 - 2/x).
template <int NJ>
__device__ __forceinline__ void score_chunk(float (&acc)[4][8], const float* __restrict__ sQ, const float* __restrict__ sK,
                                            const float* __restrict__ sva, int na, int ty, int tx) {
    constexpr float kBig = 1152921504606846976.f;     // 2^60
#pragma unroll 2
    for (int a = 0; a < na; ++a) {
        const float4 q4 = *reinterpret_cast<const float4*>(&sQ[a * SQ_LD + 4 * ty]);
        const float va = sva[a];
        float k[NJ];
#pragma unroll
        for (int j = 0; j < NJ; ++j) k[j] = sK[a * SK_LD + tx + 16 * j];
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
            const float x0 = fminf(fmaf(q4.x, k[j], 1.0f), kBig), x1 = fminf(fmaf(q4.y, k[j], 1.0f), kBig);
            const float x2 = fminf(fmaf(q4.z, k[j], 1.0f), kBig), x3 = fminf(fmaf(q4.w, k[j], 1.0f), kBig);
            const float w01 = va * fast_rcp(x0 * x1), w23 = va * fast_rcp(x2 * x3);
            acc[0][j] = fmaf(x1, w01, acc[0][j]);
            acc[1][j] = fmaf(x0, w01, acc[1][j]);
            acc[2][j] = fmaf(x3, w23, acc[2][j]);
            acc[3][j] = fmaf(x2, w23, acc[3][j]);
        }
    }
}

// A tile's rows in the global row area: rows [t0, t0 + 64) of utterance b.  t_begin is a multiple of 64 and a launch
// ends at a multiple of 64 or at T, so every tile of the area belongs to one launch only (the overlapped chunks of the
// training forward never share one).
__device__ __forceinline__ float* tile_rows(float* rows, int b, int T, int t0, int ld) {
    const int Tp = (T + AT_TT - 1) / AT_TT * AT_TT;
    return rows + (static_cast<long long>(b) * Tp + t0) * ld;
}

template <bool kGlobalRows>
__global__ void __launch_bounds__(AT_THREADS, 2)
attn_fwd_kernel(AttnFwdParams p) {
    extern __shared__ float smf[];
    const int Lr = (p.L + 31) & ~31;                  // score row pitch: keys rounded up to a warp
    const int SE_LD = Lr + 4;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int b = blockIdx.y, t0 = p.t_begin + blockIdx.x * AT_TT;
    float* sQ = smf;                                  // [AT_AC][SQ_LD]
    float* sK = sQ + AT_AC * SQ_LD;                   // [AT_AC][SK_LD]   (also the V chunk [64][AT_AC+4])
    float* sE = kGlobalRows ? tile_rows(p.rows, b, p.T, t0, SE_LD) : sK + AT_AC * SK_LD;   // [AT_TT][Lr+4]
    float* sv = kGlobalRows ? sK + AT_AC * SK_LD : sE + AT_TT * (Lr + 4);                  // [A]
    __shared__ float s_sumv;

    const int out_len = p.out_lens ? p.out_lens[b] : p.T;
    const int in_len = p.in_lens ? p.in_lens[b] : p.L;
    const int nrows = min(AT_TT, p.t_end - t0);

    if (t0 >= out_len) {      // tile entirely in the padded region: values there are outside the contract; keep them finite
        const float lp0 = logf(1e-8f);
        for (int i = tid; i < nrows * p.L; i += AT_THREADS) {
            const int tt = i / p.L, l = i % p.L;
            const long long o = (static_cast<long long>(b) * p.T + t0 + tt) * p.L + l;
            p.attn[o] = 0.f;
            p.logprob[o] = lp0;
            if (p.p_save) p.p_save[o] = 0.f;
        }
        for (int i = tid; i < nrows * p.A; i += AT_THREADS) {
            const int tt = i / p.A, a = i % p.A;
            const long long r = static_cast<long long>(t0 + tt) * p.B + b;
            p.ctx16[r * p.ldc + a] = __float2half(0.f);
            if (p.ctx32) p.ctx32[r * p.ldc32 + a] = 0.f;
        }
        return;
    }

    for (int i = tid; i < p.A; i += AT_THREADS) sv[i] = p.v[i];
    __syncthreads();
    if (warp == 0) {
        float s = 0.f;
        for (int i = lane; i < p.A; i += 32) s += sv[i];
#pragma unroll
        for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) s_sumv = s;
    }

    const int ty = tid >> 4, tx = tid & 15;           // 16 x 16 thread grid: rows 4*ty.., keys tx + 16*j
    // keys >= in_len are masked to probability exactly 0 (flowtron.py:545-553): their scores are never read, so the
    // score and context loops stop at this utterance's text length instead of the batch maximum.
    const int Lk = min(p.L, in_len);
    const int nlb = (Lk + AT_LB - 1) / AT_LB;
    for (int lb = 0; lb < nlb; ++lb) {
        const int nl = min(AT_LB, Lk - lb * AT_LB);
        const int nj = (nl + 15) >> 4;                // key columns per thread that hold real keys (block-uniform)
        float acc[4][8];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
        for (int ac = 0; ac < p.A; ac += AT_AC) {
            __syncthreads();
            {   // stage e^{2Q} chunk: 64 t x 64 a, and e^{2K}: nj*16 keys x 64 a
                const int aa = tid & 63;
                for (int tt = tid >> 6; tt < AT_TT; tt += AT_THREADS / 64) {
                    float q = 0.f;
                    if (tt < nrows && ac + aa < p.A) q = p.Q[(static_cast<long long>(t0 + tt) * p.B + b) * p.ldq + ac + aa];
                    sQ[aa * SQ_LD + tt] = exp2x_clamped(q);
                }
                for (int ll = tid >> 6; ll < nj * 16; ll += AT_THREADS / 64) {
                    const int l = lb * AT_LB + ll;
                    float k = 0.f;
                    if (l < p.L && ac + aa < p.A) k = p.K[(static_cast<long long>(l) * p.B + b) * p.ldk + ac + aa];
                    sK[aa * SK_LD + ll] = exp2x_clamped(k);
                }
            }
            __syncthreads();
            const int na = min(AT_AC, p.A - ac);
            switch ((nj + 1) >> 1) {
                case 1: score_chunk<2>(acc, sQ, sK, sv + ac, na, ty, tx); break;
                case 2: score_chunk<4>(acc, sQ, sK, sv + ac, na, ty, tx); break;
                case 3: score_chunk<6>(acc, sQ, sK, sv + ac, na, ty, tx); break;
                default: score_chunk<8>(acc, sQ, sK, sv + ac, na, ty, tx); break;
            }
        }
        const float sumv = s_sumv;
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int col = lb * AT_LB + tx + 16 * j;
                if (col < Lr) sE[(4 * ty + i) * SE_LD + col] = (sumv - 2.f * acc[i][j]) * p.inv_temperature;
            }
    }
    __syncthreads();

    // ---------------------------------------------------------------- softmax (+ prior posterior), one warp per row
    for (int tt = warp; tt < nrows; tt += AT_THREADS / 32) {
        float* e = sE + tt * SE_LD;
        const int t = t0 + tt;
        float m = -INFINITY;
        for (int l = lane; l < in_len; l += 32) m = fmaxf(m, e[l]);
#pragma unroll
        for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
        float s = 0.f;
        for (int l = lane; l < p.L; l += 32) {
            const float x = (l < in_len) ? expf(e[l] - m) : 0.f;
            e[l] = x;
            s += x;
        }
#pragma unroll
        for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        const float inv = 1.f / s;
        const long long o0 = (static_cast<long long>(b) * p.T + t) * p.L;
        if (!p.prior) {
            for (int l = lane; l < p.L; l += 32) {
                const float pr = e[l] * inv;
                e[l] = pr;
                p.attn[o0 + l] = pr;
                p.logprob[o0 + l] = logf(pr + 1e-8f);
            }
        } else {
            const int tp = p.reversed ? back_index(t, out_len, p.T) : t;
            const float* prow = p.prior + (static_cast<long long>(b) * p.T + tp) * p.L;
            float m2 = -INFINITY;
            for (int l = lane; l < p.L; l += 32) {
                const float pr = e[l] * inv;
                if (p.p_save) p.p_save[o0 + l] = pr;
                const float lp = logf(pr + 1e-20f) + logf(prow[l] + 1e-20f);
                p.logprob[o0 + l] = lp;                       // cloned before masking (flowtron.py:550)
                e[l] = lp;
                if (l < in_len) m2 = fmaxf(m2, lp);
            }
#pragma unroll
            for (int o = 16; o; o >>= 1) m2 = fmaxf(m2, __shfl_xor_sync(0xffffffffu, m2, o));
            float s2 = 0.f;
            for (int l = lane; l < p.L; l += 32) {
                const float x = (l < in_len) ? expf(e[l] - m2) : 0.f;
                e[l] = x;
                s2 += x;
            }
#pragma unroll
            for (int o = 16; o; o >>= 1) s2 += __shfl_xor_sync(0xffffffffu, s2, o);
            const float inv2 = 1.f / s2;
            for (int l = lane; l < p.L; l += 32) {
                const float a2 = e[l] * inv2;
                e[l] = a2;
                p.attn[o0 + l] = a2;
            }
        }
        for (int l = p.L + lane; l < Lr; l += 32) e[l] = 0.f;
    }
    __syncthreads();

    // ---------------------------------------------------------------- context: ctx[t, a] = sum_l attn[t,l] V[l,a]
    float* sV = sK;                                    // [64 keys][AT_AC + 4]  (64*68 floats fit inside sK's 64*132)
    constexpr int SV_LD = AT_AC + 4;
    for (int ac = 0; ac < p.A; ac += AT_AC) {
        float c4[4][4];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) c4[i][j] = 0.f;
        for (int l0 = 0; l0 < Lk; l0 += 64) {
            __syncthreads();
            {
                const int aa = tid & 63;
                for (int ll = tid >> 6; ll < 64; ll += AT_THREADS / 64) {
                    const int l = l0 + ll;
                    float x = 0.f;
                    if (l < Lk && ac + aa < p.A) x = p.V[(static_cast<long long>(l) * p.B + b) * p.ldv + ac + aa];
                    sV[ll * SV_LD + aa] = x;
                }
            }
            __syncthreads();
            const int nl = min(64, Lk - l0);
            for (int l = 0; l < nl; ++l) {
                const float4 v4 = *reinterpret_cast<const float4*>(&sV[l * SV_LD + 4 * tx]);
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const float w = sE[(4 * ty + i) * SE_LD + l0 + l];
                    c4[i][0] = fmaf(w, v4.x, c4[i][0]);
                    c4[i][1] = fmaf(w, v4.y, c4[i][1]);
                    c4[i][2] = fmaf(w, v4.z, c4[i][2]);
                    c4[i][3] = fmaf(w, v4.w, c4[i][3]);
                }
            }
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int tt = 4 * ty + i;
            if (tt < nrows && ac + 4 * tx < p.A) {
                const long long r = static_cast<long long>(t0 + tt) * p.B + b;
                __half2 h0 = __floats2half2_rn(c4[i][0], c4[i][1]), h1 = __floats2half2_rn(c4[i][2], c4[i][3]);
                uint2 pk = make_uint2(*reinterpret_cast<uint32_t*>(&h0), *reinterpret_cast<uint32_t*>(&h1));
                *reinterpret_cast<uint2*>(p.ctx16 + r * p.ldc + ac + 4 * tx) = pk;
                if (p.ctx32)
                    *reinterpret_cast<float4*>(p.ctx32 + r * p.ldc32 + ac + 4 * tx) = make_float4(c4[i][0], c4[i][1], c4[i][2], c4[i][3]);
            }
        }
    }
}

// =================================================================================================== backward
struct AttnBwdParams {
    int t_begin, t_end;                  // query rows [t_begin, t_end) of this launch
    int T, B, L, A;
    const float* Q; long long ldq;
    const float* K; long long ldk;
    const float* V; long long ldv;
    const float* v;
    const int* in_lens; const int* out_lens;
    const float* attn;                    // [B,T,L] saved output
    const float* p_save;                  // [B,T,L] first softmax when prior was used, else null
    int has_prior;
    float inv_temperature;
    const float* dctx; long long lddc;    // [T*B, lddc] gradient w.r.t. ctx (fp32)
    const float* dattn_ext;               // [B,T,L] or null : gradient w.r.t. returned attn
    const float* dlp_ext;                 // [B,T,L] or null : gradient w.r.t. returned attn_logprob
    const float* scale;                   // device {S, 1/S} or null: external grads * S, dv * 1/S
    float* dQ; long long lddq;            // [T*B, A] written
    float* dK; long long lddk;            // [L*B, A] accumulated (atomicAdd; caller zeroes)
    float* dV; long long lddv;            // [L*B, A] accumulated
    float* dv;                            // [A] accumulated
    float* rows;                          // kGlobalRows: dattn / de rows [B][T rounded up to 64][Lr + 4]
};

template <bool kGlobalRows>
__global__ void __launch_bounds__(AT_THREADS, 2)
attn_bwd_kernel(AttnBwdParams p) {
    extern __shared__ float smf[];
    const int Lr = (p.L + 31) & ~31;
    const int SE_LD = Lr + 4;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int b = blockIdx.y, t0 = p.t_begin + blockIdx.x * AT_TT;
    float* sQ = smf;                                  // [AT_AC][SQ_LD]   (phase 3: e^{2q} as [AT_TT][65])
    float* sK = sQ + AT_AC * SQ_LD;                   // [AT_AC][SK_LD]   (phase 3: e^{2k} as [AT_LB][65])
    float* sD = kGlobalRows ? tile_rows(p.rows, b, p.T, t0, SE_LD) : sK + AT_AC * SK_LD;   // [AT_TT][SE_LD]  dattn -> de
    float* sv = kGlobalRows ? sK + AT_AC * SK_LD : sD + AT_TT * SE_LD;                     // [A]
    float* sdv = sv + p.A;                            // [A]
    __shared__ float s_sumde;                         // sum of de over the tile (dv needs sum de (1 - 2r) = sum de - 2 sum de r)

    const int out_len = p.out_lens ? p.out_lens[b] : p.T;
    const int in_len = p.in_lens ? p.in_lens[b] : p.L;
    const int nrows = min(AT_TT, p.t_end - t0);
    const int ty = tid >> 4, tx = tid & 15;

    if (t0 >= out_len) {                              // forward wrote constants here: no gradient
        for (int i = tid; i < nrows * p.A; i += AT_THREADS) {
            const int tt = i / p.A, a = i % p.A;
            p.dQ[(static_cast<long long>(t0 + tt) * p.B + b) * p.lddq + a] = 0.f;
        }
        return;
    }
    for (int i = tid; i < p.A; i += AT_THREADS) { sv[i] = p.v[i]; sdv[i] = 0.f; }
    if (tid == 0) s_sumde = 0.f;
    const float S = p.scale ? p.scale[0] : 1.f, iS = p.scale ? p.scale[1] : 1.f;
    // keys >= in_len: attn == 0 and de == 0 exactly (masked softmax), so every key loop below stops at the text length
    const int Lk = min(p.L, in_len);

    // ---------------------------------------------------------------- 1. dattn[t,l] = dctx[t,:] . V[l,:]  (+ext);  dV += attn^T dctx
    for (int i = tid; i < AT_TT * SE_LD; i += AT_THREADS) sD[i] = 0.f;
    const float* attn_b = p.attn + (static_cast<long long>(b) * p.T + t0) * p.L;      // rows of this tile, pitch L (L2-resident)
    __syncthreads();
    float* sC = sQ;                                   // dctx chunk  [AT_TT][AT_AC+4]  (fits in sQ: 64*68)
    float* sV = sK;                                   // V chunk     [64 keys][AT_AC+4]  (64*68 floats fit in sK)
    constexpr int SC_LD = AT_AC + 4;
    for (int ac = 0; ac < p.A; ac += AT_AC) {
        __syncthreads();
        {
            const int aa = tid & 63;
            for (int tt = tid >> 6; tt < AT_TT; tt += AT_THREADS / 64) {
                float x = 0.f;
                if (tt < nrows && t0 + tt < out_len && ac + aa < p.A)
                    x = p.dctx[(static_cast<long long>(t0 + tt) * p.B + b) * p.lddc + ac + aa];
                sC[tt * SC_LD + aa] = x;
            }
        }
        for (int l0 = 0; l0 < Lk; l0 += 64) {
            __syncthreads();
            {
                const int aa = tid & 63;
                for (int ll = tid >> 6; ll < 64; ll += AT_THREADS / 64) {
                    const int l = l0 + ll;
                    float x = 0.f;
                    if (l < Lk && ac + aa < p.A) x = p.V[(static_cast<long long>(l) * p.B + b) * p.ldv + ac + aa];
                    sV[ll * SC_LD + aa] = x;
                }
            }
            __syncthreads();
            // dattn partial: thread (ty,tx) -> rows 4ty..+3, keys l0 + tx + 16j (j<4)
            float d[4][4];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) d[i][j] = 0.f;
            for (int a = 0; a < AT_AC; a += 4) {
                float4 c[4], vv[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) c[i] = *reinterpret_cast<const float4*>(&sC[(4 * ty + i) * SC_LD + a]);
#pragma unroll
                for (int j = 0; j < 4; ++j) vv[j] = *reinterpret_cast<const float4*>(&sV[(tx + 16 * j) * SC_LD + a]);
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int j = 0; j < 4; ++j)
                        d[i][j] += c[i].x * vv[j].x + c[i].y * vv[j].y + c[i].z * vv[j].z + c[i].w * vv[j].w;
            }
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int col = l0 + tx + 16 * j;
                    if (col < Lr) sD[(4 * ty + i) * SE_LD + col] += d[i][j];
                }
            // dV[l, a] += sum_t attn[t,l] dctx[t,a]: thread -> keys l0 + 4*ty.. +3, channels 4*tx..+3
            float g[4][4];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) g[i][j] = 0.f;
            for (int tt = 0; tt < nrows; ++tt) {
                const float4 c = *reinterpret_cast<const float4*>(&sC[tt * SC_LD + 4 * tx]);
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int l = l0 + 4 * ty + i;
                    const float w = (l < Lk) ? __ldg(attn_b + static_cast<long long>(tt) * p.L + l) : 0.f;
                    g[i][0] = fmaf(w, c.x, g[i][0]); g[i][1] = fmaf(w, c.y, g[i][1]);
                    g[i][2] = fmaf(w, c.z, g[i][2]); g[i][3] = fmaf(w, c.w, g[i][3]);
                }
            }
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int l = l0 + 4 * ty + i;
                if (l < Lk && ac + 4 * tx < p.A) {
                    float* dst = p.dV + (static_cast<long long>(l) * p.B + b) * p.lddv + ac + 4 * tx;
#pragma unroll
                    for (int j = 0; j < 4; ++j) atomicAdd(dst + j, g[i][j]);
                }
            }
        }
    }
    __syncthreads();

    // ---------------------------------------------------------------- 2. softmax backward(s): sD <- de
    for (int tt = warp; tt < nrows; tt += AT_THREADS / 32) {
        const int t = t0 + tt;
        float* d = sD + tt * SE_LD;
        const float* at = attn_b + static_cast<long long>(tt) * p.L;
        const long long o0 = (static_cast<long long>(b) * p.T + t) * p.L;
        if (t >= out_len) {
            for (int l = lane; l < Lr; l += 32) d[l] = 0.f;
            continue;
        }
        if (!p.has_prior) {
            // attn = p = softmax(e); logprob = log(p + 1e-8)
            float dot = 0.f;
            for (int l = lane; l < p.L; l += 32) {
                float g = d[l];
                if (p.dattn_ext) g += S * p.dattn_ext[o0 + l];
                if (p.dlp_ext) g += S * p.dlp_ext[o0 + l] / (at[l] + 1e-8f);
                d[l] = g;
                dot += g * at[l];
            }
#pragma unroll
            for (int o = 16; o; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
            float sde = 0.f;
            for (int l = lane; l < Lr; l += 32) {
                const float de = (l < in_len) ? at[l] * (d[l] - dot) * p.inv_temperature : 0.f;
                d[l] = de;
                sde += de;
            }
#pragma unroll
            for (int o = 16; o; o >>= 1) sde += __shfl_xor_sync(0xffffffffu, sde, o);
            if (lane == 0) atomicAdd(&s_sumde, sde);
        } else {
            // attn = softmax(mask(lp)), lp = log(p+1e-20) + log(prior+1e-20), p = softmax(e)
            float dot = 0.f;
            for (int l = lane; l < p.L; l += 32) {
                float g = d[l];
                if (p.dattn_ext) g += S * p.dattn_ext[o0 + l];
                d[l] = g;
                dot += g * at[l];
            }
#pragma unroll
            for (int o = 16; o; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
            float dot2 = 0.f;
            for (int l = lane; l < p.L; l += 32) {
                float dlp = (l < in_len) ? at[l] * (d[l] - dot) : 0.f;       // through the masked 2nd softmax
                if (p.dlp_ext) dlp += S * p.dlp_ext[o0 + l];                 // logprob is the pre-mask clone
                const float pr = p.p_save[o0 + l];
                const float dp = dlp / (pr + 1e-20f);
                d[l] = dp;
                dot2 += dp * pr;
            }
#pragma unroll
            for (int o = 16; o; o >>= 1) dot2 += __shfl_xor_sync(0xffffffffu, dot2, o);
            float sde = 0.f;
            for (int l = lane; l < Lr; l += 32) {
                const float pr = (l < p.L) ? p.p_save[o0 + l] : 0.f;
                const float de = (l < in_len) ? pr * (d[l] - dot2) * p.inv_temperature : 0.f;
                d[l] = de;
                sde += de;
            }
#pragma unroll
            for (int o = 16; o; o >>= 1) sde += __shfl_xor_sync(0xffffffffu, sde, o);
            if (lane == 0) atomicAdd(&s_sumde, sde);
        }
    }
    __syncthreads();

    // ---------------------------------------------------------------- 3. score backward, tanh recomputed
    // A thread owns (16 rows, 1 channel) and walks the keys: g = de * r (1 - r), r = 1/(e^{2q} e^{2k} + 1), feeds
    // dQ[row] (register, summed over keys) and dK[key] (register, summed over the thread's 16 rows) from ONE reciprocal
    // (tanh = 1 - 2r, 1 - tanh^2 = 4 r (1 - r)).  dK is then reduced over the four row groups through a 16 KB shared
    // buffer once per 16 keys and leaves with one global atomic per (key, channel).  History: v1 evaluated r once but
    // paid ~30 shuffles + 8 shared atomics per 32 elements; v2 ran two reduction-free passes (2 MUFU per element) and
    // sat at the MUFU bound; this version has 1 MUFU + 6 FMA-pipe ops per element.
    {
        constexpr int QP = 65;                        // [row][channel] pitch: lanes walk channels -> conflict-free
        constexpr int KB3 = 64;                       // keys staged per block
        constexpr int KS = 16;                        // keys per dK reduction round
        float* sQt = sQ;                              // [AT_TT][QP]
        float* sKt = sK;                              // [KB3][QP]
        float* sRed = sK + KB3 * QP;                  // [4 row groups][KS][64]   (4160 + 4096 floats <= AT_AC * SK_LD)
        static_assert(KB3 * QP + 4 * KS * 64 <= AT_AC * SK_LD, "phase-3 buffers must fit in sK");
        const int a_l = tid & 63, grp = tid >> 6;     // channel lane; row group
        const float sumde = s_sumde;
        for (int ac = 0; ac < p.A; ac += AT_AC) {
            float dq[16];
#pragma unroll
            for (int i = 0; i < 16; ++i) dq[i] = 0.f;
            float dvr = 0.f;                          // sum de * r
            const bool a_ok = ac + a_l < p.A;
            __syncthreads();
            for (int i = tid; i < AT_TT * AT_AC; i += AT_THREADS) {
                const int tt = i >> 6, aa = i & 63;
                float q = 0.f;
                if (tt < nrows && ac + aa < p.A) q = p.Q[(static_cast<long long>(t0 + tt) * p.B + b) * p.ldq + ac + aa];
                sQt[tt * QP + aa] = exp2x_clamped(q);
            }
            for (int l0 = 0; l0 < Lk; l0 += KB3) {
                const int nl = min(KB3, Lk - l0);
                const int nl4 = (nl + 3) & ~3;        // de is 0 in [Lk, Lr): padded keys only need finite e^{2k}
                __syncthreads();
                for (int i = tid; i < nl4 * AT_AC; i += AT_THREADS) {
                    const int ll = i >> 6, aa = i & 63;
                    const int l = l0 + ll;
                    float k = 0.f;
                    if (l < Lk && ac + aa < p.A) k = p.K[(static_cast<long long>(l) * p.B + b) * p.ldk + ac + aa];
                    sKt[ll * QP + aa] = exp2x_clamped(k);
                }
                __syncthreads();
                float eq[16];
#pragma unroll
                for (int i = 0; i < 16; ++i) eq[i] = sQt[(grp * 16 + i) * QP + a_l];
                for (int s0 = 0; s0 < nl; s0 += KS) {
                    const int ns = min(KS, nl - s0);
                    float dk[KS];
#pragma unroll
                    for (int j = 0; j < KS; ++j) dk[j] = 0.f;
#pragma unroll
                    for (int j4 = 0; j4 < KS / 4; ++j4) {
                        if (4 * j4 < ns) {            // block-uniform
                            float ek[4];
#pragma unroll
                            for (int e = 0; e < 4; ++e) ek[e] = sKt[(s0 + 4 * j4 + e) * QP + a_l];
#pragma unroll
                            for (int i = 0; i < 16; ++i) {
                                const float4 d4 = *reinterpret_cast<const float4*>(&sD[(grp * 16 + i) * SE_LD + l0 + s0 + 4 * j4]);
                                const float dd[4] = {d4.x, d4.y, d4.z, d4.w};
#pragma unroll
                                for (int e = 0; e < 4; ++e) {
                                    const float r = fast_rcp(fmaf(eq[i], ek[e], 1.0f));
                                    const float m = dd[e] * fmaf(-r, r, r);
                                    dq[i] += m;
                                    dk[4 * j4 + e] += m;
                                    dvr = fmaf(dd[e], r, dvr);
                                }
                            }
                        }
                    }
                    __syncthreads();                  // previous round's readers of sRed are done
#pragma unroll
                    for (int j = 0; j < KS; ++j) sRed[(grp * KS + j) * 64 + a_l] = dk[j];
                    __syncthreads();
#pragma unroll
                    for (int k4 = 0; k4 < (KS * 64) / AT_THREADS; ++k4) {
                        const int idx = tid + AT_THREADS * k4;
                        const int j = idx >> 6, aa = idx & 63;
                        const float x = (sRed[(0 * KS + j) * 64 + aa] + sRed[(1 * KS + j) * 64 + aa]) +
                                        (sRed[(2 * KS + j) * 64 + aa] + sRed[(3 * KS + j) * 64 + aa]);
                        if (j < ns && ac + aa < p.A && x != 0.f)
                            atomicAdd(p.dK + (static_cast<long long>(l0 + s0 + j) * p.B + b) * p.lddk + ac + aa, x * 4.f * sv[ac + aa]);
                    }
                }
            }
            if (a_ok) {
                const float s4 = 4.f * sv[ac + a_l];
#pragma unroll
                for (int i = 0; i < 16; ++i) {
                    const int tt = grp * 16 + i;
                    if (tt < nrows) p.dQ[(static_cast<long long>(t0 + tt) * p.B + b) * p.lddq + ac + a_l] = dq[i] * s4;
                }
                atomicAdd(&sdv[ac + a_l], (grp == 0 ? sumde : 0.f) - 2.f * dvr);
            }
        }
    }
    __syncthreads();
    for (int i = tid; i < p.A; i += AT_THREADS) {
        const float x = sdv[i];
        if (x != 0.f) atomicAdd(p.dv + i, x * iS);
    }
}

// =================================================================================================== host
constexpr size_t kSmemPerBlock = 227 * 1024;     // H100 opt-in shared memory per block

static size_t attn_fwd_smem(int L, int A, bool global_rows) {
    const int Lr = (L + 31) & ~31;
    const size_t rows = global_rows ? 0 : static_cast<size_t>(AT_TT) * (Lr + 4);
    return sizeof(float) * (static_cast<size_t>(AT_AC) * SQ_LD + AT_AC * SK_LD + rows + A) + 64;
}
static size_t attn_bwd_smem(int L, int A, bool global_rows) {
    const int Lr = (L + 31) & ~31;
    const size_t rows = global_rows ? 0 : static_cast<size_t>(AT_TT) * (Lr + 4);
    return sizeof(float) * (static_cast<size_t>(AT_AC) * SQ_LD + AT_AC * SK_LD + rows + 2 * A) + 64;
}

// One rule for both directions (the backward needs A floats more): the shared-memory kernels run while the backward's rows
// fit, i.e. up to L = 672 at A = 640.
bool attn_rows_in_global(int L, int A) { return attn_bwd_smem(L, A, false) > kSmemPerBlock; }
size_t attn_rows_floats(int T, int B, int L) {
    const size_t Tp = (static_cast<size_t>(T) + AT_TT - 1) / AT_TT * AT_TT;
    return static_cast<size_t>(B) * Tp * (((L + 31) & ~31) + 4);
}

int launch_attn_fwd(const AttnFwdArgs& a, cudaStream_t st) {
    if (a.L > FT_MAX_TEXT_LEN) return ft_set_error("attention: L > FT_MAX_TEXT_LEN (1024) not supported");
    if (a.A % 4) return ft_set_error("attention: A must be a multiple of 4");
    const bool global_rows = attn_rows_in_global(a.L, a.A);
    if (global_rows && !a.rows) return ft_set_error("attention: this L needs the global row area (AttnFwdArgs::rows)");
    AttnFwdParams p;
    p.T = a.T; p.B = a.B; p.L = a.L; p.A = a.A;
    p.Q = a.Q; p.ldq = a.ldq; p.K = a.K; p.ldk = a.ldk; p.V = a.V; p.ldv = a.ldv; p.v = a.v;
    p.in_lens = a.in_lens; p.out_lens = a.out_lens; p.prior = a.prior; p.reversed = a.reversed;
    p.inv_temperature = 1.0f / a.temperature;
    p.attn = a.attn; p.logprob = a.logprob; p.p_save = a.p_save;
    p.ctx16 = static_cast<__half*>(a.ctx16); p.ldc = a.ldc; p.ctx32 = a.ctx32; p.ldc32 = a.ldc32;
    p.rows = a.rows;
    const size_t smem = attn_fwd_smem(a.L, a.A, global_rows);
    auto kern = global_rows ? attn_fwd_kernel<true> : attn_fwd_kernel<false>;
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    p.t_begin = a.t_begin; p.t_end = a.t_end > 0 ? a.t_end : a.T;
    if (p.t_begin % AT_TT || p.t_begin < 0 || p.t_end > a.T || p.t_end <= p.t_begin) return ft_set_error("attention: bad query range");
    dim3 grid((p.t_end - p.t_begin + AT_TT - 1) / AT_TT, a.B);
    TimeScope ts("attn_fwd", p.t_end - p.t_begin, a.B, a.L, st);
    kern<<<grid, AT_THREADS, smem, st>>>(p);
    ft_count_launch(1);
    return ft_check_launch("attn_fwd_kernel");
}

int launch_attn_bwd(const AttnBwdArgs& a, cudaStream_t st) {
    if (a.L > FT_MAX_TEXT_LEN) return ft_set_error("attention backward: L > FT_MAX_TEXT_LEN (1024) not supported");
    const bool global_rows = attn_rows_in_global(a.L, a.A);
    if (global_rows && !a.rows) return ft_set_error("attention backward: this L needs the global row area (AttnBwdArgs::rows)");
    AttnBwdParams p;
    p.T = a.T; p.B = a.B; p.L = a.L; p.A = a.A;
    p.Q = a.Q; p.ldq = a.ldq; p.K = a.K; p.ldk = a.ldk; p.V = a.V; p.ldv = a.ldv; p.v = a.v;
    p.in_lens = a.in_lens; p.out_lens = a.out_lens; p.attn = a.attn; p.p_save = a.p_save;
    p.has_prior = a.p_save != nullptr; p.inv_temperature = 1.0f / a.temperature;
    p.dctx = a.dctx; p.lddc = a.lddc; p.dattn_ext = a.dattn_ext; p.dlp_ext = a.dlp_ext; p.scale = a.scale;
    p.dQ = a.dQ; p.lddq = a.lddq; p.dK = a.dK; p.lddk = a.lddk; p.dV = a.dV; p.lddv = a.lddv; p.dv = a.dv;
    p.rows = a.rows;
    const size_t smem = attn_bwd_smem(a.L, a.A, global_rows);
    auto kern = global_rows ? attn_bwd_kernel<true> : attn_bwd_kernel<false>;
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    p.t_begin = a.t_begin; p.t_end = a.t_end > 0 ? a.t_end : a.T;
    if (p.t_begin % AT_TT || p.t_begin < 0 || p.t_end > a.T || p.t_end <= p.t_begin) return ft_set_error("attention backward: bad query range");
    dim3 grid((p.t_end - p.t_begin + AT_TT - 1) / AT_TT, a.B);
    TimeScope ts("attn_bwd", p.t_end - p.t_begin, a.B, a.L, st);
    kern<<<grid, AT_THREADS, smem, st>>>(p);
    ft_count_launch(1);
    return ft_check_launch("attn_bwd_kernel");
}

}  // namespace ft
