// The reference `Attention` module on its own (flowtron.py:528-592): Q / K / V projections, the fused attention kernels of
// attention.cu (called, not changed), the forced-weights (`attn` given) branch and the [B, A, T] context layout, forward and
// backward (ft_attention_fwd / ft_attention_bwd).
//
// Layouts: queries [T, B, Dq] and keys / values [L, B, E] are row-major [T*B, Dq] / [L*B, E], so their projections are
// [T*B, A] / [L*B, A] with row t*B + b / l*B + b -- exactly the rows the attention kernels read.  No transposes on the way in;
// the context leaves as [B, A, T] through one batched transpose.
//
// Precision: the forward projections are split-fp16 GEMMs (x = hi + lo, products hi*hi + lo*hi + hi*lo, fp32 accumulate; one
// GEMM over a 3x contraction with activations stored [hi | lo | hi] and weights [hi | hi | lo], as the text encoder does),
// because plain fp16 operands put a ~5e-4 relative error on Q / K, which the tanh score and the softmax carry to attn.  The
// forced-weights context and its backward are batched split-fp16 tensor-core products (attn_bmm_kernel).  The backward
// projections (dgrad / wgrad) run on plain fp16 operands under a device-chosen power-of-two loss scale, as the flow step's do.
#include <mma.h>

#include "encoder_kernels.cuh"
#include "../../include/flowtron_b200.h"

namespace ft {

namespace {

// fp32 rows [R, C] -> split fp16 rows [R, 3C]: activations [hi | lo | hi], weights [hi | hi | lo]
__global__ void attn_split_kernel(const float* __restrict__ src, long long R, int C, int weight, __half* __restrict__ dst) {
    const long long n = R * C;
    for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const long long r = i / C;
        const int c = static_cast<int>(i - r * C);
        __half* row = dst + r * 3 * C;
        if (!weight) {
            store_hlh(row, C, c, src[i]);
        } else {
            __half hi, lo;
            split16(src[i], hi, lo);
            row[c] = hi; row[C + c] = hi; row[2 * C + c] = lo;
        }
    }
}

// dst(b, j, i) = scale * src(b, i, j) for i < ni, j < nj: src(b, i, j) = src[b*sb + i*si + j], dst(b, j, i) = dst[b*db + j*dj + i]
__global__ void attn_transpose_kernel(const float* __restrict__ src, long long sb, long long si, int ni, int nj,
                                      float* __restrict__ dst, long long db, long long dj, const float* __restrict__ scale) {
    __shared__ float tile[32][33];
    const int b = blockIdx.z, i0 = blockIdx.y * 32, j0 = blockIdx.x * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const float s = scale ? scale[0] : 1.f;
    for (int r = ty; r < 32; r += 8) {
        const int i = i0 + r, j = j0 + tx;
        if (i < ni && j < nj) tile[r][tx] = src[b * sb + i * si + j];
    }
    __syncthreads();
    for (int r = ty; r < 32; r += 8) {
        const int j = j0 + r, i = i0 + tx;
        if (i < ni && j < nj) dst[b * db + j * dj + i] = s * tile[tx][r];
    }
}

// Batched strided product on the tensor cores, split fp16:
//   C(b, m, n) = alpha * sum_k A(b, m, k) B(b, k, n)  (+ C(b, m, n) if beta),   alpha = *alpha_ptr or 1
// with X(b, r, c) = X[b * xb + r * xr + c * xc] for every operand.  64 x 64 output tile per CTA, 4 warps of 32 x 32, k in
// chunks of 32 staged in shared memory as hi / lo fp16 (three wmma per fragment pair).  Used for the forced-weights context
// ctx[b, :, t] = sum_l attn[b, t, l] V[l*B + b, :] and its two gradients.
// An operand's optional device `scale` multiplies it in fp32 before the split: an upstream gradient below fp16's normal range
// (6.1e-5) would otherwise land on the subnormal grid in both halves, so the backward stages S * d_output (S the device-chosen
// loss scale) and undoes S in the epilogue's alpha.
struct BmmOperand { const float* p; long long b, r, c; const float* scale = nullptr; };
constexpr int BM_T = 64, BM_K = 32, BM_LD = BM_K + 8, BM_CLD = BM_T + 4, BM_THREADS = 128;

__device__ __forceinline__ void bmm_stage(const BmmOperand& x, int b, int r0, int nr, int k0, int nk, __half* hi, __half* lo) {
    // rows r0.. of the operand (m for A, n for B), k0.. of the contraction, stored [row][k]; walk the unit-stride index fastest
    const bool k_fast = x.c == 1;
    const float s = x.scale ? x.scale[0] : 1.f;
    for (int i = threadIdx.x; i < BM_T * BM_K; i += BM_THREADS) {
        const int rr = k_fast ? i / BM_K : i % BM_T, kk = k_fast ? i % BM_K : i / BM_T;
        float v = 0.f;
        if (rr < nr && kk < nk) v = s * x.p[b * x.b + static_cast<long long>(r0 + rr) * x.r + static_cast<long long>(k0 + kk) * x.c];
        __half h, l;
        split16(v, h, l);
        hi[rr * BM_LD + kk] = h;
        lo[rr * BM_LD + kk] = l;
    }
}

__global__ void __launch_bounds__(BM_THREADS)
attn_bmm_kernel(int M, int N, int K, BmmOperand A, BmmOperand Bt, float* __restrict__ C, long long cb, long long cm, long long cn,
                const float* __restrict__ alpha_ptr, int beta) {
    using namespace nvcuda;
    __shared__ __align__(32) __half sA[2][BM_T * BM_LD];       // [hi, lo][m][k]
    __shared__ __align__(32) __half sB[2][BM_T * BM_LD];       // [hi, lo][n][k]  (col-major K x N)
    __shared__ __align__(32) float sC[BM_T * BM_CLD];
    const int b = blockIdx.z, m0 = blockIdx.y * BM_T, n0 = blockIdx.x * BM_T;
    const int warp = threadIdx.x >> 5, wm = (warp >> 1) * 32, wn = (warp & 1) * 32;
    wmma::fragment<wmma::accumulator, 16, 16, 16, float> acc[2][2];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j) wmma::fill_fragment(acc[i][j], 0.f);
    for (int k0 = 0; k0 < K; k0 += BM_K) {
        __syncthreads();
        bmm_stage(A, b, m0, M - m0, k0, K - k0, sA[0], sA[1]);
        bmm_stage(Bt, b, n0, N - n0, k0, K - k0, sB[0], sB[1]);
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < BM_K; kk += 16) {
            wmma::fragment<wmma::matrix_a, 16, 16, 16, __half, wmma::row_major> ah[2], al[2];
            wmma::fragment<wmma::matrix_b, 16, 16, 16, __half, wmma::col_major> bh[2], bl[2];
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                wmma::load_matrix_sync(ah[i], sA[0] + (wm + 16 * i) * BM_LD + kk, BM_LD);
                wmma::load_matrix_sync(al[i], sA[1] + (wm + 16 * i) * BM_LD + kk, BM_LD);
                wmma::load_matrix_sync(bh[i], sB[0] + (wn + 16 * i) * BM_LD + kk, BM_LD);
                wmma::load_matrix_sync(bl[i], sB[1] + (wn + 16 * i) * BM_LD + kk, BM_LD);
            }
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    wmma::mma_sync(acc[i][j], al[i], bh[j], acc[i][j]);
                    wmma::mma_sync(acc[i][j], ah[i], bl[j], acc[i][j]);
                    wmma::mma_sync(acc[i][j], ah[i], bh[j], acc[i][j]);
                }
        }
    }
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j)
            wmma::store_matrix_sync(sC + (wm + 16 * i) * BM_CLD + wn + 16 * j, acc[i][j], BM_CLD, wmma::mem_row_major);
    __syncthreads();
    const float alpha = alpha_ptr ? alpha_ptr[0] : 1.f;
    const bool n_fast = cn == 1;
    for (int i = threadIdx.x; i < BM_T * BM_T; i += BM_THREADS) {
        const int mm = n_fast ? i / BM_T : i % BM_T, nn = n_fast ? i % BM_T : i / BM_T;
        if (m0 + mm < M && n0 + nn < N) {
            float* dst = C + b * cb + static_cast<long long>(m0 + mm) * cm + static_cast<long long>(n0 + nn) * cn;
            const float v = alpha * sC[mm * BM_CLD + nn];
            *dst = beta ? *dst + v : v;
        }
    }
}

int launch_split(const float* src, long long R, int C, int weight, void* dst, cudaStream_t st) {
    const long long n = R * C;
    if (n <= 0) return 0;
    long long g = (n + 255) / 256;
    if (g > 132 * 16) g = 132 * 16;
    attn_split_kernel<<<static_cast<int>(g), 256, 0, st>>>(src, R, C, weight, static_cast<__half*>(dst));
    ft_count_launch(1);
    return ft_check_launch("attn_split_kernel");
}

int launch_transpose(const float* src, long long sb, long long si, int ni, int nj, float* dst, long long db, long long dj, int nb,
                     const float* scale, cudaStream_t st) {
    dim3 grid((nj + 31) / 32, (ni + 31) / 32, nb);
    attn_transpose_kernel<<<grid, 256, 0, st>>>(src, sb, si, ni, nj, dst, db, dj, scale);
    ft_count_launch(1);
    return ft_check_launch("attn_transpose_kernel");
}

int launch_bmm(int nb, int M, int N, int K, BmmOperand A, BmmOperand Bt, float* C, long long cb, long long cm, long long cn,
               const float* alpha_ptr, int beta, cudaStream_t st) {
    dim3 grid((N + BM_T - 1) / BM_T, (M + BM_T - 1) / BM_T, nb);
    TimeScope ts("attn_bmm", M, N, K, st);
    attn_bmm_kernel<<<grid, BM_THREADS, 0, st>>>(M, N, K, A, Bt, C, cb, cm, cn, alpha_ptr, beta);
    ft_count_launch(1);
    return ft_check_launch("attn_bmm_kernel");
}

struct Dims {
    long long R, RL, BTL, BA;         // BA: row pitch of the projections between consecutive t (or l)
    int T, B, L, Dq, E, A;
    explicit Dims(const FtAttentionDesc& d)
        : R(static_cast<long long>(d.T) * d.B), RL(static_cast<long long>(d.L) * d.B),
          BTL(static_cast<long long>(d.B) * d.T * d.L), BA(static_cast<long long>(d.B) * d.A), T(d.T), B(d.B), L(d.L), Dq(d.Dq),
          E(d.E), A(d.A) {}
};

// forward -> backward: the fp32 projections and, with a prior, the first softmax
struct Saved {
    float *Q, *K, *V, *p_save;
    void plan(Workspace& c, const FtAttentionDesc& d) {
        const Dims n(d);
        Q = d.attn_given ? nullptr : c.get<float>(n.R * n.A);
        K = d.attn_given ? nullptr : c.get<float>(n.RL * n.A);
        V = c.get<float>(n.RL * n.A);
        p_save = (d.has_prior && !d.attn_given) ? c.get<float>(n.BTL) : nullptr;
    }
};

struct FwdScratch {
    __half *xq, *xk, *xv, *wq, *wk, *wv, *ctx16;
    float *ctx32, *rows;
    void plan(Workspace& c, const FtAttentionDesc& d) {
        const Dims n(d);
        const bool full = !d.attn_given;
        xv = c.get<__half>(n.RL * 3 * n.E);
        wv = c.get<__half>(static_cast<size_t>(n.A) * 3 * n.E);
        xq = full ? c.get<__half>(n.R * 3 * n.Dq) : nullptr;
        xk = full ? c.get<__half>(n.RL * 3 * n.E) : nullptr;
        wq = full ? c.get<__half>(static_cast<size_t>(n.A) * 3 * n.Dq) : nullptr;
        wk = full ? c.get<__half>(static_cast<size_t>(n.A) * 3 * n.E) : nullptr;
        ctx16 = full ? c.get<__half>(n.R * n.A) : nullptr;
        ctx32 = full ? c.get<float>(n.R * n.A) : nullptr;
        rows = (full && attn_rows_in_global(n.L, n.A)) ? c.get<float>(attn_rows_floats(n.T, n.B, n.L)) : nullptr;
    }
};

struct BwdScratch {
    float *scale, *dctx, *dQ, *dK, *dV, *dv, *rows;
    __half *dQ16, *dK16, *dV16, *wq16, *wk16, *wv16, *xq16, *xk16, *xv16;
    void plan(Workspace& c, const FtAttentionDesc& d) {
        const Dims n(d);
        const bool full = !d.attn_given;
        scale = c.get<float>(8);
        dV = c.get<float>(n.RL * n.A);
        dV16 = c.get<__half>(n.RL * n.A);
        wv16 = c.get<__half>(static_cast<size_t>(n.A) * n.E);
        xv16 = c.get<__half>(n.RL * n.E);
        dctx = full ? c.get<float>(n.R * n.A) : nullptr;
        dQ = full ? c.get<float>(n.R * n.A) : nullptr;
        dK = full ? c.get<float>(n.RL * n.A) : nullptr;
        dv = full ? c.get<float>(n.A) : nullptr;
        dQ16 = full ? c.get<__half>(n.R * n.A) : nullptr;
        dK16 = full ? c.get<__half>(n.RL * n.A) : nullptr;
        wq16 = full ? c.get<__half>(static_cast<size_t>(n.A) * n.Dq) : nullptr;
        wk16 = full ? c.get<__half>(static_cast<size_t>(n.A) * n.E) : nullptr;
        xq16 = full ? c.get<__half>(n.R * n.Dq) : nullptr;
        xk16 = full ? c.get<__half>(n.RL * n.E) : nullptr;
        rows = (full && attn_rows_in_global(n.L, n.A)) ? c.get<float>(attn_rows_floats(n.T, n.B, n.L)) : nullptr;
    }
};

int check_desc(const FtAttentionDesc* d) {
    if (d->T <= 0 || d->B <= 0 || d->L <= 0 || d->Dq <= 0 || d->E <= 0 || d->A <= 0) return ft_set_error("attention: empty shape");
    if (d->L > FT_MAX_TEXT_LEN) return ft_set_error("attention: L > FT_MAX_TEXT_LEN (1024) not supported");
    if (d->B > 65535) return ft_set_error("attention: B > 65535 not supported");
    if (d->Dq % 8 || d->E % 8 || d->A % 8) return ft_set_error("attention: Dq, E and A must be multiples of 8 (GEMM operand alignment)");
    if (!(d->temperature > 0.f)) return ft_set_error("attention: temperature must be > 0");
    return 0;
}

int attention_fwd(const FtAttentionDesc& d, const FtAttentionWeights& w, const float* queries, const float* keys, const float* values,
                  const int* in_lens, const float* prior, float* output, float* attn, float* logprob, void* saved, void* scratch,
                  cudaStream_t st) {
    const Dims n(d);
    Workspace cs; cs.base = static_cast<uint8_t*>(saved);
    Saved S; S.plan(cs, d);
    Workspace cf; cf.base = static_cast<uint8_t*>(scratch);
    FwdScratch F; F.plan(cf, d);

    FT_TRY(launch_split(w.value, n.A, n.E, 1, F.wv, st));
    FT_TRY(launch_split(values, n.RL, n.E, 0, F.xv, st));
    FT_TRY(gemm_nt(st, n.RL, n.A, 3 * n.E, F.xv, 3 * n.E, F.wv, 3 * n.E, S.V, n.A));
    if (d.attn_given) {
        // output(b, a, t) = sum_l V(l*B + b, a) attn(b, t, l)
        const BmmOperand Av{S.V, n.A, 1, n.BA};
        const BmmOperand Bp{attn, static_cast<long long>(n.T) * n.L, n.L, 1};
        return launch_bmm(n.B, n.A, n.T, n.L, Av, Bp, output, static_cast<long long>(n.A) * n.T, n.T, 1, nullptr, 0, st);
    }
    FT_TRY(launch_split(w.query, n.A, n.Dq, 1, F.wq, st));
    FT_TRY(launch_split(w.key, n.A, n.E, 1, F.wk, st));
    FT_TRY(launch_split(queries, n.R, n.Dq, 0, F.xq, st));
    FT_TRY(launch_split(keys, n.RL, n.E, 0, F.xk, st));
    FT_TRY(gemm_nt(st, n.R, n.A, 3 * n.Dq, F.xq, 3 * n.Dq, F.wq, 3 * n.Dq, S.Q, n.A));
    FT_TRY(gemm_nt(st, n.RL, n.A, 3 * n.E, F.xk, 3 * n.E, F.wk, 3 * n.E, S.K, n.A));
    AttnFwdArgs a;
    a.T = n.T; a.B = n.B; a.L = n.L; a.A = n.A;
    a.Q = S.Q; a.ldq = n.A; a.K = S.K; a.ldk = n.A; a.V = S.V; a.ldv = n.A; a.v = w.v;
    a.in_lens = in_lens; a.out_lens = nullptr; a.prior = d.has_prior ? prior : nullptr; a.reversed = 0;
    a.temperature = d.temperature; a.attn = attn; a.logprob = logprob; a.p_save = S.p_save;
    a.ctx16 = F.ctx16; a.ldc = n.A; a.ctx32 = F.ctx32; a.ldc32 = n.A;
    a.rows = F.rows;
    FT_TRY(launch_attn_fwd(a, st));
    // ctx rows (t*B + b, a) -> output [B, A, T]
    return launch_transpose(F.ctx32, n.A, n.BA, n.T, n.A, output, static_cast<long long>(n.A) * n.T, n.T, n.B, nullptr, st);
}

int attention_bwd(const FtAttentionDesc& d, const FtAttentionWeights& w, const float* queries, const float* keys, const float* values,
                  const int* in_lens, const float* attn, const float* d_output, const float* d_attn, const float* d_logprob,
                  float* d_queries, float* d_keys, float* d_values, float* d_attn_given, const FtAttentionGrads& g, void* saved,
                  void* scratch, cudaStream_t st) {
    const Dims n(d);
    Workspace cs; cs.base = static_cast<uint8_t*>(saved);
    Saved S; S.plan(cs, d);
    Workspace cb; cb.base = static_cast<uint8_t*>(scratch);
    BwdScratch F; F.plan(cb, d);
    const bool need_v = d_values || g.value;
    const long long BAT = static_cast<long long>(n.B) * n.A * n.T;
    const float* iS = F.scale + 1;

    if (d.attn_given) {
        if (d_logprob) return ft_set_error("ft_attention_bwd: attn was given, so there is no attn_logprob to take a gradient of");
        // both products below stage S * d_output (max ~ 64), never d_output itself, as fp16 hi / lo
        if (d_output) FT_TRY(launch_grad_scale(d_output, BAT, nullptr, 0, nullptr, 0, 64.f, F.scale, st));
        if (d_attn_given) {
            // d attn(b, t, l) = d_attn(b, t, l) + sum_a d_output(b, a, t) V(l*B + b, a)
            int beta = 0;
            if (d_attn) {
                FT_CU(cudaMemcpyAsync(d_attn_given, d_attn, sizeof(float) * n.BTL, cudaMemcpyDeviceToDevice, st), "ft_attention_bwd");
                beta = 1;
            }
            if (d_output) {
                const BmmOperand Ad{d_output, static_cast<long long>(n.A) * n.T, 1, n.T, F.scale};
                const BmmOperand Bv{S.V, n.A, n.BA, 1};
                FT_TRY(launch_bmm(n.B, n.T, n.L, n.A, Ad, Bv, d_attn_given, static_cast<long long>(n.T) * n.L, n.L, 1, iS, beta, st));
            } else if (!d_attn) {
                FT_CU(cudaMemsetAsync(d_attn_given, 0, sizeof(float) * n.BTL, st), "attention");
            }
        }
        if (!need_v) return 0;
        if (!d_output) {
            if (d_values) FT_CU(cudaMemsetAsync(d_values, 0, sizeof(float) * n.RL * n.E, st), "attention");
            if (g.value) FT_CU(cudaMemsetAsync(g.value, 0, sizeof(float) * n.A * n.E, st), "attention");
            return 0;
        }
        // dV(l*B + b, a) = sum_t attn(b, t, l) S d_output(b, a, t): in the scaled domain, like the attention kernel's dV
        const BmmOperand Aa{attn, static_cast<long long>(n.T) * n.L, 1, n.L};
        const BmmOperand Bd{d_output, static_cast<long long>(n.A) * n.T, n.T, 1, F.scale};
        FT_TRY(launch_bmm(n.B, n.L, n.A, n.T, Aa, Bd, F.dV, n.A, n.BA, 1, nullptr, 0, st));
    } else {
        const bool need_q = d_queries || g.query, need_k = d_keys || g.key;
        if (!(need_q || need_k || need_v || g.v)) return 0;
        FT_TRY(launch_grad_scale(d_output, d_output ? BAT : 0, nullptr, 0, nullptr, 0, 64.f, F.scale, st,
                                 d_attn, d_attn ? n.BTL : 0, d_logprob, d_logprob ? n.BTL : 0));
        if (d_output) FT_TRY(launch_transpose(d_output, static_cast<long long>(n.A) * n.T, n.T, n.A, n.T, F.dctx, n.A,
                                              n.BA, n.B, F.scale, st));
        else FT_CU(cudaMemsetAsync(F.dctx, 0, sizeof(float) * n.R * n.A, st), "attention");
        FT_CU(cudaMemsetAsync(F.dK, 0, sizeof(float) * n.RL * n.A, st), "attention");
        FT_CU(cudaMemsetAsync(F.dV, 0, sizeof(float) * n.RL * n.A, st), "attention");
        float* dv = g.v ? g.v : F.dv;
        FT_CU(cudaMemsetAsync(dv, 0, sizeof(float) * n.A, st), "attention");
        AttnBwdArgs a;
        a.T = n.T; a.B = n.B; a.L = n.L; a.A = n.A;
        a.Q = S.Q; a.ldq = n.A; a.K = S.K; a.ldk = n.A; a.V = S.V; a.ldv = n.A; a.v = w.v;
        a.in_lens = in_lens; a.out_lens = nullptr; a.attn = attn; a.p_save = S.p_save; a.temperature = d.temperature;
        a.dctx = F.dctx; a.lddc = n.A; a.dattn_ext = d_attn; a.dlp_ext = d_logprob; a.scale = F.scale;
        a.dQ = F.dQ; a.lddq = n.A; a.dK = F.dK; a.lddk = n.A; a.dV = F.dV; a.lddv = n.A; a.dv = dv;
        a.rows = F.rows;
        FT_TRY(launch_attn_bwd(a, st));
        if (need_q) {
            FT_TRY(launch_cast(F.dQ, 2, F.dQ16, 0, n.R * n.A, st));
            if (d_queries) {
                FT_TRY(launch_cast(w.query, 2, F.wq16, 0, static_cast<long long>(n.A) * n.Dq, st));
                FT_TRY(gemm_dgrad(st, n.R, n.Dq, n.A, F.dQ16, n.A, F.wq16, n.Dq, d_queries, n.Dq, nullptr, 0, 0, iS));
            }
            if (g.query) {
                FT_TRY(launch_cast(queries, 2, F.xq16, 0, n.R * n.Dq, st));
                FT_TRY(gemm_wgrad(st, n.A, n.Dq, n.R, F.dQ16, n.A, F.xq16, n.Dq, g.query, n.Dq, iS));
            }
        }
        if (need_k) {
            FT_TRY(launch_cast(F.dK, 2, F.dK16, 0, n.RL * n.A, st));
            if (d_keys) {
                FT_TRY(launch_cast(w.key, 2, F.wk16, 0, static_cast<long long>(n.A) * n.E, st));
                FT_TRY(gemm_dgrad(st, n.RL, n.E, n.A, F.dK16, n.A, F.wk16, n.E, d_keys, n.E, nullptr, 0, 0, iS));
            }
            if (g.key) {
                FT_TRY(launch_cast(keys, 2, F.xk16, 0, n.RL * n.E, st));
                FT_TRY(gemm_wgrad(st, n.A, n.E, n.RL, F.dK16, n.A, F.xk16, n.E, g.key, n.E, iS));
            }
        }
        if (!need_v) return 0;
    }
    // value projection, both branches
    FT_TRY(launch_cast(F.dV, 2, F.dV16, 0, n.RL * n.A, st));
    if (d_values) {
        FT_TRY(launch_cast(w.value, 2, F.wv16, 0, static_cast<long long>(n.A) * n.E, st));
        FT_TRY(gemm_dgrad(st, n.RL, n.E, n.A, F.dV16, n.A, F.wv16, n.E, d_values, n.E, nullptr, 0, 0, iS));
    }
    if (g.value) {
        FT_TRY(launch_cast(values, 2, F.xv16, 0, n.RL * n.E, st));
        FT_TRY(gemm_wgrad(st, n.A, n.E, n.RL, F.dV16, n.A, F.xv16, n.E, g.value, n.E, iS));
    }
    return 0;
}

}  // namespace
}  // namespace ft

// =================================================================================================== C ABI
extern "C" {

size_t ft_attention_saved_bytes(const FtAttentionDesc* d) {
    if (!d || ft::check_desc(d)) return 0;
    ft::Workspace c; ft::Saved s; s.plan(c, *d);
    return c.off + 256;
}

size_t ft_attention_scratch_bytes(const FtAttentionDesc* d) {
    if (!d || ft::check_desc(d)) return 0;
    ft::Workspace cf; ft::FwdScratch f; f.plan(cf, *d);
    ft::Workspace cb; ft::BwdScratch b; b.plan(cb, *d);
    return (cf.off > cb.off ? cf.off : cb.off) + 256;
}

int ft_attention_fwd(const FtAttentionDesc* d, const FtAttentionWeights* w, const float* queries, const float* keys,
                     const float* values, const int* in_lens, const float* attn_prior, float* output, float* attn,
                     float* attn_logprob, void* saved, void* scratch, void* stream) {
    if (!d || !w || !values || !w->value || !output || !attn || !saved || !scratch) return ft::ft_set_error("ft_attention_fwd: NULL argument");
    if (ft::check_desc(d)) return -1;
    if (!d->attn_given) {
        if (!queries || !keys || !w->query || !w->key || !w->v || !attn_logprob) return ft::ft_set_error("ft_attention_fwd: NULL argument");
        if (d->has_prior && !attn_prior) return ft::ft_set_error("ft_attention_fwd: has_prior set but attn_prior is NULL");
    }
    return ft::attention_fwd(*d, *w, queries, keys, values, in_lens, attn_prior, output, attn, attn_logprob, saved, scratch,
                             static_cast<cudaStream_t>(stream));
}

int ft_attention_bwd(const FtAttentionDesc* d, const FtAttentionWeights* w, const float* queries, const float* keys,
                     const float* values, const int* in_lens, const float* attn, const float* d_output, const float* d_attn,
                     const float* d_attn_logprob, float* d_queries, float* d_keys, float* d_values, float* d_attn_given,
                     const FtAttentionGrads* g, void* saved, void* scratch, void* stream) {
    if (!d || !w || !g || !attn || !saved || !scratch) return ft::ft_set_error("ft_attention_bwd: NULL argument");
    if (ft::check_desc(d)) return -1;
    if ((d_queries || g->query) && (!queries || !w->query)) return ft::ft_set_error("ft_attention_bwd: query gradients need queries and the query weight");
    if ((d_keys || g->key) && (!keys || !w->key)) return ft::ft_set_error("ft_attention_bwd: key gradients need keys and the key weight");
    if ((d_values || g->value) && (!values || !w->value)) return ft::ft_set_error("ft_attention_bwd: value gradients need values and the value weight");
    if (!d->attn_given && d_attn_given) return ft::ft_set_error("ft_attention_bwd: d_attn_given needs attn_given");
    if (!d->attn_given && !w->v) return ft::ft_set_error("ft_attention_bwd: NULL argument");
    return ft::attention_bwd(*d, *w, queries, keys, values, in_lens, attn, d_output, d_attn, d_attn_logprob, d_queries, d_keys,
                             d_values, d_attn_given, *g, saved, scratch, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
