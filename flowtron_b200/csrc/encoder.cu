// Text Encoder (flowtron.py:467-525) as kernels: 3 x [conv k=5 -> MaskedInstanceNorm1d (affine) -> relu -> dropout], then a
// packed bidirectional LSTM (hidden 256 per direction), forward and backward.  Replaces the torch/cuDNN module of rounds 1-2
// (~700 latency-bound launches per step: cutlass tf32 implicit GEMMs, per-time-step cuDNN cells).
//
// Layout: every activation lives channels-last in ONE padded token grid  row(b, l) = b * (L + 4) + 2 + l  with two zero rows
// on either side of an utterance, so
//   * the k = 5 convolution is 5 accumulating wgmma GEMMs whose A operand is the SAME buffer shifted by k rows (no im2col,
//     no cuDNN layout transposes); its dgrad / wgrad are the same trick on the gradient grid;
//   * the recurrence's h_{t-1} / h_{t+1} of the first / last token of an utterance is a zero pad row: no special cases.
// The BiLSTM recurrences run as TWO CLUSTERS OF 8 CTAs (one per direction) in one launch: CTA r owns 32 hidden units, keeps
// its 128 x 256 slice of W_hh in REGISTERS as mma.sync B fragments (no shared-memory weight reads in the loop), exchanges h_t
// through global memory (the [rows, 256] fp16 tensor the weight-gradient GEMM needs anyway) and synchronises the 8 CTAs with
// one cluster barrier per step.  Packed-sequence semantics without packing: a token at l >= in_lens[b] gets h = c = 0, which
// is exactly the zero state the reverse direction must start from at the utterance's last token.
// The backward recurrence is the mirror image: W_hh^T slices in registers, dG_t exchanged through the [rows, 1024] fp16
// tensor the weight gradients are GEMMs over, fp32 cell-gradient carry in registers.
// Precision: SPLIT fp16.  Plain fp16 operands (the flows' choice) measured 1.2-1.5e-3 on the encoder output and 3-5 % on the
// encoder's small parameter gradients -- over the 1e-3 / 1e-2 bars, and the encoder feeds both flows.  So every
// tensor-core operand x is stored as hi = fp16(x), lo = fp16(x - hi) (22 significant bits) and every product is
// hi*hi + lo*hi + hi*lo with fp32 accumulation.  For K-major operands that is ONE GEMM over a 3x longer contraction: activations
// and gradients are stored as rows [hi | lo | hi], weights as [hi | hi | lo] (or row-stacked [hi ; hi ; lo] when the weight is
// the MN-major operand of a dgrad); weight gradients (contraction over rows) are three GEMMs over column views of the same
// buffers.  The recurrences issue three mma.sync per tile with W_hh's hi and lo fragments both resident in registers.  The
// encoder is < 1 % of the step's FLOPs, so 3x of it is free; the backward pass additionally runs on S * grad with a power-of-two
// S picked on the device from max|d_out| and multiplies everything leaving the encoder by 1/S.
#include "encoder_kernels.cuh"
#include "../../include/flowtron_b200.h"

namespace ft {


// ------------------------------------------------------------------------------------------------ layout kernels
// x [B, C, L] fp32 (embedding output, channels first) -> grid rows (split fp16 [hi|lo|hi], channels last); tokens at l >= len are zeroed
// (flowtron.py:501 masked_fill_).  32 x 32 tiles through shared memory.
__global__ void enc_in_kernel(const float* __restrict__ x, const int* __restrict__ lens, int B, int L, __half* __restrict__ X16) {
    __shared__ float tile[32][33];
    const int b = blockIdx.z, l0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;                    // 256 threads: 8 rows per pass
    const int len = lens ? lens[b] : L;
    for (int i = ty; i < 32; i += 8) {
        const int l = l0 + tx;
        tile[i][tx] = (l < L) ? x[(static_cast<long long>(b) * EC + c0 + i) * L + l] : 0.f;
    }
    __syncthreads();
    for (int i = ty; i < 32; i += 8) {
        const int l = l0 + i;
        if (l < L) store_hlh(X16 + (static_cast<long long>(b) * (L + 2 * EPADR) + EPADR + l) * (3 * EC), EC, c0 + tx, l < len ? tile[tx][i] : 0.f);
    }
}

// Token path (the reference's `self.embedding(text)` in front of the encoder, flowtron.py:873): the embedding row gather writes the
// first block's input grid directly (no [B, L, 512] tensor, no transposes) ...
__global__ void enc_embed_kernel(const long long* __restrict__ tokens, const float* __restrict__ emb, int n_text, const int* __restrict__ lens,
                                 int B, int L, __half* __restrict__ X16) {
    const int row = blockIdx.x, b = row / L, l = row - b * L;            // one CTA per token, 128 threads x 4 channels
    const int len = lens ? lens[b] : L;
    long long tok = tokens[row];
    tok = tok < 0 ? 0 : (tok >= n_text ? n_text - 1 : tok);
    __half* dst = X16 + (static_cast<long long>(b) * (L + 2 * EPADR) + EPADR + l) * (3 * EC);
    for (int c = threadIdx.x; c < EC; c += blockDim.x) store_hlh(dst, EC, c, l < len ? emb[tok * EC + c] : 0.f);
}
// ... and its backward scatters the (loss-scaled) input-grid gradient into embedding.weight.grad (zeroed by the caller)
__global__ void enc_embed_grad_kernel(const float* __restrict__ DX, const long long* __restrict__ tokens, int n_text, const int* __restrict__ lens,
                                      int B, int L, const float* __restrict__ scale2, float* __restrict__ d_emb) {
    const int row = blockIdx.x, b = row / L, l = row - b * L;
    const int len = lens ? lens[b] : L;
    if (l >= len) return;
    long long tok = tokens[row];
    tok = tok < 0 ? 0 : (tok >= n_text ? n_text - 1 : tok);
    const float inv = scale2[1];
    const float* src = DX + (static_cast<long long>(b) * (L + 2 * EPADR) + EPADR + l) * EC;
    for (int c = threadIdx.x; c < EC; c += blockDim.x) atomicAdd(d_emb + tok * EC + c, src[c] * inv);
}

// gradient grid rows (fp32, channels last, loss-scaled) -> d_x [B, C, L] fp32 (x 1/S); zero at l >= len
__global__ void enc_out_grad_kernel(const float* __restrict__ DX, const int* __restrict__ lens, int B, int L, const float* __restrict__ scale2,
                                    float* __restrict__ dx) {
    __shared__ float tile[32][33];
    const int b = blockIdx.z, l0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int len = lens ? lens[b] : L;
    const float inv = scale2[1];
    for (int i = ty; i < 32; i += 8) {
        const int l = l0 + i;
        tile[i][tx] = (l < len) ? DX[(static_cast<long long>(b) * (L + 2 * EPADR) + EPADR + l) * EC + c0 + tx] * inv : 0.f;
    }
    __syncthreads();
    for (int i = ty; i < 32; i += 8) {
        const int l = l0 + tx;
        if (l < L) dx[(static_cast<long long>(b) * EC + c0 + i) * L + l] = tile[tx][i];
    }
}

// conv.weight [co, ci, k] fp32 -> per tap k, split fp16:
//   kmajor  [k][co][3 C] = [hi | hi | lo]   (B operand of the forward GEMM, contraction over ci)
//   stacked [k][3 C (hi ; hi ; lo rows of co)][ci]   (MN-major B operand of the dgrad GEMM, contraction over co)
__global__ void enc_pack_conv_kernel(const float* __restrict__ w, __half* __restrict__ kmajor, __half* __restrict__ stacked) {
    const long long n = static_cast<long long>(EK) * EC * EC;
    for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int ci = static_cast<int>(i % EC), co = static_cast<int>((i / EC) % EC), k = static_cast<int>(i / (EC * EC));
        __half hi, lo;
        split16(w[(static_cast<long long>(co) * EC + ci) * EK + k], hi, lo);
        if (kmajor) {
            __half* r = kmajor + (static_cast<long long>(k) * EC + co) * (3 * EC);
            r[ci] = hi; r[EC + ci] = hi; r[2 * EC + ci] = lo;
        }
        if (stacked) {
            __half* t = stacked + static_cast<long long>(k) * 3 * EC * EC;
            t[static_cast<long long>(co) * EC + ci] = hi; t[static_cast<long long>(EC + co) * EC + ci] = hi; t[static_cast<long long>(2 * EC + co) * EC + ci] = lo;
        }
    }
}
// W_ih [1024, 512] fp32 -> kmajor [1024][3 C] = [hi | hi | lo] and / or stacked [3 x 1024 (hi ; hi ; lo)][512]
__global__ void enc_pack_wih_kernel(const float* __restrict__ w, __half* __restrict__ kmajor, __half* __restrict__ stacked) {
    const long long n = static_cast<long long>(EG) * EC;
    for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int c = static_cast<int>(i % EC), r = static_cast<int>(i / EC);
        __half hi, lo;
        split16(w[i], hi, lo);
        if (kmajor) { __half* q = kmajor + static_cast<long long>(r) * (3 * EC); q[c] = hi; q[EC + c] = hi; q[2 * EC + c] = lo; }
        if (stacked) { stacked[i] = hi; stacked[n + i] = hi; stacked[2 * n + i] = lo; }
    }
}
// out[c] = scale * sum_r (hi[r, c] + lo[r, c]) over a split grid [R, 3 W]
__global__ void enc_colsum_hilo_kernel(const __half* __restrict__ src, long long R, int W, const float* __restrict__ scale, float* __restrict__ out) {
    __shared__ float sm[8][33];
    const int c = blockIdx.x * 32 + (threadIdx.x & 31), ty = threadIdx.x >> 5;
    float s = 0.f;
    for (long long r = ty; r < R; r += 8) s += __half2float(src[r * (3 * W) + c]) + __half2float(src[r * (3 * W) + W + c]);
    sm[ty][threadIdx.x & 31] = s;
    __syncthreads();
    if (ty == 0) {
        float t = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) t += sm[i][threadIdx.x & 31];
        out[c] = t * scale[0];
    }
}
// dW [k][co][ci] fp32 -> conv.weight.grad [co, ci, k]
__global__ void enc_unpack_conv_grad_kernel(const float* __restrict__ dwk, float* __restrict__ dw) {
    const long long n = static_cast<long long>(EK) * EC * EC;
    for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int k = static_cast<int>(i % EK), ci = static_cast<int>((i / EK) % EC), co = static_cast<int>(i / (EK * EC));
        dw[i] = dwk[(static_cast<long long>(k) * EC + co) * EC + ci];
    }
}

// ------------------------------------------------------------------------------------------------ instance norm + relu + dropout
__device__ __forceinline__ uint32_t hash3(uint64_t seed, uint64_t ctr, uint64_t idx) {     // splitmix64 finaliser over (seed, counter, element)
    uint64_t z = seed + 0x9E3779B97F4A7C15ull * (ctr + 1) + idx * 0xD1B54A32D192ED03ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return static_cast<uint32_t>((z ^ (z >> 31)) >> 32);
}

// MaskedInstanceNorm1d (flowtron.py:53-92; use_input_stats, biased variance over the utterance's own tokens) + affine + relu +
// dropout (flowtron.py:502).  CTA = (utterance, 32 channels); lane = channel, 8 token lanes.  Y: conv output (fp32 grid),
// out: next layer's input (fp16 grid; rows at l >= len stay zero).  mean / rstd [B, C] saved for the backward pass.
__global__ void __launch_bounds__(256)
enc_norm_fwd_kernel(const float* __restrict__ Y, const int* __restrict__ lens, int L, const float* __restrict__ w, const float* __restrict__ bias,
                    float eps, float drop_p, const unsigned long long* __restrict__ rng, int layer, __half* __restrict__ out,
                    float* __restrict__ mean_out, float* __restrict__ rstd_out) {
    __shared__ float red[8][33];
    const int b = blockIdx.x, c = blockIdx.y * 32 + (threadIdx.x & 31), tl = threadIdx.x >> 5;
    const int n = lens ? lens[b] : L;
    const long long r0 = static_cast<long long>(b) * (L + 2 * EPADR) + EPADR;
    float s = 0.f;
    for (int l = tl; l < n; l += 8) s += Y[(r0 + l) * EC + c];
    red[tl][threadIdx.x & 31] = s;
    __syncthreads();
    float mean = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) mean += red[i][threadIdx.x & 31];
    mean /= static_cast<float>(n);
    __syncthreads();
    float v = 0.f;
    for (int l = tl; l < n; l += 8) { const float d = Y[(r0 + l) * EC + c] - mean; v = fmaf(d, d, v); }
    red[tl][threadIdx.x & 31] = v;
    __syncthreads();
    float var = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) var += red[i][threadIdx.x & 31];
    const float rstd = 1.0f / sqrtf(var / static_cast<float>(n) + eps);
    if (tl == 0) { mean_out[b * EC + c] = mean; rstd_out[b * EC + c] = rstd; }
    const float g = w[c] * rstd, bb = bias[c];
    const float keep_scale = drop_p > 0.f ? 1.0f / (1.0f - drop_p) : 1.0f;
    const uint32_t thr = drop_p > 0.f ? static_cast<uint32_t>(drop_p * 4294967296.0) : 0u;
    const unsigned long long seed = rng ? rng[0] : 0ull, ctr = rng ? rng[1] * 4 + layer : 0ull;
    for (int l = tl; l < n; l += 8) {
        float y = fmaxf(fmaf(Y[(r0 + l) * EC + c] - mean, g, bb), 0.f);
        if (drop_p > 0.f) y = (hash3(seed, ctr, static_cast<uint64_t>(r0 + l) * EC + c) >= thr) ? y * keep_scale : 0.f;
        store_hlh(out + (r0 + l) * (3 * EC), EC, c, y);
    }
}

// Backward of the block above.  DX: (loss-scaled) gradient w.r.t. the block's output (fp32 grid); xout: the block's fp16 output
// (> 0 <=> relu passed AND the unit was kept); writes dY (fp16 grid, zero outside the utterance) and adds the affine gradients
// (x 1/S) into dw / db [C] with one atomic per (utterance, channel).
__global__ void __launch_bounds__(256)
enc_norm_bwd_kernel(const float* __restrict__ DX, const __half* __restrict__ xout, const float* __restrict__ Y, const int* __restrict__ lens, int L,
                    const float* __restrict__ w, const float* __restrict__ mean_in, const float* __restrict__ rstd_in, float drop_p,
                    const float* __restrict__ scale2, __half* __restrict__ dY, float* __restrict__ dw, float* __restrict__ db) {
    __shared__ float red[2][8][33];
    const int b = blockIdx.x, c = blockIdx.y * 32 + (threadIdx.x & 31), tl = threadIdx.x >> 5, lc = threadIdx.x & 31;
    const int n = lens ? lens[b] : L;
    const long long r0 = static_cast<long long>(b) * (L + 2 * EPADR) + EPADR;
    const float mean = mean_in[b * EC + c], rstd = rstd_in[b * EC + c];
    const float keep_scale = drop_p > 0.f ? 1.0f / (1.0f - drop_p) : 1.0f;
    float s1 = 0.f, s2 = 0.f;                      // sum g, sum g * xhat
    for (int l = tl; l < n; l += 8) {
        const long long o = (r0 + l) * EC + c;
        const float g = __half2float(xout[(r0 + l) * (3 * EC) + c]) > 0.f ? DX[o] * keep_scale : 0.f;
        s1 += g;
        s2 = fmaf(g, (Y[o] - mean) * rstd, s2);
    }
    red[0][tl][lc] = s1; red[1][tl][lc] = s2;
    __syncthreads();
    float t1 = 0.f, t2 = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) { t1 += red[0][i][lc]; t2 += red[1][i][lc]; }
    if (tl == 0) { atomicAdd(db + c, t1 * scale2[1]); atomicAdd(dw + c, t2 * scale2[1]); }
    const float wc = w[c], m1 = t1 / static_cast<float>(n), m2 = t2 / static_cast<float>(n);
    for (int l = tl; l < n; l += 8) {
        const long long o = (r0 + l) * EC + c;
        const float g = __half2float(xout[(r0 + l) * (3 * EC) + c]) > 0.f ? DX[o] * keep_scale : 0.f;
        const float xh = (Y[o] - mean) * rstd;
        store_hlh(dY + (r0 + l) * (3 * EC), EC, c, rstd * wc * (g - m1 - xh * m2));
    }
}

__global__ void enc_rng_advance_kernel(unsigned long long* rng) { rng[1] += 1; }

// ------------------------------------------------------------------------------------------------ BiLSTM forward

// grid = 16 CTAs per 32 utterances = clusters of 8; cluster id = (batch half, direction), rank r owns hidden units [32 r, 32 r + 32).
// Warp w: units u0 = 32 r + 4 w .. +3; its two n8 tiles hold gate rows (i,f) and (g,o) of the 4 units interleaved
// [g0(u0), g1(u0), g0(u1), g1(u1), ...], so accumulator columns 2j, 2j+1 of lane j = lane % 4 are the two gates of ITS unit u0 + j
// and the whole cell update of (unit, batch row) happens in one thread without shuffles.
template <int MT>                                   // m16 tiles of batch rows per cluster (<= 32 utterances)
__global__ void __cluster_dims__(ENC_CLUSTER, 1, 1) __launch_bounds__(ENC_THREADS, 1)
enc_bilstm_fwd_kernel(EncLstmFwdParams p) {
    constexpr int HP = EH + 8;                                   // shared row pitch (halfs): conflict-free fragment loads
    __shared__ __align__(16) __half sh[2][MT * 16 * HP];         // h_{t-1}: hi, lo
    const int cid = blockIdx.x / ENC_CLUSTER, dir = cid & 1, b0 = 32 * (cid >> 1), rank = static_cast<int>(cluster_ctarank());
    const int nB = min(p.B - b0, 32);                            // utterances of this cluster
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, j = lane & 3, g = lane >> 2;
    const int Lp = p.L + 2 * EPADR;
    const int unit = ENC_UNITS * rank + 4 * warp + j;            // the unit this lane's accumulator columns belong to
    __half* const hseq = dir ? p.hseq[1] : p.hseq[0];            // (no dynamically indexed parameter arrays: they would live in local memory)
    __half* const gates = dir ? p.gates[1] : p.gates[0];
    float* const cstate = dir ? p.cstate[1] : p.cstate[0];
    // W_hh B fragments (hi and lo): tile T (0: i,f; 1: g,o), column n = lane / 4 -> gate 2T + (n & 1) of unit u0 + n / 2
    uint32_t wh[2][16][2], wl[2][16][2];
    {
        const float* W = dir ? p.whh[1] : p.whh[0];
#pragma unroll
        for (int T = 0; T < 2; ++T) {
            const int row = (2 * T + (g & 1)) * EH + ENC_UNITS * rank + 4 * warp + (g >> 1);
#pragma unroll
            for (int ks = 0; ks < 16; ++ks) {
#pragma unroll
                for (int q = 0; q < 2; ++q) {
                    const float2 v = *reinterpret_cast<const float2*>(W + static_cast<long long>(row) * EH + 16 * ks + 8 * q + 2 * j);
                    __half h0, l0, h1, l1;
                    split16(v.x, h0, l0); split16(v.y, h1, l1);
                    wh[T][ks][q] = static_cast<uint32_t>(__half_as_ushort(h0)) | (static_cast<uint32_t>(__half_as_ushort(h1)) << 16);
                    wl[T][ks][q] = static_cast<uint32_t>(__half_as_ushort(l0)) | (static_cast<uint32_t>(__half_as_ushort(l1)) << 16);
                }
            }
        }
    }
    for (int i = threadIdx.x; i < 2 * MT * 16 * HP; i += ENC_THREADS) (&sh[0][0])[i] = __float2half_rn(0.f);
    float c[MT][2];
    int len[MT][2];
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            c[mt][hh] = 0.f;
            const int bl = 16 * mt + 8 * hh + g;
            len[mt][hh] = bl < nB ? (p.lens ? p.lens[b0 + bl] : p.L) : 0;
        }
    __syncthreads();
    for (int s = 0; s < p.L; ++s) {
        const int t = dir == 0 ? s : p.L - 1 - s, tp = dir == 0 ? t - 1 : t + 1;
        // input projection of this lane's (unit, batch rows): independent of the recurrence, issued first
        float xp[MT][2][4];
#pragma unroll
        for (int mt = 0; mt < MT; ++mt)
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
                const int bl = 16 * mt + 8 * hh + g;
                if (bl < nB) {
                    const float* src = p.xproj + (static_cast<long long>(b0 + bl) * Lp + EPADR + t) * (2 * EG) + dir * EG + unit;
#pragma unroll
                    for (int q = 0; q < 4; ++q) xp[mt][hh][q] = __ldg(src + q * EH);
                } else {
#pragma unroll
                    for (int q = 0; q < 4; ++q) xp[mt][hh][q] = 0.f;
                }
            }
        // h of the previous step, hi and lo (all 256 units, written by the 8 CTAs of this cluster; pad rows = zero initial state)
        for (int idx = threadIdx.x; idx < nB * (2 * EH / 8); idx += ENC_THREADS) {
            const int bl = idx / (2 * EH / 8), i8 = idx - bl * (2 * EH / 8);          // i8 < 32: hi, else lo
            const uint4 v = ldcg_v4(hseq + (static_cast<long long>(b0 + bl) * Lp + EPADR + tp) * (2 * EH) + 8 * i8);
            *reinterpret_cast<uint4*>(&sh[i8 >> 5][bl * HP + 8 * (i8 & 31)]) = v;
        }
        __syncthreads();
        float acc[MT][2][4];
#pragma unroll
        for (int mt = 0; mt < MT; ++mt)
#pragma unroll
            for (int T = 0; T < 2; ++T)
#pragma unroll
                for (int q = 0; q < 4; ++q) acc[mt][T][q] = 0.f;
#pragma unroll
        for (int ks = 0; ks < 16; ++ks) {
#pragma unroll
            for (int mt = 0; mt < MT; ++mt) {
                const int o = (16 * mt + g) * HP + 16 * ks + 2 * j;
                const uint32_t a0 = *reinterpret_cast<const uint32_t*>(&sh[0][o]), a1 = *reinterpret_cast<const uint32_t*>(&sh[0][o + 8 * HP]);
                const uint32_t a2 = *reinterpret_cast<const uint32_t*>(&sh[0][o + 8]), a3 = *reinterpret_cast<const uint32_t*>(&sh[0][o + 8 * HP + 8]);
                const uint32_t l0 = *reinterpret_cast<const uint32_t*>(&sh[1][o]), l1 = *reinterpret_cast<const uint32_t*>(&sh[1][o + 8 * HP]);
                const uint32_t l2 = *reinterpret_cast<const uint32_t*>(&sh[1][o + 8]), l3 = *reinterpret_cast<const uint32_t*>(&sh[1][o + 8 * HP + 8]);
#pragma unroll
                for (int T = 0; T < 2; ++T) {
                    mma16816(acc[mt][T], a0, a1, a2, a3, wh[T][ks][0], wh[T][ks][1]);    // hi * hi
                    mma16816(acc[mt][T], l0, l1, l2, l3, wh[T][ks][0], wh[T][ks][1]);    // lo * hi
                    mma16816(acc[mt][T], a0, a1, a2, a3, wl[T][ks][0], wl[T][ks][1]);    // hi * lo
                }
            }
        }
#pragma unroll
        for (int mt = 0; mt < MT; ++mt)
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
                const int bl = 16 * mt + 8 * hh + g;
                if (bl < nB) {
                    const int b = b0 + bl;
                    const bool valid = t < len[mt][hh];
                    const float gi = sigmoid_f(acc[mt][0][2 * hh] + xp[mt][hh][0]), gf = sigmoid_f(acc[mt][0][2 * hh + 1] + xp[mt][hh][1]);
                    const float gg = tanh_f(acc[mt][1][2 * hh] + xp[mt][hh][2]), go = sigmoid_f(acc[mt][1][2 * hh + 1] + xp[mt][hh][3]);
                    const float cn = valid ? gf * c[mt][hh] + gi * gg : 0.f;
                    const float h = valid ? go * tanh_f(cn) : 0.f;
                    c[mt][hh] = cn;
                    const long long r = static_cast<long long>(b) * Lp + EPADR + t;
                    __half hi, lo;
                    split16(h, hi, lo);
                    hseq[r * (2 * EH) + unit] = hi; hseq[r * (2 * EH) + EH + unit] = lo;
                    p.out[b * p.out_sb + t * p.out_sl + dir * EH + unit] = h;
                    if (gates) {
                        __half* gp = gates + r * EG + unit;
                        gp[0] = __float2half_rn(gi); gp[EH] = __float2half_rn(gf); gp[2 * EH] = __float2half_rn(gg); gp[3 * EH] = __float2half_rn(go);
                    }
                    if (cstate) cstate[r * EH + unit] = cn;
                }
            }
        cluster_sync_all();                                      // h_t of all 8 CTAs visible before anyone stages it (also orders sh reuse)
    }
}

// ------------------------------------------------------------------------------------------------ BiLSTM backward

// Mirror of the forward kernel: cluster = (batch half, direction), rank r owns units [32 r, 32 r + 32); per step
//   dh_rec[b, u] = sum over the 1024 gate rows k of dG_next[b, k] W_hh[k, u]
// with warp w reducing over k in [128 w, 128 w + 128) for all 32 units (W_hh^T slice, hi and lo, in registers), partial sums
// meeting in shared memory, then the pointwise LSTM backward of (batch row, unit) pairs with the cell-gradient carry in registers.
template <int MT>
__global__ void __cluster_dims__(ENC_CLUSTER, 1, 1) __launch_bounds__(ENC_THREADS, 1)
enc_bilstm_bwd_kernel(EncLstmBwdParams p) {
    constexpr int GP = EG + 8;                                   // staged dG row pitch (halfs)
    constexpr int PP = ENC_UNITS + 1;                            // partial-sum row pitch (floats)
    extern __shared__ __align__(16) uint8_t smem_raw[];
    __half* sg = reinterpret_cast<__half*>(smem_raw);            // [2 (hi, lo)][MT*16][GP]
    float* spart = reinterpret_cast<float*>(sg + 2 * MT * 16 * GP);  // [8 warps][MT*16][PP]
    const int cid = blockIdx.x / ENC_CLUSTER, dir = cid & 1, b0 = 32 * (cid >> 1), rank = static_cast<int>(cluster_ctarank());
    const int nB = min(p.B - b0, 32);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, j = lane & 3, g = lane >> 2;
    const int Lp = p.L + 2 * EPADR;
    const float S = p.scale2[0];
    __half* const dG = dir ? p.dG[1] : p.dG[0];
    const __half* const gates = dir ? p.gates[1] : p.gates[0];
    const float* const cstate = dir ? p.cstate[1] : p.cstate[0];
    // B fragments of W_hh^T (hi, lo): n-tile nt (units 32 r + 8 nt + n, n = lane / 4), k-step ks of this warp's 128 gate rows
    uint32_t wh[4][8][2], wl[4][8][2];
    {
        const float* W = dir ? p.whh[1] : p.whh[0];
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
            const int u = ENC_UNITS * rank + 8 * nt + g;
#pragma unroll
            for (int ks = 0; ks < 8; ++ks) {
#pragma unroll
                for (int q = 0; q < 2; ++q) {
                    const int k0 = 128 * warp + 16 * ks + 8 * q + 2 * j;
                    __half h0, l0, h1, l1;
                    split16(W[static_cast<long long>(k0) * EH + u], h0, l0);
                    split16(W[static_cast<long long>(k0 + 1) * EH + u], h1, l1);
                    wh[nt][ks][q] = static_cast<uint32_t>(__half_as_ushort(h0)) | (static_cast<uint32_t>(__half_as_ushort(h1)) << 16);
                    wl[nt][ks][q] = static_cast<uint32_t>(__half_as_ushort(l0)) | (static_cast<uint32_t>(__half_as_ushort(l1)) << 16);
                }
            }
        }
    }
    for (int i = threadIdx.x; i < 2 * MT * 16 * GP; i += ENC_THREADS) sg[i] = __float2half_rn(0.f);
    // pointwise items: (batch row, unit) pairs, item = threadIdx.x + 256 q;  unit = item % 32, b = item / 32
    constexpr int NI = MT * 16 * ENC_UNITS / ENC_THREADS;        // 2 MT
    float dcc[NI];
#pragma unroll
    for (int q = 0; q < NI; ++q) dcc[q] = 0.f;
    __syncthreads();
    for (int s = 0; s < p.L; ++s) {
        const int t = dir == 0 ? p.L - 1 - s : s;                // reverse of the forward order
        const int tn = dir == 0 ? t + 1 : t - 1;                 // the step processed just before (its dG feeds dh)
        const int tp = dir == 0 ? t - 1 : t + 1;                 // the forward pass's previous step (c_prev)
        for (int idx = threadIdx.x; idx < nB * (2 * EG / 8); idx += ENC_THREADS) {
            const int bl = idx / (2 * EG / 8), i8 = idx - bl * (2 * EG / 8);          // i8 < 128: hi, else lo
            const uint4 v = ldcg_v4(dG + (static_cast<long long>(b0 + bl) * Lp + EPADR + tn) * (3 * EG) + 8 * i8);
            *reinterpret_cast<uint4*>(sg + ((i8 >> 7) * MT * 16 + bl) * GP + 8 * (i8 & 127)) = v;
        }
        __syncthreads();
        float acc[MT][4][4];
#pragma unroll
        for (int mt = 0; mt < MT; ++mt)
#pragma unroll
            for (int nt = 0; nt < 4; ++nt)
#pragma unroll
                for (int q = 0; q < 4; ++q) acc[mt][nt][q] = 0.f;
#pragma unroll
        for (int ks = 0; ks < 8; ++ks) {
#pragma unroll
            for (int mt = 0; mt < MT; ++mt) {
                const __half* a = sg + (16 * mt + g) * GP + 128 * warp + 16 * ks + 2 * j;
                const __half* l = a + MT * 16 * GP;
                const uint32_t a0 = *reinterpret_cast<const uint32_t*>(a), a1 = *reinterpret_cast<const uint32_t*>(a + 8 * GP);
                const uint32_t a2 = *reinterpret_cast<const uint32_t*>(a + 8), a3 = *reinterpret_cast<const uint32_t*>(a + 8 * GP + 8);
                const uint32_t l0 = *reinterpret_cast<const uint32_t*>(l), l1 = *reinterpret_cast<const uint32_t*>(l + 8 * GP);
                const uint32_t l2 = *reinterpret_cast<const uint32_t*>(l + 8), l3 = *reinterpret_cast<const uint32_t*>(l + 8 * GP + 8);
#pragma unroll
                for (int nt = 0; nt < 4; ++nt) {
                    mma16816(acc[mt][nt], a0, a1, a2, a3, wh[nt][ks][0], wh[nt][ks][1]);
                    mma16816(acc[mt][nt], l0, l1, l2, l3, wh[nt][ks][0], wh[nt][ks][1]);
                    mma16816(acc[mt][nt], a0, a1, a2, a3, wl[nt][ks][0], wl[nt][ks][1]);
                }
            }
        }
#pragma unroll
        for (int mt = 0; mt < MT; ++mt)
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
                float* d0 = spart + (warp * MT * 16 + 16 * mt + g) * PP + 8 * nt + 2 * j;
                d0[0] = acc[mt][nt][0]; d0[1] = acc[mt][nt][1];
                d0[8 * PP] = acc[mt][nt][2]; d0[8 * PP + 1] = acc[mt][nt][3];
            }
        __syncthreads();
#pragma unroll
        for (int q = 0; q < NI; ++q) {
            const int item = threadIdx.x + ENC_THREADS * q, ul = item & (ENC_UNITS - 1), bl = item >> 5;
            if (bl < nB) {
                const int b = b0 + bl;
                const int unit = ENC_UNITS * rank + ul;
                const int len = p.lens ? p.lens[b] : p.L;
                const long long r = static_cast<long long>(b) * Lp + EPADR + t;
                __half* dg = dG + r * (3 * EG);
                float da[4] = {0.f, 0.f, 0.f, 0.f};              // gate pre-activation gradients i, f, g, o
                if (t < len) {
                    float dh = 0.f;
#pragma unroll
                    for (int w2 = 0; w2 < 8; ++w2) dh += spart[(w2 * MT * 16 + bl) * PP + ul];
                    dh = fmaf(p.d_out[b * p.d_sb + t * p.d_sl + dir * EH + unit], S, dh);
                    const __half* gp = gates + r * EG + unit;
                    const float gi = __half2float(gp[0]), gf = __half2float(gp[EH]), gg = __half2float(gp[2 * EH]), go = __half2float(gp[3 * EH]);
                    const float ct = cstate[r * EH + unit];
                    const float cp = cstate[(static_cast<long long>(b) * Lp + EPADR + tp) * EH + unit];   // pad rows: 0
                    const float tc = tanh_f(ct);
                    const float dc = dcc[q] + dh * go * (1.f - tc * tc);
                    da[3] = dh * tc * go * (1.f - go);
                    da[0] = dc * gg * gi * (1.f - gi);
                    da[2] = dc * gi * (1.f - gg * gg);
                    da[1] = dc * cp * gf * (1.f - gf);
                    dcc[q] = dc * gf;
                } else {
                    dcc[q] = 0.f;
                }
#pragma unroll
                for (int e = 0; e < 4; ++e) store_hlh(dg, EG, e * EH + unit, da[e]);
            }
        }
        cluster_sync_all();                                      // dG_t of all 8 CTAs visible (also orders sg / spart reuse)
    }
}

// ------------------------------------------------------------------------------------------------ host orchestration
template <int MT> static int launch_bilstm_fwd(const EncLstmFwdParams& p, cudaStream_t st) {
    enc_bilstm_fwd_kernel<MT><<<2 * ((p.B + 31) / 32) * ENC_CLUSTER, ENC_THREADS, 0, st>>>(p);
    ft_count_launch(1);
    return ft_check_launch("enc_bilstm_fwd_kernel");
}
template <int MT> static int launch_bilstm_bwd(const EncLstmBwdParams& p, cudaStream_t st) {
    const int smem = 2 * MT * 16 * (EG + 8) * 2 + 8 * MT * 16 * (ENC_UNITS + 1) * 4;
    cudaFuncSetAttribute(enc_bilstm_bwd_kernel<MT>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    enc_bilstm_bwd_kernel<MT><<<2 * ((p.B + 31) / 32) * ENC_CLUSTER, ENC_THREADS, smem, st>>>(p);
    ft_count_launch(1);
    return ft_check_launch("enc_bilstm_bwd_kernel");
}
int enc_bilstm_fwd(const EncLstmFwdParams& p, cudaStream_t st) { return p.B <= 16 ? launch_bilstm_fwd<1>(p, st) : launch_bilstm_fwd<2>(p, st); }
int enc_bilstm_bwd(const EncLstmBwdParams& p, cudaStream_t st) { return p.B <= 16 ? launch_bilstm_bwd<1>(p, st) : launch_bilstm_bwd<2>(p, st); }

int enc_wgrad3(cudaStream_t st, int M, int N, long long K, const __half* A, int wa, const __half* B, long long ldb, int wb,
               const float* alpha_ptr, float* C32) {
    for (int term = 0; term < 3; ++term)
        FT_TRY(gemm_wgrad(st, M, N, K, A + (term == 1 ? wa : 0), 3 * wa, B + (term == 2 ? wb : 0), ldb, C32, N, alpha_ptr, term > 0));
    return 0;
}

// ------------------------------------------------------------------------------------------------ conv -> norm -> BiLSTM stack
EncStack enc_stack_plan(const EncStackDesc& a, int B, int L, bool masked, const void* saved, void* scratch, bool bwd) {
    EncStack P{};
    P.a = &a; P.B = B; P.L = L;
    P.rows = static_cast<long long>(B) * (L + 2 * EPADR);
    const size_t rows = static_cast<size_t>(P.rows);
    Workspace sv; sv.base = static_cast<uint8_t*>(const_cast<void*>(saved));
    for (int i = 0; i <= a.layers; ++i) P.X16[i] = sv.get<__half>(rows * 3 * (i == 0 ? a.cp0 : EC));
    for (int i = 0; i < a.layers; ++i) P.Y32[i] = sv.get<float>(rows * EC);
    for (int i = 0; i < a.layers; ++i) { P.mean[i] = sv.get<float>(size_t(B) * EC); P.rstd[i] = sv.get<float>(size_t(B) * EC); }
    for (int k = 0; k < 2; ++k) {
        P.hseq[k] = sv.get<__half>(rows * 2 * EH);
        P.gates[k] = sv.get<__half>(rows * EG);
        P.cstate[k] = sv.get<float>(rows * EH);
    }
    int* lens = sv.get<int>(size_t(B) + 4);
    P.lens = masked ? lens : nullptr;
    P.inv_n = reinterpret_cast<float*>(sv.get<uint8_t>(a.inv_n_bytes));
    P.saved_bytes = sv.off;
    Workspace sc; sc.base = static_cast<uint8_t*>(scratch);
    if (!bwd) {
        P.xproj = sc.get<float>(rows * 2 * EG);
        P.hout = reinterpret_cast<float*>(sc.get<uint8_t>(size_t(B) * L * a.hout_bytes_per_token));
        for (int i = 0; i < a.layers; ++i) P.wconv16[i] = sc.get<__half>(size_t(a.taps) * EC * 3 * (i == 0 ? a.cp0 : EC));
        P.wih16 = sc.get<__half>(size_t(2) * EG * 3 * EC);
        P.fwd_bytes = sc.off;
    } else {
        for (int k = 0; k < 2; ++k) P.dG[k] = sc.get<__half>(rows * 3 * EG);
        P.dY16 = sc.get<__half>(rows * 3 * EC);
        P.DX32 = sc.get<float>(rows * EC);
        P.dwk = sc.get<float>(size_t(a.taps) * EC * EC);
        P.scale2 = sc.get<float>(64);
        P.dmean = reinterpret_cast<float*>(sc.get<uint8_t>(size_t(B) * a.dmean_bytes_per_utt));
        P.wconv16_b = sc.get<__half>(size_t(a.taps) * 3 * EC * EC);
        P.wih16_b = sc.get<__half>(size_t(2) * 3 * EG * EC);
        P.bwd_bytes = sc.off;
    }
    return P;
}

int enc_stack_clear(const EncStack& S, const int* lens, cudaStream_t st) {
    const char* who = S.a->name;
    FT_CU(cudaMemsetAsync(S.X16[0], 0, reinterpret_cast<uint8_t*>(S.Y32[0]) - reinterpret_cast<uint8_t*>(S.X16[0]), st), who);
    for (int k = 0; k < 2; ++k) {
        FT_CU(cudaMemsetAsync(S.hseq[k], 0, S.rows * 2 * EH * 2, st), who);
        FT_CU(cudaMemsetAsync(S.cstate[k], 0, S.rows * EH * 4, st), who);
    }
    if (S.lens) FT_CU(cudaMemcpyAsync(const_cast<int*>(S.lens), lens, sizeof(int) * S.B, cudaMemcpyDeviceToDevice, st), who);
    return 0;
}

int enc_stack_fwd(const EncStack& S, const EncStackWeights& w, float eps, float drop_p, unsigned long long* rng, float* out,
                  long long out_sb, long long out_sl, cudaStream_t st) {
    const EncStackDesc& a = *S.a;
    const int tap0 = EPADR - (a.taps - 1) / 2;                       // grid row offset of tap 0
    for (int i = 0; i < a.layers; ++i) {
        const int cin = i == 0 ? a.cin0 : EC, cp = i == 0 ? a.cp0 : EC;
        a.pack_conv(w.conv_w[i], cin, cp, S.wconv16[i], nullptr, st);
        ft_count_launch(1);
        for (int k = 0; k < a.taps; ++k)                              // one GEMM per tap: contraction over [hi | lo | hi] x [hi | hi | lo]
            FT_TRY(gemm_nt(st, S.rows - 2 * EPADR, EC, 3 * cp, S.X16[i] + static_cast<size_t>(tap0 + k) * 3 * cp, 3 * cp,
                           S.wconv16[i] + static_cast<size_t>(k) * EC * 3 * cp, 3 * cp, S.Y32[i] + static_cast<size_t>(EPADR) * EC, EC,
                           nullptr, 0, k == 0 ? w.conv_b[i] : nullptr, nullptr, 0, k > 0));
        enc_norm_fwd_kernel<<<dim3(S.B, EC / 32), 256, 0, st>>>(S.Y32[i], S.lens, S.L, w.norm_w[i], w.norm_b[i], eps, drop_p,
                                                                 drop_p > 0.f ? rng : nullptr, i, S.X16[i + 1], S.mean[i], S.rstd[i]);
        ft_count_launch(1);
        FT_TRY(ft_check_launch("enc_norm_fwd_kernel"));
    }
    if (drop_p > 0.f) { enc_rng_advance_kernel<<<1, 1, 0, st>>>(rng); ft_count_launch(1); }
    for (int k = 0; k < 2; ++k) {
        __half* wih = S.wih16 + static_cast<size_t>(k) * EG * 3 * EC;
        enc_pack_wih_kernel<<<296, 256, 0, st>>>(w.w_ih[k], wih, nullptr);
        ft_count_launch(1);
        FT_TRY(gemm_nt(st, S.rows, EG, 3 * EC, S.X16[a.layers], 3 * EC, wih, 3 * EC, S.xproj + static_cast<size_t>(k) * EG, 2 * EG,
                       nullptr, 0, w.b_ih[k], w.b_hh[k]));
    }
    EncLstmFwdParams p;
    p.B = S.B; p.L = S.L; p.lens = S.lens; p.xproj = S.xproj;
    for (int k = 0; k < 2; ++k) { p.whh[k] = w.w_hh[k]; p.hseq[k] = S.hseq[k]; p.gates[k] = S.gates[k]; p.cstate[k] = S.cstate[k]; }
    p.out = out; p.out_sb = out_sb; p.out_sl = out_sl;
    return enc_bilstm_fwd(p, st);
}

int enc_stack_bwd(const EncStack& S, const EncStackWeights& w, const EncStackGrads& g, float drop_p, const float* d_out,
                  long long d_sb, long long d_sl, bool want_dx, cudaStream_t st) {
    const EncStackDesc& a = *S.a;
    const char* who = a.name;
    const long long rows = S.rows;
    for (int k = 0; k < 2; ++k) FT_CU(cudaMemsetAsync(S.dG[k], 0, rows * 3 * EG * 2, st), who);
    EncLstmBwdParams p;
    p.B = S.B; p.L = S.L; p.lens = S.lens; p.d_out = d_out; p.d_sb = d_sb; p.d_sl = d_sl; p.scale2 = S.scale2;
    for (int k = 0; k < 2; ++k) { p.whh[k] = w.w_hh[k]; p.gates[k] = S.gates[k]; p.cstate[k] = S.cstate[k]; p.dG[k] = S.dG[k]; }
    FT_TRY(enc_bilstm_bwd(p, st));
    const float* iS = S.scale2 + 1;
    const __half* xl = S.X16[a.layers];
    // BiLSTM parameter gradients and the gradient w.r.t. its input (fp32 grid, still x S)
    for (int k = 0; k < 2; ++k) {
        __half* wih = S.wih16_b + static_cast<size_t>(k) * 3 * EG * EC;
        enc_pack_wih_kernel<<<296, 256, 0, st>>>(w.w_ih[k], nullptr, wih);
        ft_count_launch(1);
        FT_TRY(enc_wgrad3(st, EG, EC, rows, S.dG[k], EG, xl, 3 * EC, EC, iS, g.d_w_ih[k]));                    // dW_ih = dG^T x
        // dW_hh = dG_t^T h_{t -+ 1}: the same grids one row apart
        FT_TRY(enc_wgrad3(st, EG, EH, rows - 1, S.dG[k] + (k == 0 ? 3 * EG : 0), EG, S.hseq[k] + (k == 0 ? 0 : 2 * EH), 2 * EH, EH, iS, g.d_w_hh[k]));
        enc_colsum_hilo_kernel<<<EG / 32, 256, 0, st>>>(S.dG[k], rows, EG, iS, g.d_b_ih[k]);
        ft_count_launch(1);
        FT_CU(cudaMemcpyAsync(g.d_b_hh[k], g.d_b_ih[k], sizeof(float) * EG, cudaMemcpyDeviceToDevice, st), who);
        // dx (+)= dG W_ih: [hi | lo | hi] x [hi ; hi ; lo]
        FT_TRY(gemm_dgrad(st, rows, EC, 3 * EG, S.dG[k], 3 * EG, wih, EC, S.DX32, EC, nullptr, 0, k > 0));
    }
    const int tap0 = EPADR - (a.taps - 1) / 2;
    for (int i = a.layers - 1; i >= 0; --i) {
        const int cin = i == 0 ? a.cin0 : EC, cp = i == 0 ? a.cp0 : EC;
        FT_CU(cudaMemsetAsync(S.dY16, 0, rows * 3 * EC * 2, st), who);
        FT_CU(cudaMemsetAsync(g.d_norm_w[i], 0, sizeof(float) * EC, st), who);
        FT_CU(cudaMemsetAsync(g.d_norm_b[i], 0, sizeof(float) * EC, st), who);
        enc_norm_bwd_kernel<<<dim3(S.B, EC / 32), 256, 0, st>>>(S.DX32, S.X16[i + 1], S.Y32[i], S.lens, S.L, w.norm_w[i], S.mean[i], S.rstd[i],
                                                                 drop_p, S.scale2, S.dY16, g.d_norm_w[i], g.d_norm_b[i]);
        ft_count_launch(1);
        FT_TRY(ft_check_launch("enc_norm_bwd_kernel"));
        enc_colsum_hilo_kernel<<<EC / 32, 256, 0, st>>>(S.dY16, rows, EC, iS, g.d_conv_b[i]);
        ft_count_launch(1);
        for (int k = 0; k < a.taps; ++k)                              // dW_k = dY^T x_i shifted by tap k
            FT_TRY(enc_wgrad3(st, EC, cp, rows - 2 * EPADR, S.dY16 + static_cast<size_t>(EPADR) * 3 * EC, EC,
                              S.X16[i] + static_cast<size_t>(tap0 + k) * 3 * cp, 3 * cp, cp, iS, S.dwk + static_cast<size_t>(k) * EC * cp));
        a.unpack_conv_grad(S.dwk, cin, cp, g.d_conv_w[i], st);
        ft_count_launch(1);
        if (i == 0 && !want_dx) break;
        // dx_i = sum_k dY shifted by -tap . W_k (the layers that get here read 512 channels)
        a.pack_conv(w.conv_w[i], cin, cp, nullptr, S.wconv16_b, st);
        ft_count_launch(1);
        for (int k = 0; k < a.taps; ++k)
            FT_TRY(gemm_dgrad(st, rows - 2 * EPADR, EC, 3 * EC, S.dY16 + static_cast<size_t>(2 * EPADR - tap0 - k) * 3 * EC, 3 * EC,
                              S.wconv16_b + static_cast<size_t>(k) * 3 * EC * EC, EC, S.DX32 + static_cast<size_t>(EPADR) * EC, EC,
                              nullptr, 0, k > 0));
    }
    return 0;
}

// ------------------------------------------------------------------------------------------------ text encoder
static void text_pack_conv(const float* w, int, int, __half* kmajor, __half* stacked, cudaStream_t st) {
    enc_pack_conv_kernel<<<592, 256, 0, st>>>(w, kmajor, stacked);
}
static void text_unpack_conv_grad(const float* dwk, int, int, float* dw, cudaStream_t st) {
    enc_unpack_conv_grad_kernel<<<592, 256, 0, st>>>(dwk, dw);
}
static const EncStackDesc kTextEncoder = {"encoder", 3, EK, EC, EC, 0, 0, 0, text_pack_conv, text_unpack_conv_grad};

static int check_desc(const FtEncoderDesc* d) {
    if (!d) return ft_set_error("encoder: NULL descriptor");
    if (d->C != EC || d->n_convs != 3 || d->ksize != EK) return ft_set_error("encoder: this build supports 3 convolutions of kernel 5 over 512 channels");
    if (d->B < 1 || d->B > 64 || d->L < 1) return ft_set_error("encoder: batch must be in [1, 64] per call");
    if (d->dropout_p < 0.f || d->dropout_p >= 1.f) return ft_set_error("encoder: dropout_p must be in [0, 1)");
    return 0;
}

static EncStack plan(const FtEncoderDesc& d, const void* saved, void* scratch, bool bwd) {
    return enc_stack_plan(kTextEncoder, d.B, d.L, d.masked != 0, saved, scratch, bwd);
}

}  // namespace ft

extern "C" {

size_t ft_encoder_saved_bytes(const FtEncoderDesc* d) { return ft::check_desc(d) ? 0 : ft::plan(*d, nullptr, nullptr, false).saved_bytes + 256; }
size_t ft_encoder_fwd_scratch_bytes(const FtEncoderDesc* d) { return ft::check_desc(d) ? 0 : ft::plan(*d, nullptr, nullptr, false).fwd_bytes + 256; }
size_t ft_encoder_bwd_scratch_bytes(const FtEncoderDesc* d) { return ft::check_desc(d) ? 0 : ft::plan(*d, nullptr, nullptr, true).bwd_bytes + 256; }

static int encoder_fwd_impl(const FtEncoderDesc* d, const FtEncoderWeights* w, const float* x, const long long* tokens, const float* emb, int n_text,
                            const int* in_lens, unsigned long long* rng_state, float* out, long long out_stride_b, long long out_stride_l,
                            void* saved, void* scratch, void* stream) {
    using namespace ft;
    FT_TRY(check_desc(d));
    if (!w || (!x && !(tokens && emb && n_text > 0)) || !out || !saved || !scratch) return ft_set_error("ft_encoder_fwd: NULL argument");
    if (d->dropout_p > 0.f && !rng_state) return ft_set_error("ft_encoder_fwd: dropout needs the device rng state");
    if (d->masked && !in_lens) return ft_set_error("ft_encoder_fwd: masked mode needs in_lens");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const EncStack S = plan(*d, saved, scratch, false);
    const int B = d->B, L = d->L;
    FT_TRY(enc_stack_clear(S, in_lens, st));
    if (x) enc_in_kernel<<<dim3((L + 31) / 32, EC / 32, B), 256, 0, st>>>(x, S.lens, B, L, S.X16[0]);
    else   enc_embed_kernel<<<B * L, 128, 0, st>>>(tokens, emb, n_text, S.lens, B, L, S.X16[0]);
    ft_count_launch(1);
    FT_TRY(ft_check_launch("enc_in_kernel"));
    return enc_stack_fwd(S, stack_weights(*w), d->eps, d->dropout_p, rng_state, out, out_stride_b, out_stride_l, st);
}

int ft_encoder_fwd(const FtEncoderDesc* d, const FtEncoderWeights* w, const float* x, const int* in_lens, unsigned long long* rng_state,
                   float* out, long long out_stride_b, long long out_stride_l, void* saved, void* scratch, void* stream) {
    if (!x) return ft::ft_set_error("ft_encoder_fwd: NULL argument");
    return encoder_fwd_impl(d, w, x, nullptr, nullptr, 0, in_lens, rng_state, out, out_stride_b, out_stride_l, saved, scratch, stream);
}
int ft_encoder_fwd_tokens(const FtEncoderDesc* d, const FtEncoderWeights* w, const long long* tokens, const float* emb_weight, int n_text,
                          const int* in_lens, unsigned long long* rng_state, float* out, long long out_stride_b, long long out_stride_l,
                          void* saved, void* scratch, void* stream) {
    if (!tokens || !emb_weight || n_text <= 0) return ft::ft_set_error("ft_encoder_fwd_tokens: NULL argument");
    return encoder_fwd_impl(d, w, nullptr, tokens, emb_weight, n_text, in_lens, rng_state, out, out_stride_b, out_stride_l, saved, scratch, stream);
}

static int encoder_bwd_impl(const FtEncoderDesc* d, const FtEncoderWeights* w, const float* d_out, long long d_stride_b, long long d_stride_l,
                            const void* saved, float* d_x, const long long* tokens, int n_text, float* d_emb, const FtEncoderGrads* gr,
                            void* scratch, void* stream) {
    using namespace ft;
    FT_TRY(check_desc(d));
    if (!w || !d_out || !saved || !gr || !scratch) return ft_set_error("ft_encoder_bwd: NULL argument");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const EncStack S = plan(*d, saved, scratch, true);
    const int B = d->B, L = d->L;
    if (d_stride_l != 2 * EH || d_stride_b != static_cast<long long>(L) * 2 * EH) return ft_set_error("ft_encoder_bwd: d_out must be dense [B, L, 512]");
    FT_TRY(launch_grad_scale(d_out, static_cast<long long>(B) * L * 2 * EH, nullptr, 0, nullptr, 0, 256.0f, S.scale2, st));
    FT_TRY(enc_stack_bwd(S, stack_weights(*w), stack_grads(*gr), d->dropout_p, d_out, d_stride_b, d_stride_l, d_x || d_emb, st));
    if (d_x) {
        enc_out_grad_kernel<<<dim3((L + 31) / 32, EC / 32, B), 256, 0, st>>>(S.DX32, S.lens, B, L, S.scale2, d_x);
        ft_count_launch(1);
        FT_TRY(ft_check_launch("enc_out_grad_kernel"));
    }
    if (d_emb) {
        FT_CU(cudaMemsetAsync(d_emb, 0, sizeof(float) * static_cast<size_t>(n_text) * EC, st), "encoder");
        enc_embed_grad_kernel<<<B * L, 128, 0, st>>>(S.DX32, tokens, n_text, S.lens, B, L, S.scale2, d_emb);
        ft_count_launch(1);
        FT_TRY(ft_check_launch("enc_embed_grad_kernel"));
    }
    return 0;
}

int ft_encoder_bwd(const FtEncoderDesc* d, const FtEncoderWeights* w, const float* d_out, long long d_stride_b, long long d_stride_l,
                   const void* saved, float* d_x, const FtEncoderGrads* gr, void* scratch, void* stream) {
    return encoder_bwd_impl(d, w, d_out, d_stride_b, d_stride_l, saved, d_x, nullptr, 0, nullptr, gr, scratch, stream);
}
int ft_encoder_bwd_tokens(const FtEncoderDesc* d, const FtEncoderWeights* w, const float* d_out, long long d_stride_b, long long d_stride_l,
                          const void* saved, const long long* tokens, int n_text, float* d_emb_weight, const FtEncoderGrads* gr, void* scratch,
                          void* stream) {
    if (!tokens || !d_emb_weight || n_text <= 0) return ft::ft_set_error("ft_encoder_bwd_tokens: NULL argument");
    return encoder_bwd_impl(d, w, d_out, d_stride_b, d_stride_l, saved, nullptr, tokens, n_text, d_emb_weight, gr, scratch, stream);
}

}  // extern "C"
