// MelEncoder of the Gaussian-mixture prior (flowtron.py:416-439): 2 x [conv k=3 -> MaskedInstanceNorm1d (affine) -> relu ->
// dropout] (80 -> 512 -> 512 channels), a packed bidirectional LSTM (hidden 256 per direction) and the mean over time, forward
// and backward (weight gradients only: nothing upstream of the mel needs a gradient).
//
// Everything after the first convolution is the text encoder's device code (encoder_kernels.cuh): the same padded channels-last
// frame grid  row(b, t) = b * (T + 4) + 2 + t  with zero pad rows, the same split-fp16 [hi | lo | hi] operands, instance-norm and
// cluster-BiLSTM kernels.  A k = 3, pad 1 convolution is 3 shifted wgmma GEMMs over that grid (taps at row offsets -1, 0, +1).
// The first layer's 80 mel channels are stored 128 wide (zero columns 80..127) so its contraction is a whole number of 64-wide
// GEMM k-blocks.  Frames at t >= out_lens[b] are written as zero and never read, so the caller's padding (even NaN) is ignored
// and the caller's mel is not written (the reference zeroes it in place, flowtron.py:428).
//
// The reference averages the padded LSTM output over max(out_lens) frames (torch.mean over pad_packed_sequence's output), so
// the divisor is the longest row of the WHOLE batch; callers that slice a batch pass all of its lengths for that maximum.
#include "encoder_kernels.cuh"
#include "../../include/flowtron_b200.h"

namespace ft {

constexpr int MK = 3;                   // conv taps
constexpr int MEL_C = 80, MEL_CP = 128; // mel channels, their padded width in the grid

// mel [B, 80, T] fp32 -> first grid (split fp16, 128 columns per part); frames at t >= len and columns >= 80 stay zero
__global__ void mel_enc_in_kernel(const float* __restrict__ mel, const int* __restrict__ lens, int T, __half* __restrict__ X16) {
    __shared__ float tile[32][33];
    const int b = blockIdx.z, t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int len = lens[b];
    for (int i = ty; i < 32; i += 8) {
        const int t = t0 + tx, c = c0 + i;
        tile[i][tx] = (t < len && c < MEL_C) ? mel[(static_cast<long long>(b) * MEL_C + c) * T + t] : 0.f;
    }
    __syncthreads();
    for (int i = ty; i < 32; i += 8) {
        const int t = t0 + i;
        if (t < T) store_hlh(X16 + (static_cast<long long>(b) * (T + 2 * EPADR) + EPADR + t) * (3 * MEL_CP), MEL_CP, c0 + tx, tile[tx][i]);
    }
}

// conv.weight [512, cin, 3] fp32 -> per tap k, split fp16 (columns cin..cp-1 zero):
//   kmajor  [k][co][3 cp] = [hi | hi | lo]                (B operand of the forward GEMM)
//   stacked [k][3 x 512 (hi ; hi ; lo rows of co)][cin]  (MN-major B operand of the dgrad GEMM; needs cp == cin)
__global__ void mel_pack_conv_kernel(const float* __restrict__ w, int cin, int cp, __half* __restrict__ kmajor, __half* __restrict__ stacked) {
    const long long n = static_cast<long long>(MK) * EC * cp;
    for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int ci = static_cast<int>(i % cp), co = static_cast<int>((i / cp) % EC), k = static_cast<int>(i / (static_cast<long long>(EC) * cp));
        __half hi = __float2half_rn(0.f), lo = hi;
        if (ci < cin) split16(w[(static_cast<long long>(co) * cin + ci) * MK + k], hi, lo);
        if (kmajor) {
            __half* r = kmajor + (static_cast<long long>(k) * EC + co) * (3 * cp);
            r[ci] = hi; r[cp + ci] = hi; r[2 * cp + ci] = lo;
        }
        if (stacked) {
            __half* t = stacked + static_cast<long long>(k) * 3 * EC * cin;
            t[static_cast<long long>(co) * cin + ci] = hi; t[static_cast<long long>(EC + co) * cin + ci] = hi; t[static_cast<long long>(2 * EC + co) * cin + ci] = lo;
        }
    }
}
// dW [k][co][cp] fp32 -> conv.weight.grad [co, cin, k]
__global__ void mel_unpack_conv_grad_kernel(const float* __restrict__ dwk, int cin, int cp, float* __restrict__ dw) {
    const long long n = static_cast<long long>(MK) * EC * cin;
    for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int k = static_cast<int>(i % MK), ci = static_cast<int>((i / MK) % cin), co = static_cast<int>(i / (static_cast<long long>(MK) * cin));
        dw[i] = dwk[(static_cast<long long>(k) * EC + co) * cp + ci];
    }
}

// emb[b, c] = sum_{t < len_b} h[b, t, c] / max(all_lens); one thread per (utterance, channel), frames summed in order.  inv_n
// (1 / the divisor) is saved for the backward pass.
__global__ void mel_enc_mean_kernel(const float* __restrict__ h, const int* __restrict__ lens, int T, const int* __restrict__ all_lens, int n_all,
                                    float* __restrict__ emb, float* __restrict__ inv_n) {
    const int b = blockIdx.x, c = blockIdx.y * blockDim.x + threadIdx.x;
    int mx = 0;
    for (int i = 0; i < n_all; ++i) mx = max(mx, all_lens[i]);
    const float inv = 1.0f / static_cast<float>(mx);
    const int len = min(lens[b], T);
    const float* src = h + static_cast<long long>(b) * T * (2 * EH) + c;
    float s = 0.f;
    for (int t = 0; t < len; ++t) s += src[static_cast<long long>(t) * (2 * EH)];
    emb[b * (2 * EH) + c] = s * inv;
    if (b == 0 && c == 0) inv_n[0] = inv;
}
// gradient of the mean: every frame t < len_b of row b receives d_emb[b] / max(all_lens) (the BiLSTM backward reads it with a zero
// frame stride)
__global__ void mel_enc_dmean_kernel(const float* __restrict__ d_emb, const float* __restrict__ inv_n, int n, float* __restrict__ dmean) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dmean[i] = d_emb[i] * inv_n[0];
}

struct MelEncPlan {
    // saved by the forward pass for the backward pass
    __half* X16[3];        // block inputs: mel grid [rows, 3 * 128], x1, x2 [rows, 3 * 512]
    float* Y32[2];         // conv outputs (fp32 grid)
    float* mean[2]; float* rstd[2];
    __half* hseq[2]; __half* gates[2]; float* cstate[2];
    int* lens;             // int32 copy of out_lens
    float* inv_n;          // 1 / max(out_lens)
    size_t saved_bytes;
    // forward scratch
    float* xproj; float* hout; __half* wconv16[2]; __half* wih16;
    size_t total_fwd;
    // backward scratch
    __half* dG[2]; __half* dY16; float* DX32; float* dwk; float* scale2; float* dmean; __half* wconv16_b; __half* wih16_b;
    size_t total_bwd;
};

static int cp_of(int layer) { return layer == 0 ? MEL_CP : EC; }

static MelEncPlan plan_mel(const FtMelEncoderDesc& d, uint8_t* saved, uint8_t* scratch, bool bwd) {
    MelEncPlan P{};
    const size_t rows = static_cast<size_t>(d.B) * (d.T + 2 * EPADR);
    size_t off = 0;
    auto get = [&](uint8_t* base, size_t bytes) { size_t o = off; off = (off + bytes + 255) & ~size_t(255); return base ? base + o : nullptr; };
    for (int i = 0; i < 3; ++i) P.X16[i] = reinterpret_cast<__half*>(get(saved, rows * 3 * (i == 0 ? MEL_CP : EC) * 2));
    for (int i = 0; i < 2; ++i) P.Y32[i] = reinterpret_cast<float*>(get(saved, rows * EC * 4));
    for (int i = 0; i < 2; ++i) { P.mean[i] = reinterpret_cast<float*>(get(saved, size_t(d.B) * EC * 4)); P.rstd[i] = reinterpret_cast<float*>(get(saved, size_t(d.B) * EC * 4)); }
    for (int k = 0; k < 2; ++k) {
        P.hseq[k] = reinterpret_cast<__half*>(get(saved, rows * 2 * EH * 2));
        P.gates[k] = reinterpret_cast<__half*>(get(saved, rows * EG * 2));
        P.cstate[k] = reinterpret_cast<float*>(get(saved, rows * EH * 4));
    }
    P.lens = reinterpret_cast<int*>(get(saved, size_t(d.B) * 4 + 16));
    P.inv_n = reinterpret_cast<float*>(get(saved, 16));
    P.saved_bytes = off;
    off = 0;
    if (!bwd) {
        P.xproj = reinterpret_cast<float*>(get(scratch, rows * 2 * EG * 4));
        P.hout = reinterpret_cast<float*>(get(scratch, size_t(d.B) * d.T * 2 * EH * 4));
        for (int i = 0; i < 2; ++i) P.wconv16[i] = reinterpret_cast<__half*>(get(scratch, size_t(MK) * EC * 3 * cp_of(i) * 2));
        P.wih16 = reinterpret_cast<__half*>(get(scratch, size_t(2) * EG * 3 * EC * 2));
        P.total_fwd = off;
    } else {
        for (int k = 0; k < 2; ++k) P.dG[k] = reinterpret_cast<__half*>(get(scratch, rows * 3 * EG * 2));
        P.dY16 = reinterpret_cast<__half*>(get(scratch, rows * 3 * EC * 2));
        P.DX32 = reinterpret_cast<float*>(get(scratch, rows * EC * 4));
        P.dwk = reinterpret_cast<float*>(get(scratch, size_t(MK) * EC * EC * 4));
        P.scale2 = reinterpret_cast<float*>(get(scratch, 256));
        P.dmean = reinterpret_cast<float*>(get(scratch, size_t(d.B) * 2 * EH * 4));
        P.wconv16_b = reinterpret_cast<__half*>(get(scratch, size_t(MK) * 3 * EC * EC * 2));
        P.wih16_b = reinterpret_cast<__half*>(get(scratch, size_t(2) * 3 * EG * EC * 2));
        P.total_bwd = off;
    }
    return P;
}

static int check_mel_desc(const FtMelEncoderDesc* d) {
    if (!d) return ft_set_error("mel encoder: NULL descriptor");
    if (d->B < 1 || d->B > FT_MEL_ENC_MAX_BATCH) return ft_set_error("mel encoder: batch must be in [1, 64] per call");
    if (d->T < 1) return ft_set_error("mel encoder: T must be positive");
    if (d->dropout_p < 0.f || d->dropout_p >= 1.f) return ft_set_error("mel encoder: dropout_p must be in [0, 1)");
    return 0;
}

}  // namespace ft

extern "C" {

size_t ft_mel_encoder_saved_bytes(const FtMelEncoderDesc* d) { return ft::check_mel_desc(d) ? 0 : ft::plan_mel(*d, nullptr, nullptr, false).saved_bytes + 256; }
size_t ft_mel_encoder_fwd_scratch_bytes(const FtMelEncoderDesc* d) { return ft::check_mel_desc(d) ? 0 : ft::plan_mel(*d, nullptr, nullptr, false).total_fwd + 256; }
size_t ft_mel_encoder_bwd_scratch_bytes(const FtMelEncoderDesc* d) { return ft::check_mel_desc(d) ? 0 : ft::plan_mel(*d, nullptr, nullptr, true).total_bwd + 256; }

#define FT_TRYM(x) do { if ((x) != 0) return -1; } while (0)
#define FT_CUM(x) do { if ((x) != cudaSuccess) return ft::ft_set_error("mel encoder: CUDA runtime call failed"); } while (0)

int ft_mel_encoder_fwd(const FtMelEncoderDesc* d, const FtMelEncoderWeights* w, const float* mel, const int* out_lens, const int* all_lens,
                       int n_all, unsigned long long* rng_state, float* emb, void* saved, void* scratch, void* stream) {
    using namespace ft;
    FT_TRYM(check_mel_desc(d));
    if (!w || !mel || !out_lens || !all_lens || n_all < 1 || !emb || !saved || !scratch) return ft_set_error("ft_mel_encoder_fwd: NULL argument");
    if (d->dropout_p > 0.f && !rng_state) return ft_set_error("ft_mel_encoder_fwd: dropout needs the device rng state");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    MelEncPlan P = plan_mel(*d, static_cast<uint8_t*>(saved), static_cast<uint8_t*>(scratch), false);
    const int B = d->B, T = d->T, Tp = T + 2 * EPADR;
    const long long rows = static_cast<long long>(B) * Tp;
    // zero the fp16 grids (pad rows and frames past a row's length read as zero), the exchange tensor and c
    FT_CUM(cudaMemsetAsync(P.X16[0], 0, reinterpret_cast<uint8_t*>(P.Y32[0]) - reinterpret_cast<uint8_t*>(P.X16[0]), st));
    for (int k = 0; k < 2; ++k) {
        FT_CUM(cudaMemsetAsync(P.hseq[k], 0, rows * 2 * EH * 2, st));
        FT_CUM(cudaMemsetAsync(P.cstate[k], 0, rows * EH * 4, st));
    }
    FT_CUM(cudaMemcpyAsync(P.lens, out_lens, sizeof(int) * B, cudaMemcpyDeviceToDevice, st));
    mel_enc_in_kernel<<<dim3((T + 31) / 32, MEL_CP / 32, B), 256, 0, st>>>(mel, P.lens, T, P.X16[0]);
    ft_count_launch(1);
    FT_TRYM(ft_check_launch("mel_enc_in_kernel"));
    for (int i = 0; i < 2; ++i) {
        const int cin = i == 0 ? MEL_C : EC, cp = cp_of(i);
        mel_pack_conv_kernel<<<592, 256, 0, st>>>(w->conv_w[i], cin, cp, P.wconv16[i], nullptr);
        ft_count_launch(1);
        for (int k = 0; k < MK; ++k) {
            GemmArgs g;                                               // tap k reads frame t + k - 1: the grid shifted by k + 1 rows
            g.M = static_cast<int>(rows - 2 * EPADR); g.N = EC; g.K = 3 * cp;
            g.A = P.X16[i] + static_cast<size_t>(k + 1) * 3 * cp; g.lda = 3 * cp; g.a_fmt = FMT_F16;
            g.B = P.wconv16[i] + static_cast<size_t>(k) * EC * 3 * cp; g.ldb = 3 * cp; g.b_fmt = FMT_F16;
            g.bias = k == 0 ? w->conv_b[i] : nullptr; g.beta = k > 0;
            g.C32 = P.Y32[i] + static_cast<size_t>(EPADR) * EC; g.ldc32 = EC;
            FT_TRYM(launch_gemm(g, st));
        }
        enc_norm_fwd_kernel<<<dim3(B, EC / 32), 256, 0, st>>>(P.Y32[i], P.lens, T, w->norm_w[i], w->norm_b[i], d->eps, d->dropout_p,
                                                               d->dropout_p > 0.f ? rng_state : nullptr, i, P.X16[i + 1], P.mean[i], P.rstd[i]);
        ft_count_launch(1);
        FT_TRYM(ft_check_launch("enc_norm_fwd_kernel"));
    }
    if (d->dropout_p > 0.f) { enc_rng_advance_kernel<<<1, 1, 0, st>>>(rng_state); ft_count_launch(1); }
    for (int k = 0; k < 2; ++k) {
        __half* wih = P.wih16 + static_cast<size_t>(k) * EG * 3 * EC;
        enc_pack_wih_kernel<<<296, 256, 0, st>>>(w->w_ih[k], wih, nullptr);
        ft_count_launch(1);
        GemmArgs g;
        g.M = static_cast<int>(rows); g.N = EG; g.K = 3 * EC;
        g.A = P.X16[2]; g.lda = 3 * EC; g.a_fmt = FMT_F16;
        g.B = wih; g.ldb = 3 * EC; g.b_fmt = FMT_F16;
        g.bias = w->b_ih[k]; g.bias2 = w->b_hh[k];
        g.C32 = P.xproj + static_cast<size_t>(k) * EG; g.ldc32 = 2 * EG;
        FT_TRYM(launch_gemm(g, st));
    }
    EncLstmFwdParams p;
    p.B = B; p.L = T; p.lens = P.lens; p.xproj = P.xproj;
    for (int k = 0; k < 2; ++k) { p.whh[k] = w->w_hh[k]; p.hseq[k] = P.hseq[k]; p.gates[k] = P.gates[k]; p.cstate[k] = P.cstate[k]; }
    p.out = P.hout; p.out_sb = static_cast<long long>(T) * 2 * EH; p.out_sl = 2 * EH;
    FT_TRYM(enc_bilstm_fwd(p, st));
    mel_enc_mean_kernel<<<dim3(B, 2 * EH / 128), 128, 0, st>>>(P.hout, P.lens, T, all_lens, n_all, emb, P.inv_n);
    ft_count_launch(1);
    return ft_check_launch("mel_enc_mean_kernel");
}

int ft_mel_encoder_bwd(const FtMelEncoderDesc* d, const FtMelEncoderWeights* w, const float* d_emb, const void* saved,
                       const FtMelEncoderGrads* gr, void* scratch, void* stream) {
    using namespace ft;
    FT_TRYM(check_mel_desc(d));
    if (!w || !d_emb || !saved || !gr || !scratch) return ft_set_error("ft_mel_encoder_bwd: NULL argument");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    MelEncPlan P = plan_mel(*d, const_cast<uint8_t*>(static_cast<const uint8_t*>(saved)), static_cast<uint8_t*>(scratch), true);
    const int B = d->B, T = d->T, Tp = T + 2 * EPADR;
    const long long rows = static_cast<long long>(B) * Tp;
    const int n_emb = B * 2 * EH;
    mel_enc_dmean_kernel<<<(n_emb + 255) / 256, 256, 0, st>>>(d_emb, P.inv_n, n_emb, P.dmean);
    ft_count_launch(1);
    FT_TRYM(ft_check_launch("mel_enc_dmean_kernel"));
    FT_TRYM(launch_grad_scale(P.dmean, n_emb, nullptr, 0, nullptr, 0, 256.0f, P.scale2, st));
    for (int k = 0; k < 2; ++k) FT_CUM(cudaMemsetAsync(P.dG[k], 0, rows * 3 * EG * 2, st));
    EncLstmBwdParams p;
    p.B = B; p.L = T; p.lens = P.lens; p.d_out = P.dmean; p.d_sb = 2 * EH; p.d_sl = 0; p.scale2 = P.scale2;
    for (int k = 0; k < 2; ++k) { p.whh[k] = w->w_hh[k]; p.gates[k] = P.gates[k]; p.cstate[k] = P.cstate[k]; p.dG[k] = P.dG[k]; }
    FT_TRYM(enc_bilstm_bwd(p, st));
    const float* iS = P.scale2 + 1;
    for (int k = 0; k < 2; ++k) {
        __half* wih = P.wih16_b + static_cast<size_t>(k) * 3 * EG * EC;
        enc_pack_wih_kernel<<<296, 256, 0, st>>>(w->w_ih[k], nullptr, wih);
        ft_count_launch(1);
        FT_TRYM(enc_wgrad3(st, EG, EC, rows, P.dG[k], EG, P.X16[2], 3 * EC, EC, iS, gr->d_w_ih[k]));           // dW_ih = dG^T x2
        // dW_hh = dG_t^T h_{t -+ 1}: the same grids one row apart
        FT_TRYM(enc_wgrad3(st, EG, EH, rows - 1, P.dG[k] + (k == 0 ? 3 * EG : 0), EG, P.hseq[k] + (k == 0 ? 0 : 2 * EH), 2 * EH, EH, iS, gr->d_w_hh[k]));
        enc_colsum_hilo_kernel<<<EG / 32, 256, 0, st>>>(P.dG[k], rows, EG, iS, gr->d_b_ih[k]);
        ft_count_launch(1);
        FT_CUM(cudaMemcpyAsync(gr->d_b_hh[k], gr->d_b_ih[k], sizeof(float) * EG, cudaMemcpyDeviceToDevice, st));
        GemmArgs x;                                                   // dx2 (+)= dG W_ih: [hi | lo | hi] x [hi ; hi ; lo]
        x.M = static_cast<int>(rows); x.N = EC; x.K = 3 * EG;
        x.A = P.dG[k]; x.lda = 3 * EG; x.a_fmt = FMT_F16;
        x.B = wih; x.ldb = EC; x.b_fmt = FMT_F16; x.b_mn = 1;
        x.beta = k > 0; x.C32 = P.DX32; x.ldc32 = EC;
        FT_TRYM(launch_gemm(x, st));
    }
    for (int i = 1; i >= 0; --i) {
        const int cin = i == 0 ? MEL_C : EC, cp = cp_of(i);
        FT_CUM(cudaMemsetAsync(P.dY16, 0, rows * 3 * EC * 2, st));
        FT_CUM(cudaMemsetAsync(gr->d_norm_w[i], 0, sizeof(float) * EC, st));
        FT_CUM(cudaMemsetAsync(gr->d_norm_b[i], 0, sizeof(float) * EC, st));
        enc_norm_bwd_kernel<<<dim3(B, EC / 32), 256, 0, st>>>(P.DX32, P.X16[i + 1], P.Y32[i], P.lens, T, w->norm_w[i], P.mean[i], P.rstd[i],
                                                               d->dropout_p, P.scale2, P.dY16, gr->d_norm_w[i], gr->d_norm_b[i]);
        ft_count_launch(1);
        FT_TRYM(ft_check_launch("enc_norm_bwd_kernel"));
        enc_colsum_hilo_kernel<<<EC / 32, 256, 0, st>>>(P.dY16, rows, EC, iS, gr->d_conv_b[i]);
        ft_count_launch(1);
        for (int k = 0; k < MK; ++k)                                  // dW_k = dY^T x_i shifted by tap k
            FT_TRYM(enc_wgrad3(st, EC, cp, rows - 2 * EPADR, P.dY16 + static_cast<size_t>(EPADR) * 3 * EC, EC,
                               P.X16[i] + static_cast<size_t>(k + 1) * 3 * cp, 3 * cp, cp, iS, P.dwk + static_cast<size_t>(k) * EC * cp));
        mel_unpack_conv_grad_kernel<<<592, 256, 0, st>>>(P.dwk, cin, cp, gr->d_conv_w[i]);
        ft_count_launch(1);
        if (i == 0) break;                                            // no gradient w.r.t. the mel
        mel_pack_conv_kernel<<<592, 256, 0, st>>>(w->conv_w[i], cin, cp, nullptr, P.wconv16_b);
        ft_count_launch(1);
        for (int k = 0; k < MK; ++k) {
            GemmArgs g;                                               // dx_1[s] = sum_k dY[s + 1 - k] . W_k
            g.M = static_cast<int>(rows - 2 * EPADR); g.N = EC; g.K = 3 * EC;
            g.A = P.dY16 + static_cast<size_t>(3 - k) * 3 * EC; g.lda = 3 * EC; g.a_fmt = FMT_F16;
            g.B = P.wconv16_b + static_cast<size_t>(k) * 3 * EC * EC; g.ldb = EC; g.b_fmt = FMT_F16; g.b_mn = 1;
            g.beta = k > 0; g.C32 = P.DX32 + static_cast<size_t>(EPADR) * EC; g.ldc32 = EC;
            FT_TRYM(launch_gemm(g, st));
        }
    }
    return 0;
}

}  // extern "C"
