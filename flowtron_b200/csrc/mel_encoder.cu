// MelEncoder of the Gaussian-mixture prior (flowtron.py:416-439): 2 x [conv k=3 -> MaskedInstanceNorm1d (affine) -> relu ->
// dropout] (80 -> 512 -> 512 channels), a packed bidirectional LSTM (hidden 256 per direction) and the mean over time, forward
// and backward (weight gradients only: nothing upstream of the mel needs a gradient).
//
// Everything between the first grid and the BiLSTM output runs on the text encoder's device and host code: the
// conv -> norm -> BiLSTM stack of encoder_kernels.cuh (enc_stack_*, in encoder.cu), driven by the descriptor below.  It keeps
// the same padded channels-last frame grid  row(b, t) = b * (T + 4) + 2 + t  with zero pad rows and the same split-fp16
// [hi | lo | hi] operands; a k = 3, pad 1 convolution is 3 shifted wgmma GEMMs over that grid (taps at row offsets -1, 0, +1).
// This file holds the mel-specific kernels: the input grid, the conv weight packing for a first layer of 80 channels, and the
// time mean.  The first layer's 80 mel channels are stored 128 wide (zero columns 80..127) so its contraction is a whole number
// of 64-wide GEMM k-blocks.  Frames at t >= out_lens[b] are written as zero and never read, so the caller's padding (even NaN)
// is ignored and the caller's mel is not written (the reference zeroes it in place, flowtron.py:428).
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

static void mel_pack_conv(const float* w, int cin, int cp, __half* kmajor, __half* stacked, cudaStream_t st) {
    mel_pack_conv_kernel<<<592, 256, 0, st>>>(w, cin, cp, kmajor, stacked);
}
static void mel_unpack_conv_grad(const float* dwk, int cin, int cp, float* dw, cudaStream_t st) {
    mel_unpack_conv_grad_kernel<<<592, 256, 0, st>>>(dwk, cin, cp, dw);
}
// saved: 1 / max(out_lens); forward scratch: the BiLSTM output [B, T, 512] the mean reads; backward scratch: its gradient [B, 512]
static const EncStackDesc kMelEncoder = {"mel encoder", 2, MK, MEL_C, MEL_CP, 16, 2 * EH * 4, 2 * EH * 4, mel_pack_conv, mel_unpack_conv_grad};

static int check_mel_desc(const FtMelEncoderDesc* d) {
    if (!d) return ft_set_error("mel encoder: NULL descriptor");
    if (d->B < 1 || d->B > FT_MEL_ENC_MAX_BATCH) return ft_set_error("mel encoder: batch must be in [1, 64] per call");
    if (d->T < 1) return ft_set_error("mel encoder: T must be positive");
    if (d->dropout_p < 0.f || d->dropout_p >= 1.f) return ft_set_error("mel encoder: dropout_p must be in [0, 1)");
    return 0;
}

static EncStack plan(const FtMelEncoderDesc& d, const void* saved, void* scratch, bool bwd) {
    return enc_stack_plan(kMelEncoder, d.B, d.T, true, saved, scratch, bwd);
}

}  // namespace ft

extern "C" {

size_t ft_mel_encoder_saved_bytes(const FtMelEncoderDesc* d) { return ft::check_mel_desc(d) ? 0 : ft::plan(*d, nullptr, nullptr, false).saved_bytes + 256; }
size_t ft_mel_encoder_fwd_scratch_bytes(const FtMelEncoderDesc* d) { return ft::check_mel_desc(d) ? 0 : ft::plan(*d, nullptr, nullptr, false).fwd_bytes + 256; }
size_t ft_mel_encoder_bwd_scratch_bytes(const FtMelEncoderDesc* d) { return ft::check_mel_desc(d) ? 0 : ft::plan(*d, nullptr, nullptr, true).bwd_bytes + 256; }

int ft_mel_encoder_fwd(const FtMelEncoderDesc* d, const FtMelEncoderWeights* w, const float* mel, const int* out_lens, const int* all_lens,
                       int n_all, unsigned long long* rng_state, float* emb, void* saved, void* scratch, void* stream) {
    using namespace ft;
    FT_TRY(check_mel_desc(d));
    if (!w || !mel || !out_lens || !all_lens || n_all < 1 || !emb || !saved || !scratch) return ft_set_error("ft_mel_encoder_fwd: NULL argument");
    if (d->dropout_p > 0.f && !rng_state) return ft_set_error("ft_mel_encoder_fwd: dropout needs the device rng state");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const EncStack S = plan(*d, saved, scratch, false);
    const int B = d->B, T = d->T;
    FT_TRY(enc_stack_clear(S, out_lens, st));
    mel_enc_in_kernel<<<dim3((T + 31) / 32, MEL_CP / 32, B), 256, 0, st>>>(mel, S.lens, T, S.X16[0]);
    ft_count_launch(1);
    FT_TRY(ft_check_launch("mel_enc_in_kernel"));
    FT_TRY(enc_stack_fwd(S, stack_weights(*w), d->eps, d->dropout_p, rng_state, S.hout, static_cast<long long>(T) * 2 * EH, 2 * EH, st));
    mel_enc_mean_kernel<<<dim3(B, 2 * EH / 128), 128, 0, st>>>(S.hout, S.lens, T, all_lens, n_all, emb, S.inv_n);
    ft_count_launch(1);
    return ft_check_launch("mel_enc_mean_kernel");
}

int ft_mel_encoder_bwd(const FtMelEncoderDesc* d, const FtMelEncoderWeights* w, const float* d_emb, const void* saved,
                       const FtMelEncoderGrads* gr, void* scratch, void* stream) {
    using namespace ft;
    FT_TRY(check_mel_desc(d));
    if (!w || !d_emb || !saved || !gr || !scratch) return ft_set_error("ft_mel_encoder_bwd: NULL argument");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const EncStack S = plan(*d, saved, scratch, true);
    const int n_emb = d->B * 2 * EH;
    mel_enc_dmean_kernel<<<(n_emb + 255) / 256, 256, 0, st>>>(d_emb, S.inv_n, n_emb, S.dmean);
    ft_count_launch(1);
    FT_TRY(ft_check_launch("mel_enc_dmean_kernel"));
    FT_TRY(launch_grad_scale(S.dmean, n_emb, nullptr, 0, nullptr, 0, 256.0f, S.scale2, st));
    // every frame of row b reads d_emb[b]: a zero frame stride; no gradient w.r.t. the mel
    return enc_stack_bwd(S, stack_weights(*w), stack_grads(*gr), d->dropout_p, S.dmean, 2 * EH, 0, false, st);
}

}  // extern "C"
