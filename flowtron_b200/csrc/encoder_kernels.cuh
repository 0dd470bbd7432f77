// Code shared by the text encoder (encoder.cu) and the mel encoder (mel_encoder.cu): the padded channels-last token grid,
// the split-fp16 operand format, the instance-norm / BiLSTM kernels and their launchers, and the host path of the
// conv -> norm -> BiLSTM stack (enc_stack_*), which runs both encoders from a descriptor of their shapes.  Kernels and host
// path are defined once, in encoder.cu; mel_encoder.cu keeps only its own kernels and entry points.
#pragma once
#include <cuda_fp16.h>
#include "ptx.cuh"
#include "ft_internal.h"

namespace ft {

constexpr int EC = 512, EH = 256, EG = 4 * EH;      // embedding / conv channels, hidden per direction, gate rows
constexpr int EK = 5, EPADR = 2;                    // conv taps, pad rows on either side of an utterance
constexpr int ENC_THREADS = 256, ENC_CLUSTER = 8, ENC_UNITS = EH / ENC_CLUSTER;   // 32 units per CTA

__device__ __forceinline__ uint32_t pack_h2(float a, float b) { const __half2 h = __floats2half2_rn(a, b); return *reinterpret_cast<const uint32_t*>(&h); }
__device__ __forceinline__ uint4 ldcg_v4(const void* p) {
    uint4 v;
    asm volatile("ld.global.cg.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ float sat16(float x) { return fminf(fmaxf(x, -65504.f), 65504.f); }
// x -> (hi, lo) fp16 pair with hi + lo = x to ~22 bits (saturating)
__device__ __forceinline__ void split16(float x, __half& hi, __half& lo) {
    x = sat16(x);
    hi = __float2half_rn(x);
    lo = __float2half_rn(x - __half2float(hi));
}
// row of an activation / gradient grid: [hi (W) | lo (W) | hi (W)]
__device__ __forceinline__ void store_hlh(__half* row, int W, int c, float x) {
    __half hi, lo;
    split16(x, hi, lo);
    row[c] = hi; row[W + c] = lo; row[2 * W + c] = hi;
}

struct EncLstmFwdParams {
    int B, L;
    const int* lens;               // [B] or null (all L)
    const float* xproj;            // [rows, 2 * 1024] fp32: W_ih x + b_ih + b_hh, direction-major columns
    const float* whh[2];           // [1024, 256] fp32 per direction (PyTorch layout, gate order i,f,g,o)
    __half* hseq[2];               // [rows, 2 * 256] split fp16 [hi | lo] per direction: h_t, zero at pads / l >= len
    __half* gates[2];              // [rows, 1024] fp16 post-activation i,f,g,o (or null)
    float* cstate[2];              // [rows, 256] fp32 (or null)
    float* out; long long out_sb, out_sl;   // fp32 output [.., 512]: element (b, l, dir * 256 + u) at out + b * out_sb + l * out_sl + ..
};

struct EncLstmBwdParams {
    int B, L;
    const int* lens;
    const float* d_out; long long d_sb, d_sl;    // gradient w.r.t. the encoder output (fp32, unscaled), same indexing as the forward output
    const float* scale2;                        // device {S, 1/S}
    const float* whh[2];
    const __half* gates[2]; const float* cstate[2];
    __half* dG[2];                               // [rows, 3 * 1024] split fp16 [hi|lo|hi], zero-initialised: S * d(gate pre-activations)
};

__global__ void enc_pack_wih_kernel(const float* __restrict__ w, __half* __restrict__ kmajor, __half* __restrict__ stacked);
__global__ void enc_colsum_hilo_kernel(const __half* __restrict__ src, long long R, int W, const float* __restrict__ scale, float* __restrict__ out);
__global__ void enc_norm_fwd_kernel(const float* __restrict__ Y, const int* __restrict__ lens, int L, const float* __restrict__ w, const float* __restrict__ bias,
                                    float eps, float drop_p, const unsigned long long* __restrict__ rng, int layer, __half* __restrict__ out,
                                    float* __restrict__ mean_out, float* __restrict__ rstd_out);
__global__ void enc_norm_bwd_kernel(const float* __restrict__ DX, const __half* __restrict__ xout, const float* __restrict__ Y, const int* __restrict__ lens, int L,
                                    const float* __restrict__ w, const float* __restrict__ mean_in, const float* __restrict__ rstd_in, float drop_p,
                                    const float* __restrict__ scale2, __half* __restrict__ dY, float* __restrict__ dw, float* __restrict__ db);
__global__ void enc_rng_advance_kernel(unsigned long long* rng);

// BiLSTM recurrences over up to 64 utterances (two clusters of 8 CTAs per 32 utterances and direction)
int enc_bilstm_fwd(const EncLstmFwdParams& p, cudaStream_t st);
int enc_bilstm_bwd(const EncLstmBwdParams& p, cudaStream_t st);
// wgrad over split grids: C32[M, N] = alpha * (A_hi^T B_hi + A_lo^T B_hi + A_hi^T B_lo); A [K rows, 3 wa] (M = wa), B [K rows, ldb] with
// its hi / lo column blocks `wb` apart
int enc_wgrad3(cudaStream_t st, int M, int N, long long K, const __half* A, int wa, const __half* B, long long ldb, int wb,
               const float* alpha_ptr, float* C32);

// ------------------------------------------------------------------------------------------------ conv -> norm -> BiLSTM stack
constexpr int ENC_MAX_LAYERS = 3;

// One encoder as data.  Layer 0 reads cin0 channels stored cp0 wide in its grid, later layers 512.  A conv of `taps` taps
// (odd, <= 2 EPADR + 1) reads grid rows k + EPADR - (taps - 1) / 2 for tap k.  The three extra regions are the MelEncoder's
// (0 bytes for the text encoder); every region is rounded to 256 bytes, so a 0-byte region moves no offset.
struct EncStackDesc {
    const char* name;                      // prefix of the CUDA runtime error message
    int layers, taps, cin0, cp0;
    size_t inv_n_bytes;                    // saved, after lens
    size_t hout_bytes_per_token;           // forward scratch, after xproj
    size_t dmean_bytes_per_utt;            // backward scratch, after scale2
    // conv.weight [512, cin, taps] -> split-fp16 tap-major kmajor [taps][512][3 cp] and / or stacked [taps][3 x 512][cin]
    void (*pack_conv)(const float* w, int cin, int cp, __half* kmajor, __half* stacked, cudaStream_t st);
    // dW [taps][512][cp] -> conv.weight.grad [512, cin, taps]
    void (*unpack_conv_grad)(const float* dwk, int cin, int cp, float* dw, cudaStream_t st);
};

// The weights / gradients of FtEncoderWeights / FtMelEncoderWeights (and their Grads) seen through their arrays
struct EncStackWeights {
    const float* const* conv_w; const float* const* conv_b; const float* const* norm_w; const float* const* norm_b;
    const float* const* w_ih; const float* const* w_hh; const float* const* b_ih; const float* const* b_hh;
};
struct EncStackGrads {
    float* const* d_conv_w; float* const* d_conv_b; float* const* d_norm_w; float* const* d_norm_b;
    float* const* d_w_ih; float* const* d_w_hh; float* const* d_b_ih; float* const* d_b_hh;
};
template <class W> EncStackWeights stack_weights(const W& w) { return {w.conv_w, w.conv_b, w.norm_w, w.norm_b, w.w_ih, w.w_hh, w.b_ih, w.b_hh}; }
template <class G> EncStackGrads stack_grads(const G& g) {
    return {g.d_conv_w, g.d_conv_b, g.d_norm_w, g.d_norm_b, g.d_w_ih, g.d_w_hh, g.d_b_ih, g.d_b_hh};
}

// Layout of the saved activations and of the forward or backward scratch for B utterances of L positions
struct EncStack {
    const EncStackDesc* a;
    int B, L; long long rows;              // rows = B * (L + 2 EPADR) grid rows
    const int* lens;                       // the saved copy of the lengths, or null when unmasked
    // saved by the forward pass for the backward pass
    __half* X16[ENC_MAX_LAYERS + 1];       // layer inputs (split fp16 grids [rows, 3 * width]); X16[layers] feeds the BiLSTM
    float* Y32[ENC_MAX_LAYERS];            // conv outputs (fp32 grid)
    float* mean[ENC_MAX_LAYERS]; float* rstd[ENC_MAX_LAYERS];
    __half* hseq[2]; __half* gates[2]; float* cstate[2];
    float* inv_n;
    size_t saved_bytes;
    // forward scratch
    float* xproj; float* hout; __half* wconv16[ENC_MAX_LAYERS]; __half* wih16;
    size_t fwd_bytes;
    // backward scratch
    __half* dG[2]; __half* dY16; float* DX32; float* dwk; float* scale2; float* dmean; __half* wconv16_b; __half* wih16_b;
    size_t bwd_bytes;
};
EncStack enc_stack_plan(const EncStackDesc& a, int B, int L, bool masked, const void* saved, void* scratch, bool bwd);
// Zeroes the saved grids, h and c (pad rows and positions past a row's length must read as zero) and saves a copy of lens
// (masked only).  The caller then writes X16[0] and runs enc_stack_fwd.
int enc_stack_clear(const EncStack& S, const int* lens, cudaStream_t st);
// Convolutions, norms, dropout, input projection and BiLSTM; output (b, l, c) at out[b * out_sb + l * out_sl + c]
int enc_stack_fwd(const EncStack& S, const EncStackWeights& w, float eps, float drop_p, unsigned long long* rng, float* out,
                  long long out_sb, long long out_sl, cudaStream_t st);
// BPTT on d_out (indexed like the forward output) scaled by S.scale2, which the caller has computed; all weight gradients and,
// when want_dx, the gradient of X16[0] (x S) in DX32
int enc_stack_bwd(const EncStack& S, const EncStackWeights& w, const EncStackGrads& g, float drop_p, const float* d_out,
                  long long d_sb, long long d_sl, bool want_dx, cudaStream_t st);

}  // namespace ft
