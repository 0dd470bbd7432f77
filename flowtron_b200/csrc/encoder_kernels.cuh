// Device code shared by the text encoder (encoder.cu) and the mel encoder (mel_encoder.cu): the padded channels-last token
// grid, the split-fp16 operand format, the instance-norm / BiLSTM kernels and their launchers.  The kernels are defined
// once, in encoder.cu; mel_encoder.cu launches the same instantiations.
#pragma once
#include <cuda_fp16.h>
#include "ptx.cuh"
#include "ft_internal.h"

namespace ft {

constexpr int EC = 512, EH = 256, EG = 4 * EH;      // embedding / conv channels, hidden per direction, gate rows
constexpr int EK = 5, EPADR = 2;                    // conv taps, pad rows on either side of an utterance
constexpr int ENC_THREADS = 256, ENC_CLUSTER = 8, ENC_UNITS = EH / ENC_CLUSTER;   // 32 units per CTA

__device__ __forceinline__ void mma16816(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
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

}  // namespace ft
