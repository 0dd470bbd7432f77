// Per-lane building blocks of the fused mel front-end (mel_fused.cu): a 1024-point real FFT done by ONE WARP as a
// 512-point complex FFT of the packed signal z[n] = x[2n] + i x[2n+1] in three radix-8 passes (512 = 8*8*8), 16 complex
// values per lane, exchanged through a warp-private shared-memory buffer, followed by the real-input split.
//
//   n = 64 n2 + 8 n1 + n0,  k = k0 + 8 k1 + 64 k2,  W = exp(-2 pi i / 512):
//   pass A: A[k0,n1,n0] = W64^{n1 k0}        sum_{n2} W8^{n2 k0} z[64 n2 + 8 n1 + n0]
//   pass B: B[k0,k1,n0] = W512^{n0(k0+8k1)}  sum_{n1} W8^{n1 k1} A[k0,n1,n0]
//   pass C: Z[k0+8k1+64k2] =                 sum_{n0} W8^{n0 k2} B[k0,k1,n0]
//   split : X[k] = E[k] + W1024^k O[k],  E = (Z[k] + conj Z[512-k])/2,  O = (Z[k] - conj Z[512-k])/(2i),  X[512] = Re Z0 - Im Z0
// Shared-memory layouts are padded so every warp-wide access is bank-conflict free: A at k0*72 + n1*8 + n0, B at
// k0*72 + k1*9 + n0, Z in natural order.  The functions are __host__ __device__ so tests/host/test_mel_fft.cu can run the
// exact device arithmetic lane by lane on the CPU (no GPU in the build container).
#pragma once
#include <cuda_runtime.h>

namespace ft {
namespace melfft {

constexpr int NFFT = 1024, NH = 512, NBINS = 513, XBUF = 576;   // XBUF floats per component (re / im) per warp

struct cf { float x, y; };
__host__ __device__ __forceinline__ cf cadd(cf a, cf b) { return {a.x + b.x, a.y + b.y}; }
__host__ __device__ __forceinline__ cf csub(cf a, cf b) { return {a.x - b.x, a.y - b.y}; }
__host__ __device__ __forceinline__ cf cmul(cf a, cf b) { return {a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x}; }

// in-place 8-point DFT, natural-order output: v[k] = sum_n v[n] exp(-2 pi i n k / 8)
__host__ __device__ __forceinline__ void dft8(cf (&v)[8]) {
    const float r = 0.70710678118654752f;
    // DIF stage 1: pairs (j, j+4), twiddle W8^j on the difference
    cf a0 = cadd(v[0], v[4]), a1 = cadd(v[1], v[5]), a2 = cadd(v[2], v[6]), a3 = cadd(v[3], v[7]);
    cf b0 = csub(v[0], v[4]), b1 = csub(v[1], v[5]), b2 = csub(v[2], v[6]), b3 = csub(v[3], v[7]);
    b1 = {r * (b1.x + b1.y), r * (b1.y - b1.x)};          // * (1 - i)/sqrt2
    b2 = {b2.y, -b2.x};                                    // * (-i)
    b3 = {r * (b3.y - b3.x), -r * (b3.x + b3.y)};         // * (-1 - i)/sqrt2
    // stage 2 on each half: pairs (j, j+2), twiddle W4^j
    cf c0 = cadd(a0, a2), c1 = cadd(a1, a3), c2 = csub(a0, a2), c3 = csub(a1, a3);
    c3 = {c3.y, -c3.x};
    cf d0 = cadd(b0, b2), d1 = cadd(b1, b3), d2 = csub(b0, b2), d3 = csub(b1, b3);
    d3 = {d3.y, -d3.x};
    // stage 3 + bit reversal
    v[0] = cadd(c0, c1); v[4] = csub(c0, c1); v[2] = cadd(c2, c3); v[6] = csub(c2, c3);
    v[1] = cadd(d0, d1); v[5] = csub(d0, d1); v[3] = cadd(d2, d3); v[7] = csub(d2, d3);
}

// tw[j] = exp(-2 pi i j / 1024), j = 0..1023 (float2 re/im)
// Pass A for butterfly id (= 8 n1 + n0, 0..63).  `src(m)` returns the windowed sample m of the frame, m in [0, 1024).
template <typename Src>
__host__ __device__ __forceinline__ void pass_a(int id, const Src& src, const float2* tw, float* xr, float* xi) {
    cf v[8];
#pragma unroll
    for (int n2 = 0; n2 < 8; ++n2) {
        const float2 s = src(64 * n2 + id);                  // (x[2n], x[2n+1]) with n = 64 n2 + id
        v[n2] = {s.x, s.y};
    }
    dft8(v);
    const int n1 = id >> 3;
#pragma unroll
    for (int k0 = 0; k0 < 8; ++k0) {
        const float2 w = tw[16 * n1 * k0];                   // W64^{n1 k0}
        const cf o = cmul(v[k0], cf{w.x, w.y});
        xr[k0 * 72 + id] = o.x; xi[k0 * 72 + id] = o.y;
    }
}
// Pass B: load phase / store phase split so one warp-private buffer is reused in place (sync between them)
__host__ __device__ __forceinline__ void pass_b_load(int id, const float* xr, const float* xi, cf (&v)[8]) {
    const int k0 = id >> 3, n0 = id & 7;
#pragma unroll
    for (int n1 = 0; n1 < 8; ++n1) v[n1] = {xr[k0 * 72 + n1 * 8 + n0], xi[k0 * 72 + n1 * 8 + n0]};
}
__host__ __device__ __forceinline__ void pass_b_store(int id, cf (&v)[8], const float2* tw, float* xr, float* xi) {
    const int k0 = id >> 3, n0 = id & 7;
    dft8(v);
#pragma unroll
    for (int k1 = 0; k1 < 8; ++k1) {
        const float2 w = tw[2 * n0 * (k0 + 8 * k1)];         // W512^{n0 (k0 + 8 k1)}
        const cf o = cmul(v[k1], cf{w.x, w.y});
        xr[k0 * 72 + k1 * 9 + n0] = o.x; xi[k0 * 72 + k1 * 9 + n0] = o.y;
    }
}
__host__ __device__ __forceinline__ void pass_c_load(int id, const float* xr, const float* xi, cf (&v)[8]) {
    const int k0 = id >> 3, k1 = id & 7;
#pragma unroll
    for (int n0 = 0; n0 < 8; ++n0) v[n0] = {xr[k0 * 72 + k1 * 9 + n0], xi[k0 * 72 + k1 * 9 + n0]};
}
__host__ __device__ __forceinline__ void pass_c_store(int id, cf (&v)[8], float* xr, float* xi) {
    const int k0 = id >> 3, k1 = id & 7;
    dft8(v);
#pragma unroll
    for (int k2 = 0; k2 < 8; ++k2) { xr[k0 + 8 * k1 + 64 * k2] = v[k2].x; xi[k0 + 8 * k1 + 64 * k2] = v[k2].y; }
}
// real-input split for bin k (0..511): returns X[k] = (re, im)
__host__ __device__ __forceinline__ cf split_bin(int k, const float* zr, const float* zi, const float2* tw) {
    const int kc = (NH - k) & (NH - 1);
    const float ar = zr[k], ai = zi[k], br = zr[kc], bi = -zi[kc];          // Z[k], conj Z[512-k]
    const cf E = {0.5f * (ar + br), 0.5f * (ai + bi)};
    const cf D = {0.5f * (ar - br), 0.5f * (ai - bi)};                      // (Z - conj Z')/2 ; O = D / i = (D.y, -D.x)
    const cf O = {D.y, -D.x};
    const float2 w = tw[k];
    return cadd(E, cmul(O, cf{w.x, w.y}));
}

// Inverse real FFT (istft.cu), the split run backwards: for a half spectrum X[0..512] the 1024-point irfft is
//   z[n] = x[2n] + i x[2n+1] = IDFT512(Z)[n],  Z[k] = (X[k] + conj X[512-k])/2 + i (X[k] - conj X[512-k]) W1024^{-k}/2,
// and IDFT512(Z) = conj(DFT512(conj Z))/512, so pass A..C above run unchanged on conj Z.  Like numpy's irfft, the
// imaginary parts of X[0] and X[512] are ignored (a real signal's DC and Nyquist bins are real).
// inv_pretwiddle returns conj Z[k] for k in [0, 512) from xk = X[k] and xc = X[512-k].
__host__ __device__ __forceinline__ cf inv_pretwiddle(int k, cf xk, cf xc, const float2* tw) {
    if (k == 0) { xk.y = 0.f; xc.y = 0.f; }
    const cf E = {0.5f * (xk.x + xc.x), 0.5f * (xk.y - xc.y)};              // (X[k] + conj X')/2
    const cf D = {0.5f * (xk.x - xc.x), 0.5f * (xk.y + xc.y)};              // (X[k] - conj X')/2
    const float2 w = tw[k];
    const cf O = cmul(D, cf{w.x, -w.y});                                     // * W1024^{-k}
    return {E.x - O.y, -(E.y + O.x)};                                        // conj(E + i O)
}
// read-out after pass C on conj Z (zr / zi in natural order): sample m in [0, 1024) of the irfft
__host__ __device__ __forceinline__ float inv_readout(int m, const float* zr, const float* zi) {
    return (m & 1) ? -zi[m >> 1] * (1.0f / 512.0f) : zr[m >> 1] * (1.0f / 512.0f);
}

}  // namespace melfft

// The utterance a global frame index f belongs to, over int64 prefix sums: frame_offsets[u] <= f < frame_offsets[u + 1].
__device__ __forceinline__ int find_utt(const long long* __restrict__ frame_offsets, int n_utt, long long f) {
    int lo = 0, hi = n_utt;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (__ldg(frame_offsets + mid) <= f) lo = mid; else hi = mid;
    }
    return lo;
}

}  // namespace ft
