// Inverse STFT for n_fft = 1024 (STFT.inverse, audio_processing.py:237-265), optionally with the Denoiser's bias
// subtraction (tacotron2/waveglow/denoiser.py) folded into the spectrum load.  ONE kernel:
//
//   per frame: X[k] = m_k (cos phi_k, sin phi_k), m_k = max(m_k - strength * bias[k], 0) when a bias is given ->
//   1024-point irfft inside one warp (mel_fft.cuh: pre-twiddle into conj Z, the forward passes A..C, read-out) ->
//   times the analysis window -> overlap-add at `hop` -> divided by the window's sum-square envelope where it exceeds
//   FLT_MIN (librosa's window_sumsquare / tiny rule) -> 512 samples dropped at each end, (F_u - 1) * hop samples out.
//
// The reference's inverse basis is pinv(scale * fourier_basis) * window, i.e. irfft(.) * window / scale, and its final
// `* filter_length / hop` cancels that scale, so neither appears here.
//
// Work split: a CTA owns TILE_SAMPLES / hop consecutive packed frames; frame j of utterance u owns output block j
// (samples [j hop, (j + 1) hop) of the trimmed signal, the last frame owns none).  Block j overlaps frames
// [j - n/2 + 1, j + n/2] (n = 1024 / hop), so a tile of T blocks recomputes n - 1 halo frames.  The 8 warps transform
// 8 frames at a time into their private buffers; then every thread adds those frames' contributions, in ascending frame
// order, to the samples it owns in a shared-memory accumulator.  Each output sample is therefore summed in an order that
// depends only on utterance-local frame indices: no atomics, and a ragged batch gives bit-identical rows to B = 1 runs.
#include <cfloat>
#include "ft_internal.h"
#include "mel_fft.cuh"
#include "../../include/flowtron_b200.h"

namespace ft {

using namespace melfft;

constexpr int IS_THREADS = 256, IS_WARPS = 8, IS_TILE_SAMPLES = 8192;
constexpr int IS_WARP_FLOATS = 2 * XBUF;

struct IstftParams {
    const float* mag; const float* phase;                // per-utterance [513, F_u] blocks at frame_offsets[u] * 513
    const long long* frame_offsets; const long long* out_offsets; int n_utt; long long total_frames;
    const float* window; int hop;
    const float* bias; float strength;                   // bias == nullptr: plain inverse
    float* out;
};

// pass A source: conj Z[n] of one frame, built from the spectrum in global memory
struct SpecSrc {
    const float* mag; const float* ph; const float* bias; float strength; int Fu; const float2* tw;
    __device__ __forceinline__ cf bin(int k) const {
        const long long o = static_cast<long long>(k) * Fu;
        float m = __ldg(mag + o);
        if (bias) m = fmaxf(__fsub_rn(m, __fmul_rn(__ldg(bias + k), strength)), 0.f);
        float s, c;
        sincosf(__ldg(ph + o), &s, &c);
        return {__fmul_rn(m, c), __fmul_rn(m, s)};
    }
    __device__ __forceinline__ float2 operator()(int n) const {
        const cf z = inv_pretwiddle(n, bin(n), bin(NH - n), tw);
        return make_float2(z.x, z.y);
    }
};

__global__ void __launch_bounds__(IS_THREADS, 2)
istft_kernel(IstftParams p) {
    extern __shared__ __align__(16) uint8_t smem_raw[];
    float2* stw = reinterpret_cast<float2*>(smem_raw);                    // [1024] exp(-2 pi i j / 1024)
    float* swin = reinterpret_cast<float*>(stw + NFFT);                   // [1024]
    float* sacc = swin + NFFT;                                            // [IS_TILE_SAMPLES] overlap-add accumulator
    float* sx = sacc + IS_TILE_SAMPLES;                                   // [8 warps][IS_WARP_FLOATS]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int i = threadIdx.x; i < NFFT; i += IS_THREADS) {
        double s, c;
        sincospi(-2.0 * i / NFFT, &s, &c);
        stw[i] = make_float2(static_cast<float>(c), static_cast<float>(s));
        swin[i] = __ldg(p.window + i);
    }
    for (int i = threadIdx.x; i < IS_TILE_SAMPLES; i += IS_THREADS) sacc[i] = 0.f;
    __syncthreads();
    float* xr = sx + warp * IS_WARP_FLOATS;
    float* xi = xr + XBUF;

    const int hop = p.hop, n_ov = NFFT / hop, half = n_ov / 2;
    const int tile_frames = IS_TILE_SAMPLES / hop;
    const long long total = min(p.total_frames, __ldg(p.frame_offsets + p.n_utt));   // the grid covers the host's bound
    const long long n_tiles = (total + tile_frames - 1) / tile_frames;
    for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const long long t_end = min(total, (tile + 1) * tile_frames);
        for (long long f = tile * tile_frames; f < t_end;) {            // one segment per utterance in the tile
            const int u = find_utt(p.frame_offsets, p.n_utt, f);
            const long long fo = __ldg(p.frame_offsets + u);
            const int Fu = static_cast<int>(__ldg(p.frame_offsets + u + 1) - fo);
            const long long seg_end = min(t_end, fo + Fu);
            const int j0 = static_cast<int>(f - fo);
            const int jend = static_cast<int>(min(seg_end - fo, static_cast<long long>(Fu - 1)));   // blocks [j0, jend)
            f = seg_end;
            if (jend <= j0) continue;
            const int i_lo = max(0, j0 - half + 1), i_hi = min(Fu - 1, jend - 1 + half);       // frames, inclusive
            const int n_samp = (jend - j0) * hop;
            const int pos0 = j0 * hop + NFFT / 2;                        // untrimmed position of the segment's first sample
            const float* mag = p.mag + fo * NBINS;
            const float* ph = p.phase + fo * NBINS;
            for (int ib = i_lo; ib <= i_hi; ib += IS_WARPS) {
                const int i = ib + warp;
                if (i <= i_hi) {                                         // warp-uniform
                    const SpecSrc src{mag + i, ph + i, p.bias, p.strength, Fu, stw};
                    cf v0[8], v1[8];
                    pass_a(lane, src, stw, xr, xi);
                    pass_a(lane + 32, src, stw, xr, xi);
                    __syncwarp();
                    pass_b_load(lane, xr, xi, v0); pass_b_load(lane + 32, xr, xi, v1);
                    __syncwarp();
                    pass_b_store(lane, v0, stw, xr, xi); pass_b_store(lane + 32, v1, stw, xr, xi);
                    __syncwarp();
                    pass_c_load(lane, xr, xi, v0); pass_c_load(lane + 32, xr, xi, v1);
                    __syncwarp();
                    pass_c_store(lane, v0, xr, xi); pass_c_store(lane + 32, v1, xr, xi);
                }
                __syncthreads();
                const int last = min(i_hi, ib + IS_WARPS - 1);
                for (int s = threadIdx.x; s < n_samp; s += IS_THREADS) {
                    const int pos = pos0 + s;
                    float acc = sacc[s];
                    for (int i2 = ib; i2 <= last; ++i2) {
                        const int m = pos - i2 * hop;
                        if (m >= 0 && m < NFFT) {
                            const float* zr = sx + (i2 - ib) * IS_WARP_FLOATS;
                            acc += inv_readout(m, zr, zr + XBUF) * swin[m];
                        }
                    }
                    sacc[s] = acc;
                }
                __syncthreads();
            }
            float* dst = p.out + __ldg(p.out_offsets + u) + static_cast<long long>(j0) * hop;
            for (int s = threadIdx.x; s < n_samp; s += IS_THREADS) {      // same thread -> sample map as the adds above
                const int pos = pos0 + s, q = pos / hop;
                float env = 0.f;
                for (int i2 = max(0, q - n_ov + 1); i2 <= min(Fu - 1, q); ++i2) {
                    const float w = swin[pos - i2 * hop];
                    env += w * w;
                }
                const float a = sacc[s];
                dst[s] = env > FLT_MIN ? a / env : a;
                sacc[s] = 0.f;
            }
        }
    }
}

// Rows of a padded batch -> the packed layout ft_stft_transform reads, planned on the device.  Block (x, b) sums the
// clamped lengths of rows 0..b-1 for row b's sample and frame offsets, then copies its chunk of row b.
constexpr int PK_THREADS = 256, PK_CHUNK = 8192;

__device__ __forceinline__ long long pk_len(const long long* lengths, int b, long long N) {
    const long long n = __ldg(lengths + b);
    return n <= NFFT / 2 ? 0 : min(n, N);                 // rows up to the reflect padding are empty
}

__global__ void __launch_bounds__(PK_THREADS) stft_pack_kernel(const float* __restrict__ audio, long long N,
                                                               const long long* __restrict__ lengths, int B, int hop,
                                                               float* __restrict__ packed, long long* __restrict__ so,
                                                               long long* __restrict__ fo) {
    __shared__ long long s_red[2][PK_THREADS / 32];
    const int b = blockIdx.y, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    long long s = 0, f = 0;
    for (int j = threadIdx.x; j < b; j += PK_THREADS) {
        const long long n = pk_len(lengths, j, N);
        s += n;
        f += n ? 1 + n / hop : 0;
    }
#pragma unroll
    for (int off = 16; off; off >>= 1) {
        s += __shfl_xor_sync(0xffffffffu, s, off);
        f += __shfl_xor_sync(0xffffffffu, f, off);
    }
    if (lane == 0) { s_red[0][warp] = s; s_red[1][warp] = f; }
    __syncthreads();
    s = 0; f = 0;
#pragma unroll
    for (int w = 0; w < PK_THREADS / 32; ++w) { s += s_red[0][w]; f += s_red[1][w]; }
    const long long n = pk_len(lengths, b, N);
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        so[b] = s; fo[b] = f;
        if (b == B - 1) { so[B] = s + n; fo[B] = f + (n ? 1 + n / hop : 0); }
    }
    const long long c0 = static_cast<long long>(blockIdx.x) * PK_CHUNK, c1 = min(n, c0 + PK_CHUNK);
    const float* src = audio + static_cast<long long>(b) * N;
    for (long long i = c0 + threadIdx.x; i < c1; i += PK_THREADS) packed[s + i] = __ldg(src + i);
}

}  // namespace ft

extern "C" {

int ft_stft_pack_rows(const float* audio, int B, long long N, const long long* lengths, int n_fft, int hop, float* packed,
                      long long* sample_offsets, long long* frame_offsets, void* stream) {
    using namespace ft;
    if (!audio || !lengths || !packed || !sample_offsets || !frame_offsets) return ft_set_error("ft_stft_pack_rows: NULL argument");
    if (n_fft != 1024) return ft_set_error("ft_stft_pack_rows: n_fft must be 1024");
    if (B < 1 || B > 65535 || N < 1 || hop < 1) return ft_set_error("ft_stft_pack_rows: need 1 <= B <= 65535, N >= 1, hop >= 1");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const dim3 grid(static_cast<unsigned>((N + PK_CHUNK - 1) / PK_CHUNK), static_cast<unsigned>(B));
    TimeScope ts("stft_pack", B, N, hop, st);
    stft_pack_kernel<<<grid, PK_THREADS, 0, st>>>(audio, N, lengths, B, hop, packed, sample_offsets, frame_offsets);
    ft_count_launch(1);
    return ft_check_launch("stft_pack_kernel");
}

int ft_stft_inverse(const float* magnitude, const float* phase, const long long* frame_offsets, const long long* out_offsets,
                    int n_utt, long long total_frames, const float* window, int n_fft, int hop, const float* bias,
                    float strength, float* out, void* stream) {
    using namespace ft;
    if (!magnitude || !phase || !frame_offsets || !out_offsets || !window || !out) return ft_set_error("ft_stft_inverse: NULL argument");
    if (n_fft != 1024) return ft_set_error("ft_stft_inverse: n_fft must be 1024");
    if (hop != 128 && hop != 256 && hop != 512) return ft_set_error("ft_stft_inverse: hop must be 128, 256 or 512");
    if (total_frames <= 0 || n_utt <= 0) return 0;
    IstftParams p;
    p.mag = magnitude; p.phase = phase; p.frame_offsets = frame_offsets; p.out_offsets = out_offsets; p.n_utt = n_utt;
    p.total_frames = total_frames; p.window = window; p.hop = hop; p.bias = bias; p.strength = strength; p.out = out;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t smem = sizeof(float) * (2 * NFFT + NFFT + IS_TILE_SAMPLES + IS_WARPS * IS_WARP_FLOATS);
    cudaFuncSetAttribute(istft_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    int dev = 0, sms = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const long long tile_frames = IS_TILE_SAMPLES / hop;
    const long long n_tiles = (total_frames + tile_frames - 1) / tile_frames;
    const long long cap = 2LL * sms;                                     // persistent: 2 CTAs per SM
    const int grid = static_cast<int>(n_tiles < cap ? n_tiles : cap);
    TimeScope ts("stft_inverse", total_frames, NFFT, hop, st);
    istft_kernel<<<grid, IS_THREADS, smem, st>>>(p);
    ft_count_launch(1);
    return ft_check_launch("istft_kernel");
}

}  // extern "C"
