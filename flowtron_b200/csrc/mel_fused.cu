// Fused mel front-end for n_fft = 1024 (TacotronSTFT.mel_spectrogram, audio_processing.py:117-134; STFT.transform
// :207-235): ONE kernel reads the waveform once and writes the log-mel spectrogram once.
//
//   reflect padding + window (index math on the load) -> 1024-point real FFT inside one warp (mel_fft.cuh: three radix-8
//   passes over a warp-private shared-memory buffer) -> |X| in shared memory -> sparse triangular filterbank (727
//   non-zeros) -> log(max(., clip)) -> a [n_mel][32 frames] tile staged in shared memory -> row-wise coalesced stores
//   into the reference's per-utterance [n_mel, F] layout.
//
// The round-1 pipeline (frame_kernel -> cuFFT R2C -> mag_mel_kernel, mel.cu) wrote and re-read the windowed frames (4 KB)
// and the spectrum (4.1 KB) per frame: 17.7 KB of DRAM traffic against 1,344 algorithmic bytes.  Here the only DRAM
// traffic is the waveform (each sample is used by 4 overlapping frames; the re-reads hit L1/L2 because a CTA owns 32
// consecutive frames) and the output.  Bound: HBM by the task's rule (1,344 B/frame); in practice the fp32 FFT
// (~30 kFLOP/frame) and its shared-memory exchange (~25 KB/frame) are the limiters (DESIGN.md 4.5).
// Waveform formats: f32 in [-1, 1], or int16 PCM scaled by 1/32768 on load (data.py:150 `audio / max_wav_value`).
#include "ft_internal.h"
#include "mel_fft.cuh"
#include "../../include/flowtron_b200.h"

namespace ft {

using namespace melfft;

constexpr int MF_THREADS = 256, MF_WARPS = 8, MF_TILE = 32;     // frames per CTA tile
constexpr int MF_WARP_FLOATS = 2 * XBUF + 520;                  // xr, xi, smag

struct MelFusedParams {
    const void* wav; int wav_fmt;                    // 0 = f32, 1 = s16
    const long long* sample_offsets; const long long* frame_offsets; int n_utt; long long total_frames;
    const float* window; const float* basis; const int* band_lo; const int* band_hi; int n_mel; int hop; float clip;
    float* mel_out;                                  // per-utterance [n_mel, F_u] blocks
    float* mag_out; float* phase_out;                // transform mode: per-utterance [513, F_u] blocks
    const float2* twiddle;                           // [1024] exp(-2 pi i j / 1024)
};

template <int kFmt>
struct FrameSrc {
    const void* wav; long long s0, N, start; const float* window; bool fast;
    __device__ __forceinline__ float ld(long long i) const {
        if (kFmt == 0) return __ldg(static_cast<const float*>(wav) + s0 + i);
        return static_cast<float>(__ldg(static_cast<const short*>(wav) + s0 + i)) * (1.0f / 32768.0f);
    }
    __device__ __forceinline__ float2 operator()(int n) const {
        const int m = 2 * n;
        float a, b;
        if (fast) {                                   // interior frame, even absolute index: one vector load
            if (kFmt == 0) {
                const float2 v = __ldg(reinterpret_cast<const float2*>(static_cast<const float*>(wav) + s0 + start + m));
                a = v.x; b = v.y;
            } else {
                const short2 v = __ldg(reinterpret_cast<const short2*>(static_cast<const short*>(wav) + s0 + start + m));
                a = static_cast<float>(v.x) * (1.0f / 32768.0f); b = static_cast<float>(v.y) * (1.0f / 32768.0f);
            }
        } else {
            long long i0 = start + m, i1 = i0 + 1;
            if (i0 < 0) i0 = -i0;                     // reflect without repeating the edge (F.pad mode='reflect')
            if (i1 < 0) i1 = -i1;
            if (i0 >= N) i0 = 2 * (N - 1) - i0;
            if (i1 >= N) i1 = 2 * (N - 1) - i1;
            i0 = i0 < 0 ? 0 : (i0 >= N ? N - 1 : i0);   // only reachable for N <= 512 (torch raises there)
            i1 = i1 < 0 ? 0 : (i1 >= N ? N - 1 : i1);
            a = ld(i0); b = ld(i1);
        }
        const float2 w = __ldg(reinterpret_cast<const float2*>(window + m));
        return make_float2(a * w.x, b * w.y);
    }
};

// Compiled for MF_OCC CTAs per SM (at most 80 registers): 24 FFT warps per SM rather than 16, because the kernel is
// latency-bound on its shared-memory FFT passes.
constexpr int MF_OCC = 3;

template <int kFmt, bool kTransform>
__global__ void __launch_bounds__(MF_THREADS, MF_OCC)
mel_fused_kernel(MelFusedParams p) {
    extern __shared__ __align__(16) uint8_t smem_raw[];
    float2* stw = reinterpret_cast<float2*>(smem_raw);                       // [1024]
    float* sx = reinterpret_cast<float*>(stw + 1024);                        // [8 warps][MF_WARP_FLOATS]
    float* smel = sx + MF_WARPS * MF_WARP_FLOATS;                            // [n_mel][33]
    long long* sbase = reinterpret_cast<long long*>(smel + ((p.n_mel * 33 + 1) & ~1));   // [32] output offset of (m = 0, frame)
    int* sFu = reinterpret_cast<int*>(sbase + MF_TILE);                      // [32] frames of the frame's utterance (0 = no frame)

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int i = threadIdx.x; i < 1024; i += MF_THREADS) stw[i] = p.twiddle[i];
    __syncthreads();
    float* xr = sx + warp * MF_WARP_FLOATS;
    float* xi = xr + XBUF;
    float* smag = xi + XBUF;

    // transform: total_frames bounds the grid, frame_offsets[n_utt] (planned on the device) is the live total
    const long long total = kTransform ? min(p.total_frames, __ldg(p.frame_offsets + p.n_utt)) : p.total_frames;
    const long long n_tiles = (total + MF_TILE - 1) / MF_TILE;
    for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        for (int q = 0; q < MF_TILE / MF_WARPS; ++q) {
            const int fr = warp + q * MF_WARPS;
            const long long f = tile * MF_TILE + fr;
            if (f >= total) { if (lane == 0) sFu[fr] = 0; continue; }      // warp-uniform
            const int u = find_utt(p.frame_offsets, p.n_utt, f);
            const long long fo = __ldg(p.frame_offsets + u);
            const int Fu = static_cast<int>(__ldg(p.frame_offsets + u + 1) - fo);
            const long long j = f - fo;
            FrameSrc<kFmt> src;
            src.wav = p.wav; src.window = p.window;
            src.s0 = __ldg(p.sample_offsets + u);
            src.N = __ldg(p.sample_offsets + u + 1) - src.s0;
            src.start = j * p.hop - NFFT / 2;
            src.fast = src.start >= 0 && src.start + NFFT <= src.N && (((src.s0 + src.start) & 1) == 0);
            if (lane == 0) { sbase[fr] = kTransform ? fo * NBINS + j : fo * p.n_mel + j; sFu[fr] = Fu; }

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
            __syncwarp();
            if (kTransform) {
                float* mo = p.mag_out + fo * NBINS + j;
                float* po = p.phase_out + fo * NBINS + j;
                for (int k = lane; k < NH; k += 32) {
                    const cf X = split_bin(k, xr, xi, stw);
                    mo[static_cast<long long>(k) * Fu] = sqrtf(X.x * X.x + X.y * X.y);
                    po[static_cast<long long>(k) * Fu] = atan2f(X.y, X.x);
                }
                if (lane == 0) {
                    const float x512 = xr[0] - xi[0];
                    mo[static_cast<long long>(NH) * Fu] = fabsf(x512);
                    po[static_cast<long long>(NH) * Fu] = atan2f(0.f, x512);
                }
                __syncwarp();
                continue;
            }
            for (int k = lane; k < NH; k += 32) {
                const cf X = split_bin(k, xr, xi, stw);
                smag[k] = sqrtf(X.x * X.x + X.y * X.y);
            }
            if (lane == 0) smag[NH] = fabsf(xr[0] - xi[0]);
            __syncwarp();
            for (int m = lane; m < p.n_mel; m += 32) {
                const int lo = __ldg(p.band_lo + m), hi = __ldg(p.band_hi + m);
                const float* bm = p.basis + static_cast<long long>(m) * NBINS;
                float s = 0.f;
                for (int k = lo; k < hi; ++k) s = fmaf(__ldg(bm + k), smag[k], s);
                smel[m * 33 + fr] = logf(fmaxf(s, p.clip));
            }
            __syncwarp();
        }
        if (kTransform) continue;
        __syncthreads();
        // tile store: thread -> (frame = tid % 32, band = tid / 32 + 8 i): 32 consecutive frames = one 128-byte row segment
        {
            const int fr = threadIdx.x & 31;
            const int Fu = sFu[fr];
            if (Fu > 0) {
                float* dst = p.mel_out + sbase[fr];
                for (int m = threadIdx.x >> 5; m < p.n_mel; m += MF_WARPS) dst[static_cast<long long>(m) * Fu] = smel[m * 33 + fr];
            }
        }
        __syncthreads();
    }
}

static float2* g_twiddle = nullptr;       // device table, built once per process (first call; NOT on the caller's stream)
static int ensure_twiddle() {
    if (g_twiddle) return 0;
    float2 h[1024];
    for (int j = 0; j < 1024; ++j) {
        const double a = -2.0 * 3.14159265358979323846 * j / 1024.0;
        h[j] = make_float2(static_cast<float>(cos(a)), static_cast<float>(sin(a)));
    }
    if (cudaMalloc(&g_twiddle, sizeof(h)) != cudaSuccess) return ft_set_error("mel_fused: cudaMalloc(twiddle) failed");
    if (cudaMemcpy(g_twiddle, h, sizeof(h), cudaMemcpyHostToDevice) != cudaSuccess) return ft_set_error("mel_fused: twiddle upload failed");
    return 0;
}

template <int kFmt, bool kTransform>
static int launch_mel_fused(MelFusedParams& p, cudaStream_t st) {
    const size_t smem = 1024 * 8 + sizeof(float) * MF_WARPS * MF_WARP_FLOATS +
                        sizeof(float) * ((p.n_mel * 33 + 1) & ~1) + MF_TILE * 8 + MF_TILE * 4 + 16;
    auto fn = mel_fused_kernel<kFmt, kTransform>;
    cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    int dev = 0, sms = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const long long n_tiles = (p.total_frames + MF_TILE - 1) / MF_TILE;
    const long long cap = static_cast<long long>(sms) * MF_OCC;        // persistent: MF_OCC CTAs per SM
    const int grid = static_cast<int>(n_tiles < cap ? n_tiles : cap);
    TimeScope ts(kTransform ? "stft_fused" : "mel_fused", p.total_frames, NFFT, p.n_mel, st);
    fn<<<grid, MF_THREADS, smem, st>>>(p);
    ft_count_launch(1);
    return ft_check_launch("mel_fused_kernel");
}

}  // namespace ft

extern "C" {

int ft_mel_spectrogram_fused(const void* wav, int wav_fmt, const long long* sample_offsets, const long long* frame_offsets,
                             int n_utt, long long total_frames, const float* window, const float* mel_basis, const int* band_lo,
                             const int* band_hi, int n_mel, int n_fft, int hop, float clip, float* mel_out, void* stream) {
    using namespace ft;
    if (!wav || !sample_offsets || !frame_offsets || !window || !mel_basis || !band_lo || !band_hi || !mel_out)
        return ft_set_error("ft_mel_spectrogram_fused: NULL argument");
    if (n_fft != 1024) return ft_set_error("ft_mel_spectrogram_fused: n_fft must be 1024 (use ft_mel_spectrogram otherwise)");
    if (n_mel <= 0 || n_mel > 256 || hop <= 0) return ft_set_error("ft_mel_spectrogram_fused: bad n_mel / hop");
    if (wav_fmt != 0 && wav_fmt != 1) return ft_set_error("ft_mel_spectrogram_fused: wav_fmt must be 0 (f32) or 1 (s16)");
    if (total_frames <= 0 || n_utt <= 0) return 0;
    if (ensure_twiddle()) return -1;
    MelFusedParams p;
    p.wav = wav; p.wav_fmt = wav_fmt; p.sample_offsets = sample_offsets; p.frame_offsets = frame_offsets; p.n_utt = n_utt;
    p.total_frames = total_frames; p.window = window; p.basis = mel_basis; p.band_lo = band_lo; p.band_hi = band_hi;
    p.n_mel = n_mel; p.hop = hop; p.clip = clip; p.mel_out = mel_out; p.mag_out = nullptr; p.phase_out = nullptr; p.twiddle = g_twiddle;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    return wav_fmt == 0 ? launch_mel_fused<0, false>(p, st) : launch_mel_fused<1, false>(p, st);
}

int ft_stft_transform(const float* wav, const long long* sample_offsets, const long long* frame_offsets, int n_utt,
                      long long total_frames, const float* window, int n_fft, int hop, float* magnitude, float* phase,
                      void* stream) {
    using namespace ft;
    if (!wav || !sample_offsets || !frame_offsets || !window || !magnitude || !phase) return ft_set_error("ft_stft_transform: NULL argument");
    if (n_fft != 1024) return ft_set_error("ft_stft_transform: n_fft must be 1024");
    if (total_frames <= 0 || n_utt <= 0) return 0;
    if (ensure_twiddle()) return -1;
    MelFusedParams p;
    p.wav = wav; p.wav_fmt = 0; p.sample_offsets = sample_offsets; p.frame_offsets = frame_offsets; p.n_utt = n_utt;
    p.total_frames = total_frames; p.window = window; p.basis = nullptr; p.band_lo = nullptr; p.band_hi = nullptr;
    p.n_mel = 0; p.hop = hop; p.clip = 0.f; p.mel_out = nullptr; p.mag_out = magnitude; p.phase_out = phase; p.twiddle = g_twiddle;
    return launch_mel_fused<0, true>(p, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
