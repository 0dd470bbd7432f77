// TacotronSTFT.mel_spectrogram (audio_processing.py:117-134, STFT.transform :207-235) for ragged batches.
//
// Reference: reflect-pad, conv1d with a dense windowed DFT basis [1026,1,1024] (2.1 MFLOP/frame, ~20x an FFT),
// magnitude (+ an unused atan2), dense [80,513] mel matmul, log(clamp(.,1e-5)); one utterance at a time on a CPU
// DataLoader worker.  Here, per chunk of frames:
//   frame_kernel  : gather + reflect padding (index math) + window -> frames[chunk, n_fft]     (HBM-bound)
//   cuFFT R2C     : batched n_fft-point real FFT                     -> spec[chunk, n_fft/2+1] (library call)
//   mag_mel_kernel: |X| staged in shared memory, the filterbank applied as the SPARSE operator it is (each
//                   triangular band touches ~13 of 513 bins; 97% of the dense basis is zero), log-clamp, and
//                   coalesced stores into the reference's [80, F] layout.  Magnitudes never go back to HBM.
#include <cufft.h>

#include <map>
#include <mutex>

#include "ptx.cuh"
#include "ft_internal.h"
#include "../../include/flowtron_b200.h"

namespace ft {

// mel_fft.cuh's ft::find_utt reads the offsets through __ldg, which changes these kernels' SASS; this copy keeps them as
// they are.
__device__ __forceinline__ int find_utt_plain(const long long* __restrict__ frame_offsets, int n_utt, long long f) {
    int lo = 0, hi = n_utt;                     // frame_offsets[lo] <= f < frame_offsets[hi]
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (frame_offsets[mid] <= f) lo = mid; else hi = mid;
    }
    return lo;
}

__global__ void frame_kernel(const float* __restrict__ wav, const long long* __restrict__ sample_offsets,
                             const long long* __restrict__ frame_offsets, int n_utt, long long f0, long long nf,
                             const float* __restrict__ window, int n_fft, int hop, float* __restrict__ frames) {
    // one warp per frame, lanes stride over samples (coalesced reads and writes)
    const int lane = threadIdx.x & 31;
    const long long w0 = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const long long nw = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
    for (long long fi = w0; fi < nf; fi += nw) {
        const long long f = f0 + fi;
        const int u = find_utt_plain(frame_offsets, n_utt, f);
        const long long j = f - frame_offsets[u];
        const long long s0 = sample_offsets[u], N = sample_offsets[u + 1] - s0;
        const long long start = j * hop - n_fft / 2;
        float* dst = frames + fi * n_fft;
        for (int n = lane; n < n_fft; n += 32) {
            long long idx = start + n;
            if (idx < 0) idx = -idx;                            // reflect (no edge repeat), audio_processing.py:214-219
            if (idx >= N) idx = 2 * (N - 1) - idx;
            idx = idx < 0 ? 0 : (idx >= N ? N - 1 : idx);       // only reachable for N <= n_fft/2 (torch would raise)
            dst[n] = wav[s0 + idx] * window[n];
        }
    }
}

constexpr int MM_FRAMES = 32;

__global__ void __launch_bounds__(256)
mag_mel_kernel(const float2* __restrict__ spec, const long long* __restrict__ frame_offsets, int n_utt, long long f0,
               long long nf, int n_bins, const float* __restrict__ basis, const int* __restrict__ band_lo,
               const int* __restrict__ band_hi, int n_mel, float clip, float* __restrict__ mel_out) {
    extern __shared__ float smag[];                             // [MM_FRAMES][n_bins | 1]  (odd pitch: conflict-free)
    const int pitch = n_bins | 1;
    const long long fb = static_cast<long long>(blockIdx.x) * MM_FRAMES;
    const long long rem = nf - fb;
    const int nfr = static_cast<int>(rem < MM_FRAMES ? rem : MM_FRAMES);
    for (int i = threadIdx.x; i < nfr * n_bins; i += blockDim.x) {
        const int fr = i / n_bins, k = i % n_bins;
        const float2 c = spec[(fb + fr) * n_bins + k];
        smag[fr * pitch + k] = sqrtf(c.x * c.x + c.y * c.y);
    }
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane >= nfr) return;
    const long long f = f0 + fb + lane;
    const int u = find_utt_plain(frame_offsets, n_utt, f);
    const long long Fu = frame_offsets[u + 1] - frame_offsets[u], j = f - frame_offsets[u];
    float* out = mel_out + frame_offsets[u] * n_mel + j;       // per-utterance [n_mel, Fu] block
    const float* mg = smag + lane * pitch;
    for (int m = warp; m < n_mel; m += blockDim.x / 32) {
        const int lo = band_lo[m], hi = band_hi[m];
        const float* bm = basis + static_cast<long long>(m) * n_bins;
        float s = 0.f;
        for (int k = lo; k < hi; ++k) s = fmaf(__ldg(bm + k), mg[k], s);
        out[static_cast<long long>(m) * Fu] = logf(fmaxf(s, clip));
    }
}

static std::map<long long, cufftHandle> g_plans;
static std::mutex g_plan_mu;

static int get_plan(int n_fft, long long batch, cufftHandle* out) {
    std::lock_guard<std::mutex> lk(g_plan_mu);
    const long long key = (static_cast<long long>(n_fft) << 40) | batch;
    auto it = g_plans.find(key);
    if (it != g_plans.end()) { *out = it->second; return 0; }
    cufftHandle h;
    int n[1] = {n_fft};
    if (cufftPlanMany(&h, 1, n, nullptr, 1, n_fft, nullptr, 1, n_fft / 2 + 1, CUFFT_R2C, static_cast<int>(batch)) != CUFFT_SUCCESS)
        return ft_set_error("cufftPlanMany failed");
    g_plans[key] = h;
    *out = h;
    return 0;
}

}  // namespace ft

extern "C" {

size_t ft_mel_scratch_bytes(int n_fft, long long chunk_frames) {
    return static_cast<size_t>(chunk_frames) * (static_cast<size_t>(n_fft) * 4 + static_cast<size_t>(n_fft / 2 + 1) * 8) + 512;
}

int ft_mel_spectrogram(const float* wav, const long long* sample_offsets, const long long* frame_offsets, int n_utt,
                       long long total_frames, const float* window, const float* mel_basis, const int* band_lo,
                       const int* band_hi, int n_mel, int n_fft, int hop, float clip, float* mel_out, void* scratch,
                       long long chunk_frames, void* stream) {
    using namespace ft;
    if (!wav || !sample_offsets || !frame_offsets || !window || !mel_basis || !band_lo || !band_hi || !mel_out || !scratch)
        return ft_set_error("ft_mel_spectrogram: NULL argument");
    if (n_fft % 2 || n_fft > 4096 || chunk_frames <= 0) return ft_set_error("ft_mel_spectrogram: bad n_fft / chunk");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int n_bins = n_fft / 2 + 1;
    Workspace ws; ws.base = static_cast<uint8_t*>(scratch);
    float* frames = ws.get<float>(static_cast<size_t>(chunk_frames) * n_fft);
    float2* spec = ws.get<float2>(static_cast<size_t>(chunk_frames) * n_bins);
    int dev = 0, sms = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const size_t smem = sizeof(float) * MM_FRAMES * (n_bins | 1);
    cudaFuncSetAttribute(mag_mel_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    for (long long f0 = 0; f0 < total_frames; f0 += chunk_frames) {
        const long long nf = total_frames - f0 < chunk_frames ? total_frames - f0 : chunk_frames;
        {
            TimeScope ts("mel_frame", nf, n_fft, 0, st);
            long long blocks = (nf * 32 + 255) / 256;
            const long long cap = static_cast<long long>(sms) * 16;
            frame_kernel<<<static_cast<int>(blocks > cap ? cap : blocks), 256, 0, st>>>(wav, sample_offsets, frame_offsets, n_utt, f0,
                                                                                         nf, window, n_fft, hop, frames);
            ft_count_launch(1);
            if (ft_check_launch("frame_kernel")) return -1;
        }
        cufftHandle plan;
        if (get_plan(n_fft, nf, &plan)) return -1;
        if (cufftSetStream(plan, st) != CUFFT_SUCCESS) return ft_set_error("cufftSetStream failed");
        {
            TimeScope ts("mel_cufft", nf, n_fft, 0, st);
            if (cufftExecR2C(plan, frames, reinterpret_cast<cufftComplex*>(spec)) != CUFFT_SUCCESS) return ft_set_error("cufftExecR2C failed");
        }
        {
            TimeScope ts("mel_magmel", nf, n_bins, n_mel, st);
            mag_mel_kernel<<<static_cast<int>((nf + MM_FRAMES - 1) / MM_FRAMES), 256, smem, st>>>(
                spec, frame_offsets, n_utt, f0, nf, n_bins, mel_basis, band_lo, band_hi, n_mel, clip, mel_out);
            ft_count_launch(1);
            if (ft_check_launch("mag_mel_kernel")) return -1;
        }
    }
    return 0;
}

}  // extern "C"
