// Small bandwidth-bound kernels around the Flowtron AR step: dtype casts, the teacher-forcing shift and
// AR_Back_Step index map (flowtron.py:606-626, 726-729), the gate GEMV (:756-758), the affine coupling and
// its backward (:770-772), column sums for bias gradients, and the NLL / gate-BCE reductions of
// FlowtronLoss (:200-243).  All are HBM-bound: 128-bit accesses, grid-stride loops, grids sized to the SM count.
#include "ptx.cuh"
#include "ft_internal.h"

namespace ft {

static int num_sms() {
    static int n = 0;
    if (!n) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    }
    return n;
}
static inline int grid_for(long long work_items, int threads, int per_sm = 8) {
    long long blocks = (work_items + threads - 1) / threads;
    long long cap = static_cast<long long>(num_sms()) * per_sm;
    return static_cast<int>(blocks < 1 ? 1 : (blocks > cap ? cap : blocks));
}

// ------------------------------------------------------------------------------------------------ casts
template <typename TO>
__device__ __forceinline__ TO cvt_from_float(float x);
template <> __device__ __forceinline__ __half cvt_from_float<__half>(float x) { return __float2half_rn(fminf(fmaxf(x, -65504.f), 65504.f)); }
template <> __device__ __forceinline__ __nv_bfloat16 cvt_from_float<__nv_bfloat16>(float x) { return __float2bfloat16_rn(x); }
template <> __device__ __forceinline__ float cvt_from_float<float>(float x) { return x; }
__device__ __forceinline__ float cvt_to_float(float x) { return x; }
__device__ __forceinline__ float cvt_to_float(__half x) { return __half2float(x); }
__device__ __forceinline__ float cvt_to_float(__nv_bfloat16 x) { return __bfloat162float(x); }

template <typename TI, typename TO>
__global__ void cast_kernel(const TI* __restrict__ src, TO* __restrict__ dst, long long n) {
    const long long stride = static_cast<long long>(gridDim.x) * blockDim.x * 4;
    for (long long i = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) * 4; i < n; i += stride) {
        if (i + 3 < n) {
            TO o[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) o[j] = cvt_from_float<TO>(cvt_to_float(src[i + j]));
#pragma unroll
            for (int j = 0; j < 4; ++j) dst[i + j] = o[j];
        } else {
            for (long long j = i; j < n; ++j) dst[j] = cvt_from_float<TO>(cvt_to_float(src[j]));
        }
    }
}

// dst[c, r] = src[r, c]  (fp32 -> fp16), used for W_hh^T
__global__ void transpose_cast_f16_kernel(const float* __restrict__ src, __half* __restrict__ dst, int rows, int cols) {
    __shared__ float tile[32][33];
    const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int r = r0 + i, c = c0 + threadIdx.x;
        tile[i][threadIdx.x] = (r < rows && c < cols) ? src[static_cast<long long>(r) * cols + c] : 0.f;
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int c = c0 + i, r = r0 + threadIdx.x;
        if (c < cols && r < rows) dst[static_cast<long long>(c) * rows + r] = __float2half_rn(tile[threadIdx.x][i]);
    }
}

int launch_cast(const void* src, int src_fmt, void* dst, int dst_fmt, long long n, cudaStream_t st) {
    // formats: 0 f16, 1 bf16, 2 f32
    if (n <= 0) return 0;
    const int th = 256, g = grid_for((n + 3) / 4, th);
    if (src_fmt == 2 && dst_fmt == 0) cast_kernel<float, __half><<<g, th, 0, st>>>(static_cast<const float*>(src), static_cast<__half*>(dst), n);
    else if (src_fmt == 2 && dst_fmt == 1) cast_kernel<float, __nv_bfloat16><<<g, th, 0, st>>>(static_cast<const float*>(src), static_cast<__nv_bfloat16*>(dst), n);
    else if (src_fmt == 0 && dst_fmt == 1) cast_kernel<__half, __nv_bfloat16><<<g, th, 0, st>>>(static_cast<const __half*>(src), static_cast<__nv_bfloat16*>(dst), n);
    else if (src_fmt == 0 && dst_fmt == 2) cast_kernel<__half, float><<<g, th, 0, st>>>(static_cast<const __half*>(src), static_cast<float*>(dst), n);
    else if (src_fmt == 1 && dst_fmt == 2) cast_kernel<__nv_bfloat16, float><<<g, th, 0, st>>>(static_cast<const __nv_bfloat16*>(src), static_cast<float*>(dst), n);
    else return ft_set_error("cast: unsupported format pair");
    ft_count_launch(1);
    return ft_check_launch("cast_kernel");
}

int launch_transpose_cast_f16(const float* src, void* dst, int rows, int cols, cudaStream_t st) {
    dim3 grid((cols + 31) / 32, (rows + 31) / 32), block(32, 8);
    transpose_cast_f16_kernel<<<grid, block, 0, st>>>(src, static_cast<__half*>(dst), rows, cols);
    ft_count_launch(1);
    return ft_check_launch("transpose_cast_f16_kernel");
}

// ------------------------------------------------------------------------------------------------ backward loss scale
// Backward tensor-core operands are fp16 (11-bit significand).  Every backward op is linear in the incoming
// gradient, so the flow's backward runs on S * grad with S a power of two chosen on the device from the
// incoming gradients (max|.| -> `target`), and every result leaving the flow is multiplied by 1/S.  This is the
// reference's own fp16 recipe (train.py:254 GradScaler) applied per flow and without host involvement.
__global__ void absmax_kernel(const float* __restrict__ a, long long na, const float* __restrict__ b, long long nb,
                              const float* __restrict__ c, long long nc, unsigned int* __restrict__ out) {
    float m = 0.f;
    const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
    const long long i0 = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (a) for (long long i = i0; i < na; i += stride) m = fmaxf(m, fabsf(a[i]));
    if (b) for (long long i = i0; i < nb; i += stride) m = fmaxf(m, fabsf(b[i]));
    if (c) for (long long i = i0; i < nc; i += stride) m = fmaxf(m, fabsf(c[i]));
#pragma unroll
    for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0 && m > 0.f && isfinite(m)) atomicMax(out, __float_as_uint(m));   // non-negative floats order as uints
}
__global__ void scale_finalize_kernel(const unsigned int* __restrict__ mx, float target, float* __restrict__ scale2) {
    const float m = __uint_as_float(mx[0]);
    float s = 1.f;
    if (m > 0.f) {
        int e = static_cast<int>(floorf(log2f(target / m)));
        e = e < -60 ? -60 : (e > 60 ? 60 : e);
        s = exp2f(static_cast<float>(e));
    }
    scale2[0] = s;
    scale2[1] = 1.f / s;
}
int launch_grad_scale(const float* a, long long na, const float* b, long long nb, const float* c, long long nc, float target,
                      float* scale2, cudaStream_t st, const float* d, long long nd, const float* e, long long ne) {
    unsigned int* mx = reinterpret_cast<unsigned int*>(scale2 + 2);
    FT_CU(cudaMemsetAsync(mx, 0, sizeof(unsigned int), st), "grad_scale");
    long long n = na > nb ? na : nb;
    n = n > nc ? n : nc;
    if (n > 0) absmax_kernel<<<grid_for(n, 256, 4), 256, 0, st>>>(a, na, b, nb, c, nc, mx);
    // the attention-side external gradients (CTC loss path: d_attn, d_attn_logprob) are multiplied by the same S inside
    // attn_bwd and their products are cast to fp16 too, so they take part in choosing S
    const long long n2 = nd > ne ? nd : ne;
    if (n2 > 0 && (d || e)) absmax_kernel<<<grid_for(n2, 256, 4), 256, 0, st>>>(d, d ? nd : 0, e, e ? ne : 0, nullptr, 0, mx);
    scale_finalize_kernel<<<1, 1, 0, st>>>(mx, target, scale2);
    ft_count_launch(3);
    return ft_check_launch("grad_scale");
}

// ------------------------------------------------------------------------------------------------ mel prep
// mel [T,B,M] fp32 (natural time).  Flow time q maps to natural r_b(q) when reversed.
//   mel_in16[q,b,:]  = (q == 0) ? 0 : mel[src(q-1), b, :]      (teacher-forcing shift, fp16 GEMM operand)
//   mel_flow[q,b,:]  = mel[src(q), b, :]                        (fp32, only written when reversed)
__global__ void prep_mel_kernel(const float* __restrict__ mel, const int* __restrict__ lens, int T, int B, int M,
                                int reversed, __half* __restrict__ mel_in16, float* __restrict__ mel_flow) {
    const long long n = static_cast<long long>(T) * B * M;
    for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int m = static_cast<int>(i % M);
        const long long rb = i / M;
        const int b = static_cast<int>(rb % B), q = static_cast<int>(rb / B);
        const int len = lens ? lens[b] : T;
        float xin = 0.f;
        if (q > 0) {
            const int s = reversed ? back_index(q - 1, len, T) : q - 1;
            xin = mel[(static_cast<long long>(s) * B + b) * M + m];
        }
        mel_in16[i] = __float2half_rn(xin);
        if (reversed && mel_flow) {
            const int s = back_index(q, len, T);
            mel_flow[i] = mel[(static_cast<long long>(s) * B + b) * M + m];
        }
    }
}
int launch_prep_mel(const float* mel, const int* lens, int T, int B, int M, int reversed, void* mel_in16, float* mel_flow,
                    cudaStream_t st) {
    const long long n = static_cast<long long>(T) * B * M;
    prep_mel_kernel<<<grid_for(n, 256), 256, 0, st>>>(mel, lens, T, B, M, reversed, static_cast<__half*>(mel_in16), mel_flow);
    ft_count_launch(1);
    return ft_check_launch("prep_mel_kernel");
}

// ------------------------------------------------------------------------------------------------ gate GEMV
// gate[r] = d16[r,:] . wg + bg   (one warp per row)
__global__ void gate_fwd_kernel(const __half* __restrict__ d16, long long ldd, int K, const float* __restrict__ wg,
                                const float* __restrict__ bg, long long R, float* __restrict__ gate) {
    const int lane = threadIdx.x & 31;
    const long long w0 = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const long long nw = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
    for (long long r = w0; r < R; r += nw) {
        const __half* row = d16 + r * ldd;
        float s = 0.f;
        for (int k = lane * 8; k < K; k += 256) {
            const uint4 pk = *reinterpret_cast<const uint4*>(row + k);
            const __half2* h = reinterpret_cast<const __half2*>(&pk);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float2 f = __half22float2(h[j]);
                s = fmaf(f.x, __ldg(wg + k + 2 * j), s);
                s = fmaf(f.y, __ldg(wg + k + 2 * j + 1), s);
            }
        }
#pragma unroll
        for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) gate[r] = s + bg[0];
    }
}
int launch_gate_fwd(const void* d16, long long ldd, int K, const float* wg, const float* bg, long long R, float* gate,
                    cudaStream_t st) {
    if (K % 8) return ft_set_error("gate: K must be a multiple of 8");
    gate_fwd_kernel<<<grid_for(R * 32, 256), 256, 0, st>>>(static_cast<const __half*>(d16), ldd, K, wg, bg, R, gate);
    ft_count_launch(1);
    return ft_check_launch("gate_fwd_kernel");
}

// fp32-input form: gate[r] = [hA32[r,0:H] ; ctx32[r,0:A]] . wg + bg.  The fp16 copies in d16 carry 2^-11 input rounding per
// element, which over 1664 terms put the gate logits at 1.6e-3 of their range at T=1000 (bar: 1e-3); the fp32 copies of the
// same activations are written off the critical path by the producing kernels.
__global__ void gate_fwd_f32_kernel(const float* __restrict__ h32, long long ldh, int H, const float* __restrict__ c32, long long ldc,
                                    int A, const float* __restrict__ wg, const float* __restrict__ bg, long long R,
                                    float* __restrict__ gate) {
    const int lane = threadIdx.x & 31;
    const long long w0 = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    const long long nw = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
    for (long long r = w0; r < R; r += nw) {
        float s = 0.f;
        const float* a = h32 + r * ldh;
        for (int k = lane * 4; k < H; k += 128) {
            const float4 x = *reinterpret_cast<const float4*>(a + k);
            const float4 w = __ldg(reinterpret_cast<const float4*>(wg + k));
            s = fmaf(x.x, w.x, s); s = fmaf(x.y, w.y, s); s = fmaf(x.z, w.z, s); s = fmaf(x.w, w.w, s);
        }
        const float* c = c32 + r * ldc;
        for (int k = lane * 4; k < A; k += 128) {
            const float4 x = *reinterpret_cast<const float4*>(c + k);
            const float4 w = __ldg(reinterpret_cast<const float4*>(wg + H + k));
            s = fmaf(x.x, w.x, s); s = fmaf(x.y, w.y, s); s = fmaf(x.z, w.z, s); s = fmaf(x.w, w.w, s);
        }
#pragma unroll
        for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) gate[r] = s + bg[0];
    }
}
int launch_gate_fwd_f32(const float* h32, long long ldh, int H, const float* c32, long long ldc, int A, const float* wg,
                        const float* bg, long long R, float* gate, cudaStream_t st) {
    if ((H % 4) || (A % 4) || (ldh % 4) || (ldc % 4)) return ft_set_error("gate: H, A and the row pitches must be multiples of 4");
    gate_fwd_f32_kernel<<<grid_for(R * 32, 256), 256, 0, st>>>(h32, ldh, H, c32, ldc, A, wg, bg, R, gate);
    ft_count_launch(1);
    return ft_check_launch("gate_fwd_f32_kernel");
}

// backward of the gate GEMV: dd[r,:] += dgate[r] * wg ;  dwg[k] += sum_r dgate[r] d[r,k] ;  dbg += sum_r dgate[r]
// kDd = false: the parameter gradients only (a frozen flow step whose gate alone trains); dd is neither read nor written.
template <bool kDd>
__global__ void gate_bwd_kernel(const __half* __restrict__ d16, long long ldd, int K, const float* __restrict__ wg,
                                const float* __restrict__ dgate, long long R, float* __restrict__ dd, long long lddd,
                                float* __restrict__ dwg, float* __restrict__ dbg, const float* __restrict__ scale) {
    const float S = scale ? scale[0] : 1.f;      // dd lives in the loss-scaled domain, dwg / dbg do not
    // A block walks a slab of rows; thread t owns columns t, t+256, ... (<= GB_KJ of them): every row is one coalesced
    // sweep with GB_KJ independent loads in flight per thread (walking the rows per column instead is
    // latency-bound).
    constexpr int GB_KJ = 8;                          // K <= 2048 (checked by the launcher)
    const long long rows_per_block = (R + gridDim.x - 1) / gridDim.x;
    const long long r0 = blockIdx.x * rows_per_block, r1 = min(R, r0 + rows_per_block);
    float acc[GB_KJ], w[GB_KJ];
#pragma unroll
    for (int j = 0; j < GB_KJ; ++j) {
        const int k = threadIdx.x + 256 * j;
        acc[j] = 0.f;
        if (kDd) w[j] = k < K ? S * wg[k] : 0.f;
    }
    float db = 0.f;
    for (long long r = r0; r < r1; ++r) {
        const float g = dgate[r];                     // block-uniform
        if (g == 0.f) continue;                       // padded frames
        db += g;
        const __half* drow = d16 + r * ldd;
        float* ddrow = dd + r * lddd;
#pragma unroll
        for (int j = 0; j < GB_KJ; ++j) {
            const int k = threadIdx.x + 256 * j;
            if (k < K) {
                acc[j] = fmaf(g, __half2float(drow[k]), acc[j]);
                if (kDd) ddrow[k] = fmaf(g, w[j], ddrow[k]);
            }
        }
    }
    if (threadIdx.x == 0 && db != 0.f) atomicAdd(dbg, db);
#pragma unroll
    for (int j = 0; j < GB_KJ; ++j) {
        const int k = threadIdx.x + 256 * j;
        if (k < K && acc[j] != 0.f) atomicAdd(dwg + k, acc[j]);
    }
}
int launch_gate_bwd(const void* d16, long long ldd, int K, const float* wg, const float* dgate, long long R, float* dd,
                    long long lddd, float* dwg, float* dbg, const float* scale, cudaStream_t st) {
    long long gl = (R + 15) / 16, gcap = static_cast<long long>(num_sms()) * 4;
    int g = static_cast<int>(gl > gcap ? gcap : gl);
    if (g < 1) g = 1;
    if (K > 2048) return ft_set_error("gate_bwd: K > 2048 not supported");
    if (dd)
        gate_bwd_kernel<true><<<g, 256, 0, st>>>(static_cast<const __half*>(d16), ldd, K, wg, dgate, R, dd, lddd, dwg, dbg, scale);
    else
        gate_bwd_kernel<false><<<g, 256, 0, st>>>(static_cast<const __half*>(d16), ldd, K, wg, dgate, R, dd, lddd, dwg, dbg, scale);
    ft_count_launch(1);
    return ft_check_launch("gate_bwd_kernel");
}

// ------------------------------------------------------------------------------------------------ affine coupling
// o [R,2M] = (log_s | b) in flow time; mel_flow [R,M] flow-time input.  z is written in natural time:
//   z[src(q), b, :] = exp(log_s[q,b,:]) * mel_flow[q,b,:] + b[q,b,:]   (src = identity unless reversed)
__global__ void affine_fwd_kernel(const float* __restrict__ o, const float* __restrict__ mel_flow, const int* __restrict__ lens,
                                  int T, int B, int M, int reversed, float* __restrict__ z, float* __restrict__ log_s) {
    const long long n = static_cast<long long>(T) * B * M;
    for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int m = static_cast<int>(i % M);
        const long long rb = i / M;
        const int b = static_cast<int>(rb % B), q = static_cast<int>(rb / B);
        const float ls = o[rb * 2 * M + m], bb = o[rb * 2 * M + M + m];
        log_s[i] = ls;
        const float zz = expf(ls) * mel_flow[i] + bb;
        int s = q;
        if (reversed) s = back_index(q, lens ? lens[b] : T, T);
        z[(static_cast<long long>(s) * B + b) * M + m] = zz;
    }
}
int launch_affine_fwd(const float* o, const float* mel_flow, const int* lens, int T, int B, int M, int reversed, float* z,
                      float* log_s, cudaStream_t st) {
    const long long n = static_cast<long long>(T) * B * M;
    affine_fwd_kernel<<<grid_for(n, 256), 256, 0, st>>>(o, mel_flow, lens, T, B, M, reversed, z, log_s);
    ft_count_launch(1);
    return ft_check_launch("affine_fwd_kernel");
}

// backward: dz natural time, dlog_s_ext flow time (may be null).  Writes do16 (bf16 [R,2M]) and dmel_flow [R,M]:
//   dzq = dz[src(q)] ;  d log_s = dlog_s_ext + dzq * mel_flow * exp(log_s) ;  d b = dzq ;  d mel_flow = dzq * exp(log_s)
__global__ void affine_bwd_kernel(const float* __restrict__ dz, const float* __restrict__ dlog_s_ext,
                                  const float* __restrict__ o, const float* __restrict__ mel_flow, const int* __restrict__ lens,
                                  int T, int B, int M, int reversed, __half* __restrict__ do16,
                                  float* __restrict__ dmel_flow, const float* __restrict__ scale) {
    const float S = scale ? scale[0] : 1.f;
    const long long n = static_cast<long long>(T) * B * M;
    for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int m = static_cast<int>(i % M);
        const long long rb = i / M;
        const int b = static_cast<int>(rb % B), q = static_cast<int>(rb / B);
        const int len = lens ? lens[b] : T;
        int s = q;
        if (reversed) s = back_index(q, len, T);
        const float dzq = dz ? S * dz[(static_cast<long long>(s) * B + b) * M + m] : 0.f;
        const float es = expf(o[rb * 2 * M + m]);
        float dls = dzq * mel_flow[i] * es;
        if (dlog_s_ext) dls += S * dlog_s_ext[i];
        do16[rb * 2 * M + m] = cvt_from_float<__half>(dls);
        do16[rb * 2 * M + M + m] = cvt_from_float<__half>(dzq);
        dmel_flow[i] = dzq * es;
    }
}
int launch_affine_bwd(const float* dz, const float* dlog_s_ext, const float* o, const float* mel_flow, const int* lens, int T,
                      int B, int M, int reversed, void* do16, float* dmel_flow, const float* scale, cudaStream_t st) {
    const long long n = static_cast<long long>(T) * B * M;
    affine_bwd_kernel<<<grid_for(n, 256), 256, 0, st>>>(dz, dlog_s_ext, o, mel_flow, lens, T, B, M, reversed,
                                                         static_cast<__half*>(do16), dmel_flow, scale);
    ft_count_launch(1);
    return ft_check_launch("affine_bwd_kernel");
}

// final input gradient of a flow, natural time:
//   dmel[src(q), b, :] = dmel_flow[q,b,:] + (q+1 < T ? dmel_in[q+1,b,:] : 0)      (undo the teacher-forcing shift)
__global__ void combine_dmel_kernel(const float* __restrict__ dmel_flow, const float* __restrict__ dmel_in,
                                    const int* __restrict__ lens, int T, int B, int M, int reversed, float* __restrict__ dmel,
                                    const float* __restrict__ inv_scale) {
    const float iS = inv_scale ? inv_scale[0] : 1.f;
    const long long n = static_cast<long long>(T) * B * M;
    for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int m = static_cast<int>(i % M);
        const long long rb = i / M;
        const int b = static_cast<int>(rb % B), q = static_cast<int>(rb / B);
        float g = dmel_flow[i];
        if (q + 1 < T) g += dmel_in[i + static_cast<long long>(B) * M];
        int s = q;
        if (reversed) s = back_index(q, lens ? lens[b] : T, T);
        dmel[(static_cast<long long>(s) * B + b) * M + m] = g * iS;
    }
}
int launch_combine_dmel(const float* dmel_flow, const float* dmel_in, const int* lens, int T, int B, int M, int reversed,
                        float* dmel, const float* inv_scale, cudaStream_t st) {
    const long long n = static_cast<long long>(T) * B * M;
    combine_dmel_kernel<<<grid_for(n, 256), 256, 0, st>>>(dmel_flow, dmel_in, lens, T, B, M, reversed, dmel, inv_scale);
    ft_count_launch(1);
    return ft_check_launch("combine_dmel_kernel");
}

// ------------------------------------------------------------------------------------------------ column sums
// out[c] (+)= sum_r src[r, c]   (src bf16 or fp32, row pitch ld)
template <typename TI>
__global__ void colsum_kernel(const TI* __restrict__ src, long long ld, long long R, int C, float* __restrict__ out,
                              const float* __restrict__ out_scale) {
    // grid.x tiles columns by 32*? ; grid.y slabs of rows; block (32, 8)
    const int c = blockIdx.x * 32 + threadIdx.x;
    const long long rows_per = (R + gridDim.y - 1) / gridDim.y;
    const long long r0 = blockIdx.y * rows_per, r1 = min(R, r0 + rows_per);
    float s = 0.f;
    if (c < C)
        for (long long r = r0 + threadIdx.y; r < r1; r += blockDim.y) s += cvt_to_float(src[r * ld + c]);
    __shared__ float sm[8][33];
    sm[threadIdx.y][threadIdx.x] = s;
    __syncthreads();
    if (threadIdx.y == 0 && c < C) {
        float t = 0.f;
        for (int i = 0; i < blockDim.y; ++i) t += sm[i][threadIdx.x];
        atomicAdd(out + c, out_scale ? t * out_scale[0] : t);
    }
}
int launch_colsum(const void* src, int fmt, long long ld, long long R, int C, float* out, const float* out_scale, cudaStream_t st) {
    FT_CU(cudaMemsetAsync(out, 0, sizeof(float) * C, st), "colsum");
    long long gyl = (R + 255) / 256;
    int gy = static_cast<int>(gyl > 64 ? 64 : gyl);
    if (gy < 1) gy = 1;
    dim3 grid((C + 31) / 32, gy), block(32, 8);
    if (fmt == 1) colsum_kernel<__nv_bfloat16><<<grid, block, 0, st>>>(static_cast<const __nv_bfloat16*>(src), ld, R, C, out, out_scale);
    else if (fmt == 0) colsum_kernel<__half><<<grid, block, 0, st>>>(static_cast<const __half*>(src), ld, R, C, out, out_scale);
    else if (fmt == 2) colsum_kernel<float><<<grid, block, 0, st>>>(static_cast<const float*>(src), ld, R, C, out, out_scale);
    else return ft_set_error("colsum: unsupported format");
    ft_count_launch(1);
    return ft_check_launch("colsum_kernel");
}

// ------------------------------------------------------------------------------------------------ loss reductions
// FlowtronLoss default branch (flowtron.py:205-243).  sums[0] = sum (z*m)^2, sums[1] = sum_flows sum log_s*m,
// sums[2] = sum m * BCEWithLogits(gate*m, target), sums[3] = n = sum m.   z/log_s: [T,B,M]; gate [T,B]; target [B,T].
constexpr int NLL_MAX_FLOWS = 16;
struct LogSList { const float* p[NLL_MAX_FLOWS]; };      // passed BY VALUE: no device-side pointer table, nothing to upload
__global__ void nll_reduce_kernel(const float* __restrict__ z, const LogSList log_s_list, int n_flows,
                                  const float* __restrict__ gate, const float* __restrict__ gate_target,
                                  const int* __restrict__ lens, int T, int B, int M, float* __restrict__ sums) {
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    const long long n = static_cast<long long>(T) * B * M;
    for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int m = static_cast<int>(i % M);
        const long long rb = i / M;
        const int b = static_cast<int>(rb % B), t = static_cast<int>(rb / B);
        if (t < lens[b]) {
            const float zz = z[i];
            a0 = fmaf(zz, zz, a0);
            for (int f = 0; f < n_flows; ++f) a1 += log_s_list.p[f][i];
            if (m == 0) {
                a3 += 1.f;
                if (gate) {
                    const float x = gate[rb], y = gate_target[static_cast<long long>(b) * T + t];
                    a2 += fmaxf(x, 0.f) - x * y + log1pf(expf(-fabsf(x)));
                }
            }
        }
    }
    __shared__ float sm[4][32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        a0 += __shfl_xor_sync(0xffffffffu, a0, o); a1 += __shfl_xor_sync(0xffffffffu, a1, o);
        a2 += __shfl_xor_sync(0xffffffffu, a2, o); a3 += __shfl_xor_sync(0xffffffffu, a3, o);
    }
    if (lane == 0) { sm[0][warp] = a0; sm[1][warp] = a1; sm[2][warp] = a2; sm[3][warp] = a3; }
    __syncthreads();
    if (warp == 0) {
        const int nw = blockDim.x >> 5;
        for (int k = 0; k < 4; ++k) {
            float v = lane < nw ? sm[k][lane] : 0.f;
#pragma unroll
            for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
            if (lane == 0) atomicAdd(sums + k, v);
        }
    }
}
int launch_nll_reduce(const float* z, const float* const* log_s_list_host, int n_flows, const float* gate,
                      const float* gate_target, const int* lens, int T, int B, int M, float* sums, cudaStream_t st) {
    if (n_flows < 0 || n_flows > NLL_MAX_FLOWS) return ft_set_error("nll_reduce: more than 16 flows not supported");
    FT_CU(cudaMemsetAsync(sums, 0, sizeof(float) * 4, st), "nll");
    LogSList ls;
    for (int f = 0; f < NLL_MAX_FLOWS; ++f) ls.p[f] = f < n_flows ? log_s_list_host[f] : nullptr;
    const long long n = static_cast<long long>(T) * B * M;
    nll_reduce_kernel<<<grid_for(n, 256, 4), 256, 0, st>>>(z, ls, n_flows, gate, gate_target, lens, T, B, M, sums);
    ft_count_launch(1);
    return ft_check_launch("nll_reduce_kernel");
}

// Per-utterance form of the same sums (Flowtron.score).  One CTA per row b; rows[b * 4 + {0, 1, 2, 3}] = sum z^2,
// sum_flows sum log_s, sum BCEWithLogits(gate, target) over the row's n = min(lens[b], T) frames, and n.  Thread i of the
// CTA takes elements i, i + 256, ... of the row's [n, M] block and frames i, i + 256, ... of its gate; the flows are added
// per element in flow order, then the threads' partials in a fixed tree.  Nothing depends on B or on other rows (no
// atomics), so a row's values are bit-identical whatever batch, padding or graph replay it comes from.
constexpr int NLL_ROWS_THREADS = 256;
__global__ void __launch_bounds__(NLL_ROWS_THREADS) nll_rows_kernel(
        const float* __restrict__ z, const LogSList log_s_list, int n_flows, const float* __restrict__ gate,
        const float* __restrict__ gate_target, const int* __restrict__ lens, int T, int B, int M, float* __restrict__ rows) {
    const int b = blockIdx.x;
    const int n = max(0, min(lens[b], T));
    float a0 = 0.f, a1 = 0.f, a2 = 0.f;
    const long long ne = static_cast<long long>(n) * M;
    for (long long j = threadIdx.x; j < ne; j += NLL_ROWS_THREADS) {
        const int t = static_cast<int>(j / M), m = static_cast<int>(j - static_cast<long long>(t) * M);
        const long long i = (static_cast<long long>(t) * B + b) * M + m;
        const float zz = z[i];
        a0 = fmaf(zz, zz, a0);
        float ls = 0.f;
        for (int f = 0; f < n_flows; ++f) ls += log_s_list.p[f][i];
        a1 += ls;
    }
    if (gate)
        for (int t = threadIdx.x; t < n; t += NLL_ROWS_THREADS) {
            const float x = gate[static_cast<long long>(t) * B + b], y = gate_target[static_cast<long long>(b) * T + t];
            a2 += fmaxf(x, 0.f) - x * y + log1pf(expf(-fabsf(x)));
        }
    __shared__ float sm[3][NLL_ROWS_THREADS / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        a0 += __shfl_xor_sync(0xffffffffu, a0, o); a1 += __shfl_xor_sync(0xffffffffu, a1, o);
        a2 += __shfl_xor_sync(0xffffffffu, a2, o);
    }
    if (lane == 0) { sm[0][warp] = a0; sm[1][warp] = a1; sm[2][warp] = a2; }
    __syncthreads();
    if (threadIdx.x < 3) {
        float s = 0.f;
        for (int w = 0; w < NLL_ROWS_THREADS / 32; ++w) s += sm[threadIdx.x][w];
        rows[static_cast<long long>(b) * 4 + threadIdx.x] = s;
    }
    if (threadIdx.x == 3) rows[static_cast<long long>(b) * 4 + 3] = static_cast<float>(n);
}
int launch_nll_rows(const float* z, const float* const* log_s_list_host, int n_flows, const float* gate,
                    const float* gate_target, const int* lens, int T, int B, int M, float* rows, cudaStream_t st) {
    if (n_flows < 0 || n_flows > NLL_MAX_FLOWS) return ft_set_error("ft_nll_rows: more than 16 flows not supported");
    if (T < 1 || B < 1 || M < 1) return ft_set_error("ft_nll_rows: T, B and M must be positive");
    if (!z || !lens || !rows || (n_flows > 0 && !log_s_list_host)) return ft_set_error("ft_nll_rows: NULL argument");
    if (gate && !gate_target) return ft_set_error("ft_nll_rows: gate needs gate_target");
    LogSList ls;
    for (int f = 0; f < NLL_MAX_FLOWS; ++f) {
        ls.p[f] = f < n_flows ? log_s_list_host[f] : nullptr;
        if (f < n_flows && !ls.p[f]) return ft_set_error("ft_nll_rows: NULL log_s pointer");
    }
    nll_rows_kernel<<<B, NLL_ROWS_THREADS, 0, st>>>(z, ls, n_flows, gate, gate_target, lens, T, B, M, rows);
    ft_count_launch(1);
    return ft_check_launch("nll_rows_kernel");
}

// gradients of  loss = g_nll * nll + g_gate * gate_loss  with  nll = (S0/(2 s^2) - S1)/(n M),  gate_loss = S2/n:
//   dz = g_nll * z m /(s^2 n M) ;  dlog_s = -g_nll * m/(n M) (same for every flow) ;  dgate = g_gate * m (sigmoid(x) - y)/n
__global__ void nll_grad_kernel(const float* __restrict__ z, const float* __restrict__ gate, const float* __restrict__ gate_target,
                                const int* __restrict__ lens, int T, int B, int M, float sigma, const float* __restrict__ sums,
                                const float* __restrict__ g_nll, const float* __restrict__ g_gate, float* __restrict__ dz,
                                float* __restrict__ dlog_s, float* __restrict__ dgate) {
    const float n = sums[3];
    const float gn = g_nll ? g_nll[0] : 1.f, gg = g_gate ? g_gate[0] : 1.f;
    const float cz = gn / (sigma * sigma * n * M), cl = -gn / (n * M), cg = gg / n;
    const long long tot = static_cast<long long>(T) * B * M;
    for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < tot;
         i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int m = static_cast<int>(i % M);
        const long long rb = i / M;
        const int b = static_cast<int>(rb % B), t = static_cast<int>(rb / B);
        const bool valid = t < lens[b];
        dz[i] = valid ? cz * z[i] : 0.f;
        dlog_s[i] = valid ? cl : 0.f;
        if (m == 0 && dgate) {
            float g = 0.f;
            if (valid) {
                const float x = gate[rb], y = gate_target[static_cast<long long>(b) * T + t];
                g = cg * (1.f / (1.f + expf(-x)) - y);
            }
            dgate[rb] = g;
        }
    }
}
int launch_nll_grad(const float* z, const float* gate, const float* gate_target, const int* lens, int T, int B, int M,
                    float sigma, const float* sums, const float* g_nll, const float* g_gate, float* dz, float* dlog_s,
                    float* dgate, cudaStream_t st) {
    const long long n = static_cast<long long>(T) * B * M;
    nll_grad_kernel<<<grid_for(n, 256), 256, 0, st>>>(z, gate, gate_target, lens, T, B, M, sigma, sums, g_nll, g_gate, dz,
                                                       dlog_s, dgate);
    ft_count_launch(1);
    return ft_check_launch("nll_grad_kernel");
}

}  // namespace ft
