// Internal declarations shared by the .cu files of libflowtron_b200.so (not part of the C ABI).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <vector>

namespace ft {

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// error plumbing (api.cu)
int ft_set_error(const char* msg);            // records msg, returns -1
int ft_check_launch(const char* what);        // cudaGetLastError -> ft_set_error
int ft_runtime_error(const char* who);        // records "<who>: CUDA runtime call failed", returns -1
int* ft_status_word();                        // device int written by kernel watchdogs (0 = ok)
void ft_count_launch(int n);

// propagate a failure whose message is already recorded
#define FT_TRY(x) do { if ((x) != 0) return -1; } while (0)
// check a CUDA runtime call; `who` prefixes the recorded message
#define FT_CU(x, who) do { if ((x) != cudaSuccess) return ::ft::ft_runtime_error(who); } while (0)

// Carves a caller-owned workspace into regions, each starting on a 256-byte boundary, in the order they are asked for.
// base == nullptr plans sizes only (off is then the size); regs, when set, records every region for a by-name lookup.
struct Region { const char* name; size_t off, bytes; };
struct Workspace {
    uint8_t* base = nullptr;
    size_t off = 0;
    std::vector<Region>* regs = nullptr;
    size_t take(size_t bytes) {                     // offset of the next region of `bytes`
        const size_t o = off;
        off = (off + bytes + 255) & ~static_cast<size_t>(255);
        return o;
    }
    template <typename T>
    T* get(const char* name, size_t n) {
        const size_t o = take(n * sizeof(T));
        if (regs) regs->push_back({name, o, n * sizeof(T)});
        return base ? reinterpret_cast<T*>(base + o) : nullptr;
    }
    template <typename T> T* get(size_t n) { return get<T>(nullptr, n); }
};

// RAII device-time bracket around a launch (no-op unless ft_timing_enable(1))
struct TimeScope {
    TimeScope(const char* name, long long m, long long n, long long k, cudaStream_t st);
    ~TimeScope();
    cudaStream_t st_; int idx_;
};

enum { FMT_F16 = 0, FMT_BF16 = 1, FMT_TF32 = 2 };

struct GemmArgs {
    int M = 0, N = 0, K = 0;
    const void* A = nullptr; long long lda = 0; int a_fmt = 0; int a_mn = 0;
    const void* B = nullptr; long long ldb = 0; int b_fmt = 0; int b_mn = 0;
    const float* bias = nullptr; const float* bias2 = nullptr;
    int act = 0; int beta = 0; float alpha = 1.0f; const float* alpha_ptr = nullptr;
    const void* aux16 = nullptr; long long ldaux = 0;   // act == 2: fp16 [M,N] saved tanh output
    float* C32 = nullptr; long long ldc32 = 0;
    void* C16 = nullptr; long long ldc16 = 0; int c16_fmt = 0;
};
int launch_gemm(const GemmArgs& g, cudaStream_t st);
// The three roles of launch_gemm on fp16 operands (gemm.cu).  Outputs: fp32 C32 and / or fp16 C16; beta: C32 += the product;
// alpha_ptr: a device scalar the product is multiplied by (the inverse loss scale of a backward; null = 1).
// forward: C[M, N] = A[M, K] B[N, K]^T (+ bias[N] + bias2[N]), act 1 = tanh
int gemm_nt(cudaStream_t st, long long M, int N, int K, const void* A, long long lda, const void* B, long long ldb, float* C32,
            long long ldc32, void* C16 = nullptr, long long ldc16 = 0, const float* bias = nullptr, const float* bias2 = nullptr,
            int act = 0, int beta = 0);
// dgrad: dX[M, Kout] = dY[M, N] W[N, Kout] (W given MN-major); aux16 (fp16 [M, Kout] tanh output) multiplies by 1 - aux^2
int gemm_dgrad(cudaStream_t st, long long M, int Kout, int N, const void* dY, long long lddy, const void* W, long long ldw,
               float* C32, long long ldc32, void* C16 = nullptr, long long ldc16 = 0, int beta = 0, const float* alpha_ptr = nullptr,
               const void* aux16 = nullptr, long long ldaux = 0);
// wgrad: dW[N, K] = dY[R, N]^T X[R, K] (both MN-major views of the natural tensors), dW row pitch ldw; a sum over R <= 0
// rows sets dW to 0 (or, with beta, leaves it)
int gemm_wgrad(cudaStream_t st, int N, int K, long long R, const void* dY, long long lddy, const void* X, long long ldx, float* dW,
               long long ldw, const float* alpha_ptr, int beta = 0);
void set_gemm_pair_mode(int mode);   // 0 never, 1 big contractions only (default), 2 whenever eligible
int make_tmap_2d(CUtensorMap* out, const void* ptr, int fmt, long long rows, long long cols, long long ld,
                 int box_cols, int box_rows, int swizzle_bytes = 128);   // 128 or 64: the box's inner extent in bytes

void set_lstm_trace(long long* p);
int launch_lstm_fwd(int T, int B, const float* xproj, const void* whh16, const int* lens, void* hseq16, long long ldh,
                    void* gates16, float* cstate, float* h32, long long ldh32, int* flags, cudaStream_t st);
int launch_lstm_fwd_xin(int T, int B, const void* x16, long long ldx, int kx, const void* wih16, const float* b_ih, const float* b_hh,
                        const void* whh16, const int* lens, void* hseq16, long long ldh, void* gates16, float* cstate, float* h32,
                        long long ldh32, int* flags, cudaStream_t st);    // input projection folded into the recurrence (kx <= 128)
int launch_lstm_fwd_chunk(int T, int B, int t0, int t1, const float* xproj, const void* whh16, const int* lens, void* hseq16,
                          long long ldh, void* gates16, float* cstate, int* flags, cudaStream_t st, float* h32 = nullptr,
                          long long ldh32 = 0);
int launch_lstm_bwd_chunk(int T, int B, int t0, int t1, const float* dh_ext, long long ldd, const void* whhT16, const void* gates16,
                          const float* cstate, const int* lens, void* dG16, float* dc_carry, int* flags, float* xchg, cudaStream_t st);
int lstm_bwd_max_clusters(int B);
int launch_lstm_bwd(int T, int B, const float* dh_ext, long long ldd, const void* whhT16, const void* gates16,
                    const float* cstate, const int* lens, void* dG16, int* flags, cudaStream_t st);

int launch_cast(const void* src, int src_fmt, void* dst, int dst_fmt, long long n, cudaStream_t st);   // 0 f16, 1 bf16, 2 f32
int launch_transpose_cast_f16(const float* src, void* dst, int rows, int cols, cudaStream_t st);
int launch_grad_scale(const float* a, long long na, const float* b, long long nb, const float* c, long long nc, float target,
                      float* scale2, cudaStream_t st, const float* d = nullptr, long long nd = 0, const float* e = nullptr,
                      long long ne = 0);   // scale2[0] = S (power of two) from max|a..e|, scale2[1] = 1/S
int launch_prep_mel(const float* mel, const int* lens, int T, int B, int M, int reversed, void* mel_in16, float* mel_flow, cudaStream_t st);
int launch_gate_fwd(const void* d16, long long ldd, int K, const float* wg, const float* bg, long long R, float* gate, cudaStream_t st);
int launch_gate_fwd_f32(const float* h32, long long ldh, int H, const float* c32, long long ldc, int A, const float* wg,
                        const float* bg, long long R, float* gate, cudaStream_t st);
// dd NULL: only dwg / dbg (the params-only kernel variant)
int launch_gate_bwd(const void* d16, long long ldd, int K, const float* wg, const float* dgate, long long R, float* dd,
                    long long lddd, float* dwg, float* dbg, const float* scale, cudaStream_t st);
int launch_affine_fwd(const float* o, const float* mel_flow, const int* lens, int T, int B, int M, int reversed, float* z,
                      float* log_s, cudaStream_t st);
int launch_affine_bwd(const float* dz, const float* dlog_s_ext, const float* o, const float* mel_flow, const int* lens, int T,
                      int B, int M, int reversed, void* do16, float* dmel_flow, const float* scale, cudaStream_t st);
int launch_combine_dmel(const float* dmel_flow, const float* dmel_in, const int* lens, int T, int B, int M, int reversed,
                        float* dmel, const float* inv_scale, cudaStream_t st);
int launch_colsum(const void* src, int fmt, long long ld, long long R, int C, float* out, const float* out_scale, cudaStream_t st);
int launch_nll_reduce(const float* z, const float* const* log_s_list_host, int n_flows, const float* gate,
                      const float* gate_target, const int* lens, int T, int B, int M, float* sums, cudaStream_t st);
int launch_nll_rows(const float* z, const float* const* log_s_list_host, int n_flows, const float* gate,
                    const float* gate_target, const int* lens, int T, int B, int M, float* rows, cudaStream_t st);
int launch_nll_grad(const float* z, const float* gate, const float* gate_target, const int* lens, int T, int B, int M,
                    float sigma, const float* sums, const float* g_nll, const float* g_gate, float* dz, float* dlog_s,
                    float* dgate, cudaStream_t st);

struct AttnFwdArgs {
    int T, B, L, A;
    const float* Q; long long ldq; const float* K; long long ldk; const float* V; long long ldv; const float* v;
    const int* in_lens; const int* out_lens; const float* prior; int reversed; float temperature;
    float* attn; float* logprob; float* p_save; void* ctx16; long long ldc; float* ctx32; long long ldc32;
    int t_begin = 0, t_end = 0;          // query rows of this launch (t_end == 0: all T; t_begin a multiple of 64)
    float* rows = nullptr;               // attn_rows_in_global(L, A): attn_rows_floats(T, B, L) floats of scratch
};
struct AttnBwdArgs {
    int T, B, L, A;
    const float* Q; long long ldq; const float* K; long long ldk; const float* V; long long ldv; const float* v;
    const int* in_lens; const int* out_lens; const float* attn; const float* p_save; float temperature;
    const float* dctx; long long lddc; const float* dattn_ext; const float* dlp_ext;
    const float* scale;      // device [2] = {S, 1/S}: external grads are multiplied by S, dv by 1/S (null = 1)
    float* dQ; long long lddq; float* dK; long long lddk; float* dV; long long lddv; float* dv;
    int t_begin = 0, t_end = 0;          // query rows of this launch (t_end == 0: all T; t_begin a multiple of 64); dK / dV / dv accumulate
    float* rows = nullptr;               // attn_rows_in_global(L, A): attn_rows_floats(T, B, L) floats of scratch
};
// The attention kernels keep a 64-query tile's score / gradient rows in shared memory while they fit (L <= 672 at A = 640);
// past that they keep them in a global area of attn_rows_floats(T, B, L) floats the caller passes as `rows`.
bool attn_rows_in_global(int L, int A);
size_t attn_rows_floats(int T, int B, int L);
int launch_attn_fwd(const AttnFwdArgs& a, cudaStream_t st);
int launch_attn_bwd(const AttnBwdArgs& a, cudaStream_t st);

}  // namespace ft
