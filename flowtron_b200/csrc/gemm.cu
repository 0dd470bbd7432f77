// Host side of the GEMM (kernel: gemm_kernel.cuh): TMA descriptors, tile / split-K / cluster policy, launch.
#include "gemm_kernel.cuh"

namespace ft {

// ------------------------------------------------------------------------------------------------ host
static PFN_encodeTiled g_encode = nullptr;

int ensure_tma_encoder() {
    if (g_encode) return 0;
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !fn) return ft_set_error("cuTensorMapEncodeTiled entry point unavailable");
    g_encode = reinterpret_cast<PFN_encodeTiled>(fn);
    return 0;
}

PFN_encodeTiled get_tma_encoder() { return ensure_tma_encoder() ? nullptr : g_encode; }

// 2D row-major tensor [rows, cols] (cols contiguous, row pitch ld elements), box {box_cols, box_rows}, SW128 (or SW64).
int make_tmap_2d(CUtensorMap* out, const void* ptr, int fmt, long long rows, long long cols, long long ld,
                 int box_cols, int box_rows, int swizzle_bytes) {
    if (ensure_tma_encoder()) return -1;
    const int elt = (fmt == 2) ? 4 : 2;
    CUtensorMapDataType dt = fmt == 0 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16
                           : fmt == 1 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
    if ((reinterpret_cast<uintptr_t>(ptr) & 15) || ((ld * elt) & 15)) return ft_set_error("TMA operand must be 16-byte aligned with a 16-byte-multiple row pitch");
    if (box_cols * elt != swizzle_bytes || (swizzle_bytes != 128 && swizzle_bytes != 64))
        return ft_set_error("TMA box inner extent must be the swizzle span (128 or 64 bytes)");
    cuuint64_t dims[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
    cuuint64_t strides[1] = {static_cast<cuuint64_t>(ld * elt)};
    cuuint32_t box[2] = {static_cast<cuuint32_t>(box_cols), static_cast<cuuint32_t>(box_rows)};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = g_encode(out, dt, 2, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                          swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return ft_set_error("cuTensorMapEncodeTiled failed");
    return 0;
}

// 0 never (default), 1 big contractions only, 2 whenever eligible.  On the H100 80GB HBM3 (700 W) CTA pairs were slower
// than single-CTA tiles at every training shape they were eligible for (tools/gemm_shapes.py, DESIGN 4.1), so by default
// they are not used; ft_set_gemm_pair_mode keeps them selectable.
static int g_pair_mode = 0;
void set_gemm_pair_mode(int mode) { g_pair_mode = mode; }

// 0: schedule by shape (launch_gemm).  tools/gemm_shapes.py builds private copies with 1 (cooperative only) and 2 (ping-pong
// wherever eligible) to time both schedules on every shape.
#ifndef FT_GEMM_SCHEDULE
#define FT_GEMM_SCHEDULE 0
#endif

extern template const void* gemm_kernel_ptr<FMT_F16, 0>(int, int, int, int);
extern template const void* gemm_kernel_ptr<FMT_F16, 1>(int, int, int, int);
extern template const void* gemm_kernel_ptr<FMT_BF16, 0>(int, int, int, int);
extern template const void* gemm_kernel_ptr<FMT_BF16, 1>(int, int, int, int);
extern template const void* gemm_kernel_ptr<FMT_TF32, 0>(int, int, int, int);

int launch_gemm(const GemmArgs& g, cudaStream_t st) {
    if (g.M <= 0 || g.N <= 0 || g.K <= 0) return 0;
    const bool tf32 = (g.a_fmt == 2);
    if ((g.a_fmt == 2) != (g.b_fmt == 2)) return ft_set_error("gemm: tf32 must be used for both operands");
    if (!tf32 && g.a_fmt != g.b_fmt) return ft_set_error("gemm: both 16-bit operands must have the same format");
    if (tf32 && (g.a_mn || g.b_mn)) return ft_set_error("gemm: MN-major tf32 operands not supported");
    const int elt = tf32 ? 4 : 2, BK = 128 / elt;
    CUtensorMap tmA, tmB;
    GemmParams p;
    p.M = g.M; p.N = g.N; p.K = g.K;
    p.bias = g.bias; p.bias2 = g.bias2; p.act = g.act; p.alpha_ptr = g.alpha_ptr; p.aux16 = static_cast<const __half*>(g.aux16); p.ldaux = g.ldaux; p.beta = g.beta; p.alpha = g.alpha;
    p.C32 = g.C32; p.ldc32 = g.ldc32; p.C16 = g.C16; p.ldc16 = g.ldc16; p.c16_fmt = g.c16_fmt;
    p.status = ft_status_word();
    static int sms = 0;
    if (!sms) { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev); }
    bool wide = (g.N % 256 == 0) || g.N > 1024;
    if (wide && static_cast<long long>((g.N + 255) / 256) * ((g.M + BM - 1) / BM) < sms) wide = false;   // few tiles: prefer more CTAs
    int bn = wide ? 256 : 128;
    int tiles_n = (g.N + bn - 1) / bn;
    const int tiles_m = (g.M + BM - 1) / BM;
    const long long n_tiles_ll = static_cast<long long>(tiles_n) * tiles_m;
    if (n_tiles_ll > 0x7fffffff) return ft_set_error("gemm: too many tiles");
    int n_tiles = static_cast<int>(n_tiles_ll);
    // split-K: long reductions with few output tiles (the dense / projection weight gradients: K = T*B rows, 8-64 tiles)
    // would leave most SMs idle; each K range is reduced by its own CTA and added into a zeroed C32
    const int num_kb_all = (g.K + BK - 1) / BK;
    int splitk = 1;
    const bool splittable = g.C32 && !g.C16 && !g.beta && !g.bias && !g.bias2 && g.act == 0 && (g.N % 4 == 0) &&
                            g.ldc32 == g.N && ((reinterpret_cast<uintptr_t>(g.C32) & 15) == 0);
    if (splittable && n_tiles * 2 <= sms && num_kb_all >= 64) {
        splitk = sms / n_tiles;
        if (splitk > 16) splitk = 16;
        while (splitk > 1 && num_kb_all / splitk < 16) --splitk;
    }
    if (splitk > 1) FT_CU(cudaMemsetAsync(g.C32, 0, sizeof(float) * static_cast<size_t>(g.M) * g.N, st), "gemm");
    p.splitk = splitk;
    // Staged TMA-store epilogue wherever the outputs allow it (16-byte aligned base and row pitch, even N, the pair loads of
    // bias / aux aligned); anything else keeps the fragment stores.  C32 += tile goes through TMA reduce-add for split-K
    // partial tiles and for beta without a 16-bit output (with one, the old C32 is read so that C16 gets the sum too).
    auto al = [](const void* q, int a) { return (reinterpret_cast<uintptr_t>(q) & (a - 1)) == 0; };
    const bool tma_c = (g.N % 2 == 0) &&
                       (!g.C32 || (al(g.C32, 16) && (g.ldc32 * 4) % 16 == 0)) &&
                       (!g.C16 || (al(g.C16, 16) && (g.ldc16 * 2) % 16 == 0)) &&
                       (g.act != 2 || (al(g.aux16, 4) && g.ldaux % 2 == 0)) &&
                       (!g.bias || al(g.bias, 8)) && (!g.bias2 || al(g.bias2, 8));
    // 2-CTA clusters (B multicast) for wide outputs with enough 256 x 256 tiles to fill the machine, only when
    // ft_set_gemm_pair_mode asks for them.  Mode 1: only for the big contractions (>= 1e11 FLOP).  Mode 2: whenever eligible.
    const long long tiles_m2 = (g.M + 2 * BM - 1) / (2 * BM);
    const bool big = 2.0 * g.M * g.N * g.K >= 1e11;
    const int ncta = ((g_pair_mode == 2 || (g_pair_mode == 1 && big)) && wide && splitk == 1 && tiles_m2 * tiles_n >= sms / 2) ? 2 : 1;
    // Ping-pong (128 x 128 tiles, one per consumer warpgroup, each epilogue under the other warpgroup's main loop) for the
    // staged epilogue without split-K or CTA pairs.  Its epilogue reads nothing from global memory but the biases, so
    // act = 2 and beta with a 16-bit output stay cooperative.  By shape (tools/gemm_shapes.py --schedules, DESIGN 4.1): it
    // wins wherever a CTA has at least 3 tiles to alternate over and K <= 4096 (xproj0 0.80 vs 1.25 ms, dgrad ih0 0.75 vs
    // 0.78); with fewer tiles (dgrad xproj1 chunk, 200 tiles: 0.064 vs 0.060-0.062) or long K (wgrad ih0, 416 tiles over
    // K = 32000: 0.90 vs 0.65-0.67) the cooperative 128 x BN tile is as fast or faster.
    const bool pp_ok = tma_c && splitk == 1 && ncta == 1 && g.act != 2 && !(g.beta && g.C16);
    const bool pp_shape = g.K <= 4096 && static_cast<long long>((g.N + 127) / 128) * tiles_m >= 3LL * sms;
    const bool pp = pp_ok && (FT_GEMM_SCHEDULE == 2 || (FT_GEMM_SCHEDULE == 0 && pp_shape));
    if (pp) {
        bn = 128;
        tiles_n = (g.N + bn - 1) / bn;
        if (static_cast<long long>(tiles_n) * tiles_m > 0x7fffffff) return ft_set_error("gemm: too many tiles");
        n_tiles = tiles_n * tiles_m;
    }
    CUtensorMap tmC32 = {}, tmC16 = {};
    if (tma_c) {                         // stores of 64-row chunks by a warpgroup (cooperative) or 16-row ones by a warp
        p.tma_c = 1;
        p.c32_add = g.C32 && (splitk > 1 || (g.beta && !g.C16));
        const int box_rows = pp ? 16 : 64;
        if (g.C32 && make_tmap_2d(&tmC32, g.C32, FMT_TF32, g.M, g.N, g.ldc32, 32, box_rows)) return -1;
        if (g.C16 && make_tmap_2d(&tmC16, g.C16, g.c16_fmt, g.M, g.N, g.ldc16, 32, box_rows, 64)) return -1;
    }
    int rc;
    if (!g.a_mn) rc = make_tmap_2d(&tmA, g.A, g.a_fmt, g.M, g.K, g.lda, BK, BM);
    else         rc = make_tmap_2d(&tmA, g.A, g.a_fmt, g.K, g.M, g.lda, BK, BK);
    if (rc) return rc;
    if (!g.b_mn) rc = make_tmap_2d(&tmB, g.B, g.b_fmt, g.N, g.K, g.ldb, BK, bn / ncta);     // each CTA of a pair fetches half of B
    else         rc = make_tmap_2d(&tmB, g.B, g.b_fmt, g.K, g.N, g.ldb, BK, BK);
    if (rc) return rc;
    if (ncta == 2) n_tiles = static_cast<int>(tiles_m2 * tiles_n);
    const long long n_work = static_cast<long long>(n_tiles) * splitk;
    const int units = ncta == 2 ? sms / 2 : sms;
    const int grid = ncta * static_cast<int>(n_work < units ? n_work : units);
    const int smem = bn == 256 ? G2Cfg<256>::SMEM : G2Cfg<128>::SMEM;
    const void* fn = g.a_fmt == FMT_TF32 ? gemm_kernel_ptr<FMT_TF32, 0>(bn, ncta, 0, pp)
                   : g.a_fmt == FMT_BF16 ? (g.a_mn ? gemm_kernel_ptr<FMT_BF16, 1>(bn, ncta, g.b_mn, pp) : gemm_kernel_ptr<FMT_BF16, 0>(bn, ncta, g.b_mn, pp))
                                         : (g.a_mn ? gemm_kernel_ptr<FMT_F16, 1>(bn, ncta, g.b_mn, pp) : gemm_kernel_ptr<FMT_F16, 0>(bn, ncta, g.b_mn, pp));
    static bool attr_set[3][2][2][2][2][2] = {};
    bool& done = attr_set[g.a_fmt][bn == 256][ncta - 1][g.a_mn][g.b_mn][pp];
    if (!done) {
        if (cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess) return ft_set_error("gemm: shared-memory opt-in failed");
        done = true;
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid); cfg.blockDim = dim3(G2_THREADS); cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = 2; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr; cfg.numAttrs = ncta == 2 ? 1 : 0;
    void* args[] = {&tmA, &tmB, &tmC32, &tmC16, &p, &tiles_n, &n_tiles};
    TimeScope ts(g.a_mn ? "gemm_wgrad" : (g.b_mn ? "gemm_dgrad" : "gemm_fwd"), g.M, g.N, g.K, st);
    cudaError_t e = cudaLaunchKernelExC(&cfg, fn, args);
    if (e != cudaSuccess) return ft_set_error(cudaGetErrorString(e));
    ft_count_launch(1);
    return ft_check_launch(ncta == 2 ? "gemm2_kernel<pair>" : "gemm2_kernel");
}

int gemm_nt(cudaStream_t st, long long M, int N, int K, const void* A, long long lda, const void* B, long long ldb, float* C32,
            long long ldc32, void* C16, long long ldc16, const float* bias, const float* bias2, int act, int beta) {
    GemmArgs g;
    g.M = static_cast<int>(M); g.N = N; g.K = K;
    g.A = A; g.lda = lda; g.a_fmt = FMT_F16; g.B = B; g.ldb = ldb; g.b_fmt = FMT_F16;
    g.bias = bias; g.bias2 = bias2; g.act = act; g.beta = beta;
    g.C32 = C32; g.ldc32 = ldc32; g.C16 = C16; g.ldc16 = ldc16; g.c16_fmt = FMT_F16;
    return launch_gemm(g, st);
}

int gemm_dgrad(cudaStream_t st, long long M, int Kout, int N, const void* dY, long long lddy, const void* W, long long ldw,
               float* C32, long long ldc32, void* C16, long long ldc16, int beta, const float* alpha_ptr, const void* aux16,
               long long ldaux) {
    GemmArgs g;
    g.M = static_cast<int>(M); g.N = Kout; g.K = N;
    g.A = dY; g.lda = lddy; g.a_fmt = FMT_F16; g.B = W; g.ldb = ldw; g.b_fmt = FMT_F16; g.b_mn = 1;
    g.alpha_ptr = alpha_ptr; g.beta = beta;
    g.C32 = C32; g.ldc32 = ldc32; g.C16 = C16; g.ldc16 = ldc16; g.c16_fmt = FMT_F16;
    if (aux16) { g.act = 2; g.aux16 = aux16; g.ldaux = ldaux; }
    return launch_gemm(g, st);
}

int gemm_wgrad(cudaStream_t st, int N, int K, long long R, const void* dY, long long lddy, const void* X, long long ldx, float* dW,
               long long ldw, const float* alpha_ptr, int beta) {
    if (R <= 0) {
        if (!beta) FT_CU(cudaMemsetAsync(dW, 0, sizeof(float) * N * ldw, st), "gemm_wgrad");
        return 0;
    }
    GemmArgs g;
    g.M = N; g.N = K; g.K = static_cast<int>(R);
    g.A = dY; g.lda = lddy; g.a_fmt = FMT_F16; g.a_mn = 1; g.B = X; g.ldb = ldx; g.b_fmt = FMT_F16; g.b_mn = 1;
    g.alpha_ptr = alpha_ptr; g.beta = beta;
    g.C32 = dW; g.ldc32 = ldw;
    return launch_gemm(g, st);
}

}  // namespace ft
