// C-ABI entry points of libflowtron_b200.so that are not tied to one kernel file: error plumbing,
// watchdog status, launch counting, and the primitive GEMM export.  See include/flowtron_b200.h.
#include <mutex>
#include <string>
#include <atomic>
#include <cstdio>
#include <vector>
#include <map>
#include <tuple>

#include "ft_internal.h"
#include "../../include/flowtron_b200.h"

namespace ft {

static thread_local std::string g_err;
static std::atomic<long long> g_launches{0};
static int* g_status_dev = nullptr;
static std::mutex g_mu;

int ft_set_error(const char* msg) {
    g_err = msg ? msg : "unknown error";
    return -1;
}
int ft_runtime_error(const char* who) {
    g_err = std::string(who) + ": CUDA runtime call failed";
    return -1;
}
int ft_check_launch(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        g_err = std::string(what) + ": " + cudaGetErrorString(e);
        return -1;
    }
    return 0;
}
int* ft_status_word() {
    std::lock_guard<std::mutex> lk(g_mu);
    if (!g_status_dev) {
        if (cudaMalloc(&g_status_dev, 64) != cudaSuccess) return nullptr;
        cudaMemset(g_status_dev, 0, 64);
    }
    return g_status_dev;
}
void ft_count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

// ---- optional per-kernel device timing (CUDA events on the launching stream; bench.py's roofline leg)
struct TimeRec { const char* name; long long m, n, k; cudaEvent_t a, b; };
static bool g_timing = false;
static std::vector<TimeRec> g_recs;
static std::vector<cudaEvent_t> g_pool;
static cudaEvent_t get_event() {
    if (!g_pool.empty()) { cudaEvent_t e = g_pool.back(); g_pool.pop_back(); return e; }
    cudaEvent_t e; cudaEventCreate(&e); return e;
}
TimeScope::TimeScope(const char* name, long long m, long long n, long long k, cudaStream_t st) : st_(st), idx_(-1) {
    if (!g_timing) return;
    std::lock_guard<std::mutex> lk(g_mu);
    TimeRec r{name, m, n, k, get_event(), get_event()};
    cudaEventRecord(r.a, st);              // unchecked: a timing bracket must not fail the launch it measures
    g_recs.push_back(r);
    idx_ = static_cast<int>(g_recs.size()) - 1;
}
TimeScope::~TimeScope() {
    if (idx_ < 0) return;
    std::lock_guard<std::mutex> lk(g_mu);
    cudaEventRecord(g_recs[idx_].b, st_);  // unchecked: as above; ft_timing_report skips a bracket it cannot time
}

}  // namespace ft

extern "C" {

int ft_version(void) { return 100; }
int ft_max_text_len(void) { return FT_MAX_TEXT_LEN; }

const char* ft_last_error(void) { return ft::g_err.c_str(); }

int ft_device_status(void) {
    int* w = ft::ft_status_word();
    if (!w) return -1;
    int v = 0;
    if (cudaMemcpy(&v, w, sizeof(int), cudaMemcpyDeviceToHost) != cudaSuccess) return -2;
    return v;
}

void ft_timing_enable(int on) { ft::g_timing = on != 0; }
void ft_timing_reset(void) {
    std::lock_guard<std::mutex> lk(ft::g_mu);
    for (auto& r : ft::g_recs) { ft::g_pool.push_back(r.a); ft::g_pool.push_back(r.b); }
    ft::g_recs.clear();
}
/* Synchronises the device; writes one line per (kernel, shape): "name m n k count total_ms\n". Returns bytes written. */
int ft_timing_report(char* buf, int cap) {
    cudaDeviceSynchronize();
    std::lock_guard<std::mutex> lk(ft::g_mu);
    std::map<std::tuple<std::string, long long, long long, long long>, std::pair<int, double>> agg;
    for (auto& r : ft::g_recs) {
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, r.a, r.b) != cudaSuccess) continue;
        auto& e = agg[std::make_tuple(std::string(r.name), r.m, r.n, r.k)];
        e.first += 1; e.second += ms;
    }
    int off = 0;
    for (auto& kv : agg) {
        int w = snprintf(buf + off, cap - off, "%s %lld %lld %lld %d %.6f\n", std::get<0>(kv.first).c_str(),
                         std::get<1>(kv.first), std::get<2>(kv.first), std::get<3>(kv.first), kv.second.first, kv.second.second);
        if (w < 0 || off + w >= cap) break;
        off += w;
    }
    return off;
}

long long ft_launch_count(void) { return ft::g_launches.load(); }
void ft_reset_launch_count(void) { ft::g_launches.store(0); }

int ft_gemm(int M, int N, int K, const void* A, long long lda, int a_fmt, int a_mn, const void* B, long long ldb,
            int b_fmt, int b_mn, const float* bias, const float* bias2, int act, int beta, float alpha, float* C32,
            long long ldc32, void* C16, long long ldc16, int c16_fmt, void* stream) {
    ft::GemmArgs g;
    g.M = M; g.N = N; g.K = K;
    g.A = A; g.lda = lda; g.a_fmt = a_fmt; g.a_mn = a_mn;
    g.B = B; g.ldb = ldb; g.b_fmt = b_fmt; g.b_mn = b_mn;
    g.bias = bias; g.bias2 = bias2; g.act = act; g.beta = beta; g.alpha = alpha;
    g.C32 = C32; g.ldc32 = ldc32; g.C16 = C16; g.ldc16 = ldc16; g.c16_fmt = c16_fmt;
    return ft::launch_gemm(g, static_cast<cudaStream_t>(stream));
}

/* debug: device buffer [T][8] receiving clock64 stamps of CTA 0 of the next lstm_fwd launches (NULL disables) */
void ft_debug_set_lstm_trace(long long* buf) { ft::set_lstm_trace(buf); }

/* debug: how many 4-CTA clusters of the BPTT cluster kernel fit on the device at its launch configuration for batch B
   (cudaOccupancyMaxActiveClusters), or -1 */
int ft_debug_lstm_bwd_max_clusters(int B) { return ft::lstm_bwd_max_clusters(B); }

/* debug: steps [t0, t1) of one layer-pipeline BPTT chunk, on the flat kernel (xchg non-null) or the cluster kernel (NULL) */
int ft_debug_lstm_bwd_chunk(int T, int B, int t0, int t1, const float* dh_ext, long long ldd, const void* whhT16,
                            const void* gates16, const float* cstate, const int* lens, void* dG16, float* dc_carry, int* flags,
                            float* xchg, void* stream) {
    return ft::launch_lstm_bwd_chunk(T, B, t0, t1, dh_ext, ldd, whhT16, gates16, cstate, lens, dG16, dc_carry, flags, xchg,
                                     static_cast<cudaStream_t>(stream));
}

void ft_set_gemm_pair_mode(int mode) { ft::set_gemm_pair_mode(mode); }

int ft_lstm_fwd(int T, int B, const float* xproj, const void* whh16, const int* lens, void* hseq16, long long ldh,
                void* gates16, float* cstate, float* h32, long long ldh32, int* flags, void* stream) {
    return ft::launch_lstm_fwd(T, B, xproj, whh16, lens, hseq16, ldh, gates16, cstate, h32, ldh32, flags,
                               static_cast<cudaStream_t>(stream));
}

int ft_lstm_bwd(int T, int B, const float* dh_ext, long long ldd, const void* whhT16, const void* gates16,
                const float* cstate, const int* lens, void* dG16, int* flags, void* stream) {
    return ft::launch_lstm_bwd(T, B, dh_ext, ldd, whhT16, gates16, cstate, lens, dG16, flags,
                               static_cast<cudaStream_t>(stream));
}

}  // extern "C"
