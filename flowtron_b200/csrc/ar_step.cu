// Host-side orchestration of one Flowtron AR flow step (training direction) on a CUDA stream:
// AR_Step.forward / AR_Back_Step.forward (flowtron.py:725-773, 605-627) and their autograd.
// No allocation, no synchronisation: every intermediate lives in the caller's `saved` / `scratch` areas,
// whose layouts are planned by the same code that uses them (Workspace, ft_internal.h).
//
// Precision plan (DESIGN.md): forward tensor-core operands are fp16 (11-bit significand, same as tf32; every
// forward operand is either a weight or a bounded activation); backward operands are fp16 too, on gradients
// multiplied by a per-flow power-of-two loss scale chosen on the device (launch_grad_scale); accumulation, LSTM cell state, softmax, exp/log and all reductions are fp32.
#include <algorithm>
#include <cstring>
#include <initializer_list>
#include <map>
#include <mutex>
#include <string>
#include <vector>

#include "ft_internal.h"
#include "../../include/flowtron_b200.h"

namespace ft {

namespace {

constexpr int H = 1024, G = 4096;

struct Dims {
    long long R, RL;
    int T, B, L, M, A, E, D;
    explicit Dims(const FtArStepDesc& d)
        : R(static_cast<long long>(d.T) * d.B), RL(static_cast<long long>(d.L) * d.B), T(d.T), B(d.B), L(d.L), M(d.n_mel),
          A(d.n_attn), E(d.n_text), D(H + d.n_attn) {}
};

// ---- tensors that persist from forward to backward
struct Saved {
    uint16_t *mel_in16, *d16, *gatesA, *text16, *h0_16, *gates0, *h1_16, *gates1, *y1_16, *y2_16;
    float *mel_flow, *cA, *Kp, *Vp, *Q, *p_save, *c0, *c1, *o32;
    void plan(Workspace& p, const FtArStepDesc& d) {
        const Dims n(d);
        mel_in16 = p.get<uint16_t>("mel_in16", n.R * n.M);
        mel_flow = d.reversed ? p.get<float>("mel_flow", n.R * n.M) : nullptr;
        d16 = p.get<uint16_t>("d16", n.R * n.D);
        gatesA = p.get<uint16_t>("gatesA", n.R * G);
        cA = p.get<float>("cA", n.R * H);
        text16 = p.get<uint16_t>("text16", n.RL * n.E);
        Kp = p.get<float>("Kp", n.RL * n.A);
        Vp = p.get<float>("Vp", n.RL * n.A);
        Q = p.get<float>("Q", n.R * n.A);
        p_save = d.has_prior ? p.get<float>("p_save", static_cast<size_t>(n.B) * n.T * n.L) : nullptr;
        h0_16 = p.get<uint16_t>("h0_16", n.R * H);
        gates0 = p.get<uint16_t>("gates0", n.R * G);
        c0 = p.get<float>("c0", n.R * H);
        h1_16 = p.get<uint16_t>("h1_16", n.R * H);
        gates1 = p.get<uint16_t>("gates1", n.R * G);
        c1 = p.get<float>("c1", n.R * H);
        y1_16 = p.get<uint16_t>("y1_16", n.R * H);
        y2_16 = p.get<uint16_t>("y2_16", n.R * H);
        o32 = p.get<float>("o32", n.R * 2 * n.M);
    }
};

// ---- 16-bit weight copies (fp16 for forward, bf16 for backward)
struct W16 {
    uint16_t *w_ih_a, *w_hh_a, *w_ih0, *w_hh0, *w_ih1, *w_hh1, *wq, *wk, *wv, *w1, *w2, *wc;
    void plan(Workspace& p, const Dims& n) {
        w_ih_a = p.get<uint16_t>("w_ih_a", static_cast<size_t>(G) * n.M);
        w_hh_a = p.get<uint16_t>("w_hh_a", static_cast<size_t>(G) * H);
        w_ih0 = p.get<uint16_t>("w_ih0", static_cast<size_t>(G) * n.D);
        w_hh0 = p.get<uint16_t>("w_hh0", static_cast<size_t>(G) * H);
        w_ih1 = p.get<uint16_t>("w_ih1", static_cast<size_t>(G) * H);
        w_hh1 = p.get<uint16_t>("w_hh1", static_cast<size_t>(G) * H);
        wq = p.get<uint16_t>("wq", static_cast<size_t>(n.A) * H);
        wk = p.get<uint16_t>("wk", static_cast<size_t>(n.A) * n.E);
        wv = p.get<uint16_t>("wv", static_cast<size_t>(n.A) * n.E);
        w1 = p.get<uint16_t>("w1", static_cast<size_t>(H) * H);
        w2 = p.get<uint16_t>("w2", static_cast<size_t>(H) * H);
        wc = p.get<uint16_t>("wc", static_cast<size_t>(2 * n.M) * H);
    }
};

// Layer pipeline (DESIGN.md 4.2): lstm layers 0 and 1 run as two 64-CTA recurrences one chunk of kLayerChunk steps apart,
// forward and BPTT; a sequence of at most kLayerChunk steps is a single chunk.  On a 132-SM H100 the two recurrences leave
// 4 SMs to the per-chunk GEMMs, which mostly run between recurrence steps; the schedule still wins there (DESIGN.md 4.11:
// B=32, T=1000, 74 ms/step with both pipelines, 84 without).
constexpr int kLayerChunk = 100;
// Attention-LSTM overlap chunk in steps (a multiple of 64): the overlap runs when T >= kAttnChunk + 64.
constexpr int kAttnChunk = 256;

static int layer_chunk(int T) { return T < kLayerChunk ? T : kLayerChunk; }
constexpr int kBwdXchgPerRow = 2 * 16 * 4 * 64;   // flat BPTT partial-sum ring, floats per batch row: [2][16 groups][4 ranks][B][64]

struct FwdScratch {
    W16 w;
    float* X;
    int* flags;
    float* X1;                  // second input-projection buffer: the attention LSTM's (overlap), then layer 1's (pipeline)
    float *hA32 = nullptr, *ctx32 = nullptr;     // fp32 copies of [hA ; ctx] for the gate logits (gated flow only)
    float* attn_rows = nullptr;                  // long texts: the attention's score rows (attn_rows_in_global)
    void plan(Workspace& p, const FtArStepDesc& d) {
        const Dims n(d);
        w.plan(p, n);
        X = p.get<float>("X", n.R * G);
        flags = p.get<int>("flags", static_cast<size_t>(n.T) * 64);
        X1 = p.get<float>("X1", n.R * G);
        if (d.has_gate) {
            hA32 = p.get<float>("hA32", n.R * H);
            ctx32 = p.get<float>("ctx32", n.R * n.A);
        }
        if (attn_rows_in_global(n.L, n.A)) attn_rows = p.get<float>("attn_rows", attn_rows_floats(n.T, n.B, n.L));
    }
};

// What the attention-LSTM part of the backward (ar_step_bwd_attn) needs from the main part (ar_step_bwd_main): the two are
// separate entry points so that the caller's autograd can run whatever depends only on d_text (the text encoder's backward)
// concurrently with the attention LSTM's BPTT, a 64-SM kernel.  Lives in caller memory (`carry`), not in the shared scratch.
struct BwdCarry {
    float *dd, *dmel_flow, *scale;
    void plan(Workspace& p, const FtArStepDesc& d) {
        const Dims n(d);
        dd = p.get<float>("dd", n.R * n.D);                 // [R, D]: cols 0:H = dhA (attention-LSTM output gradient), H: = dctx
        dmel_flow = p.get<float>("dmel_flow", n.R * n.M);
        scale = p.get<float>("scale", 8);
    }
};

struct BwdScratch {
    W16 w;                      // fp16, natural layouts (w_hh* hold the TRANSPOSED recurrent weights [H, 4H])
    uint16_t *dG1, *dG0, *dGa, *do16, *dy2, *dy1, *dQ16, *dK16, *dV16;
    float *dh, *dQ, *dK, *dV, *dmel_in;
    int* flags;
    float *dcarry1, *dcarry0;   // dc*f hand-over between BPTT chunks of the layer pipeline
    float *xchg1, *xchg0;       // partial-sum rings of the two pipelined BPTT recurrences (flat kernel, lstm.cu)
    float* attn_rows = nullptr; // long texts: the attention backward's gradient rows (attn_rows_in_global)
    float* sink;
    void plan(Workspace& p, const FtArStepDesc& d) {
        const Dims n(d);
        w.plan(p, n);
        dG1 = p.get<uint16_t>("dG1", n.R * G);      // one per LSTM layer: the wgrad GEMMs of a layer run on the side
        dG0 = p.get<uint16_t>("dG0", n.R * G);      // stream while the next BPTT already writes its own dG
        dGa = p.get<uint16_t>("dGa", n.R * G);
        do16 = p.get<uint16_t>("do16", n.R * 2 * n.M);
        dy2 = p.get<uint16_t>("dy2", n.R * H);
        dy1 = p.get<uint16_t>("dy1", n.R * H);
        dQ16 = p.get<uint16_t>("dQ16", n.R * n.A);
        dK16 = p.get<uint16_t>("dK16", n.RL * n.A);
        dV16 = p.get<uint16_t>("dV16", n.RL * n.A);
        dh = p.get<float>("dh", n.R * H);
        dQ = p.get<float>("dQ", n.R * n.A);
        dK = p.get<float>("dK", n.RL * n.A);
        dV = p.get<float>("dV", n.RL * n.A);
        dmel_in = p.get<float>("dmel_in", n.R * n.M);
        // 64 per step for the attention LSTM's BPTT (T steps), 128 per step for one chunk of each of the layer pipeline's two
        // recurrences (dG release + partial-sum exchange flags)
        flags = p.get<int>("flags", std::max(static_cast<size_t>(n.T) * 64, static_cast<size_t>(2 * layer_chunk(n.T)) * 128));
        dcarry1 = p.get<float>("dcarry1", static_cast<size_t>(n.B) * H);
        dcarry0 = p.get<float>("dcarry0", static_cast<size_t>(n.B) * H);
        xchg1 = p.get<float>("xchg1", static_cast<size_t>(kBwdXchgPerRow) * n.B);
        xchg0 = p.get<float>("xchg0", static_cast<size_t>(kBwdXchgPerRow) * n.B);
        if (attn_rows_in_global(n.L, n.A)) attn_rows = p.get<float>("attn_rows", attn_rows_floats(n.T, n.B, n.L));
        // target of the gradients the attention / gate kernels always accumulate but the caller may not want (v, and one
        // of the gate's weight / bias); never read
        sink = p.get<float>("sink", static_cast<size_t>(n.A) + n.D + 1);
    }
};

// The dependency rule of the backward (ft_ar_step_bwd_plan in flowtron_b200.h): one bit per stage, set when something
// downstream of the stage is wanted.  The two backward entry points branch on this mask only.
unsigned bwd_plan(const FtArStepDesc& d, const FtArStepWeights& g, bool want_d_text, bool want_d_mel) {
    auto any = [](std::initializer_list<const float*> ps) {
        for (const float* q : ps) if (q) return true;
        return false;
    };
    unsigned m = 0;
    if (any({g.conv_w, g.conv_b})) m |= FT_BWD_G_CONV;
    if (any({g.dense_w1, g.dense_b1})) m |= FT_BWD_G_DENSE1;
    if (any({g.dense_w0, g.dense_b0})) m |= FT_BWD_G_DENSE0;
    if (any({g.lstm_w_ih1, g.lstm_w_hh1, g.lstm_b_ih1, g.lstm_b_hh1})) m |= FT_BWD_G_LSTM1;
    if (any({g.lstm_w_ih0, g.lstm_w_hh0, g.lstm_b_ih0, g.lstm_b_hh0})) m |= FT_BWD_G_LSTM0;
    if (g.att_query) m |= FT_BWD_G_QUERY;
    if (g.att_key) m |= FT_BWD_G_KEY;
    if (g.att_value) m |= FT_BWD_G_VALUE;
    if (g.att_v) m |= FT_BWD_G_V;
    if (any({g.attn_lstm_w_ih, g.attn_lstm_w_hh, g.attn_lstm_b_ih, g.attn_lstm_b_hh})) m |= FT_BWD_G_ATTN_LSTM;
    if (d.has_gate && any({g.gate_w, g.gate_b})) m |= FT_BWD_G_GATE;
    if (want_d_mel) m |= FT_BWD_D_MEL;
    if (m & (FT_BWD_D_MEL | FT_BWD_G_ATTN_LSTM)) m |= FT_BWD_ATTN_LSTM;
    if (m & FT_BWD_ATTN_LSTM) m |= FT_BWD_QUERY_DGRAD;
    if (want_d_text) m |= FT_BWD_D_TEXT;
    if (m & (FT_BWD_QUERY_DGRAD | FT_BWD_D_TEXT | FT_BWD_G_QUERY | FT_BWD_G_KEY | FT_BWD_G_VALUE | FT_BWD_G_V)) m |= FT_BWD_ATTN;
    if (d.has_gate && (m & (FT_BWD_ATTN | FT_BWD_ATTN_LSTM))) m |= FT_BWD_GATE_DD;
    if (m & (FT_BWD_ATTN | FT_BWD_ATTN_LSTM | FT_BWD_G_LSTM0)) m |= FT_BWD_LSTM0;
    if (m & (FT_BWD_LSTM0 | FT_BWD_G_LSTM1)) m |= FT_BWD_LSTM1;
    if (m & FT_BWD_LSTM1) m |= FT_BWD_DENSE0_DGRAD;
    if (m & (FT_BWD_DENSE0_DGRAD | FT_BWD_G_DENSE0)) m |= FT_BWD_DENSE1_DGRAD;
    if (m & (FT_BWD_DENSE1_DGRAD | FT_BWD_G_DENSE1)) m |= FT_BWD_CONV_DGRAD;
    if (m & (FT_BWD_CONV_DGRAD | FT_BWD_G_CONV | FT_BWD_D_MEL)) m |= FT_BWD_COUPLING;
    return m;
}

int check_desc(const FtArStepDesc& d) {
    if (d.n_hidden != H) return ft_set_error("ar_step: this build supports n_hidden == 1024 only");
    if (d.T <= 0 || d.B <= 0 || d.L <= 0) return ft_set_error("ar_step: empty shape");
    if (d.B > 32) return ft_set_error("ar_step: batch > 32 per call not supported (split the batch)");
    if (d.n_mel > 128 || d.n_mel % 8 || d.n_attn % 64 || d.n_text % 8)
        return ft_set_error("ar_step: n_mel <= 128 and %8, n_attn %64, n_text %8 required");
    if (d.L > FT_MAX_TEXT_LEN) return ft_set_error("ar_step: L > FT_MAX_TEXT_LEN (1024) not supported");
    return 0;
}

// Streams of one caller stream's flow steps, created on its first call; ordering between them is by events only.
// side: work off the backward critical path (weight gradients, bias column sums), which runs under the next persistent BPTT
// kernel (64 of the SMs); fork: side waits for "main so far", join: main waits for "side so far".
// sA / sB run the recurrences of the layer pipeline and the attention overlap at HIGH priority, so that when a chunk ends its
// 64 SMs go to the next chunk (a cooperative launch that needs all of them at once) and not to queued CTAs of the GEMM /
// attention kernels that share the machine; sC runs their per-chunk GEMMs one priority level above default streams.
struct Streams {
    cudaStream_t side = nullptr, sA = nullptr, sB = nullptr, sC = nullptr;
    cudaEvent_t ev_main = nullptr, ev_side = nullptr, evA = nullptr, evG = nullptr, evB = nullptr, ev0 = nullptr, evJ = nullptr;
};
static std::map<cudaStream_t, Streams> g_streams;
static std::mutex g_streams_mu;

static Streams* get_streams(cudaStream_t main) {
    std::lock_guard<std::mutex> lk(g_streams_mu);
    auto it = g_streams.find(main);
    if (it != g_streams.end()) return &it->second;
    Streams s;
    int prio_lo = 0, prio_hi = 0;
    if (cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi) != cudaSuccess) return nullptr;   // hi is numerically smaller
    const int mid = prio_hi < prio_lo - 1 ? prio_lo - 1 : prio_lo;
    if (cudaStreamCreateWithFlags(&s.side, cudaStreamNonBlocking) != cudaSuccess ||
        cudaStreamCreateWithPriority(&s.sA, cudaStreamNonBlocking, prio_hi) != cudaSuccess ||
        cudaStreamCreateWithPriority(&s.sB, cudaStreamNonBlocking, prio_hi) != cudaSuccess ||
        cudaStreamCreateWithPriority(&s.sC, cudaStreamNonBlocking, mid) != cudaSuccess)
        return nullptr;
    for (cudaEvent_t* e : {&s.ev_main, &s.ev_side, &s.evJ, &s.evA, &s.evG, &s.evB, &s.ev0})
        if (cudaEventCreateWithFlags(e, cudaEventDisableTiming) != cudaSuccess) return nullptr;
    return &(g_streams[main] = s);
}

// Every stream in `waiters` waits for what `producer` has been given so far.
static int order(cudaEvent_t ev, cudaStream_t producer, std::initializer_list<cudaStream_t> waiters) {
    FT_CU(cudaEventRecord(ev, producer), "ar_step");
    for (cudaStream_t w : waiters) FT_CU(cudaStreamWaitEvent(w, ev, 0), "ar_step");
    return 0;
}
static int fork_side(const Streams* s, cudaStream_t main) { return order(s->ev_main, main, {s->side}); }
static int join_side(const Streams* s, cudaStream_t main) { return order(s->ev_side, s->side, {main}); }

}  // namespace

// =================================================================================================== forward
int ar_step_fwd(const FtArStepDesc& d, const FtArStepWeights& w, const float* mel, const float* text, const int* in_lens,
                const int* out_lens, const float* prior, float* mel_out, float* log_s, float* gates, float* attn,
                float* logprob, void* saved, void* scratch, cudaEvent_t text_ready, cudaStream_t st) {
    FT_TRY(check_desc(d));
    if (d.has_prior && !prior) return ft_set_error("ar_step_fwd: has_prior set but attn_prior is NULL");
    if (d.has_gate && (!gates || !w.gate_w)) return ft_set_error("ar_step_fwd: has_gate set but gate pointers are NULL");
    const Dims n(d);
    Workspace ps; ps.base = static_cast<uint8_t*>(saved);
    Saved S; S.plan(ps, d);
    Workspace pf; pf.base = static_cast<uint8_t*>(scratch);
    FwdScratch F; F.plan(pf, d);

    // fp16 operand copies of the weights (61 M params; redone every call so optimizer updates are seen)
    FT_TRY(launch_cast(w.attn_lstm_w_ih, 2, F.w.w_ih_a, 0, static_cast<long long>(G) * n.M, st));
    FT_TRY(launch_cast(w.attn_lstm_w_hh, 2, F.w.w_hh_a, 0, static_cast<long long>(G) * H, st));
    FT_TRY(launch_cast(w.lstm_w_ih0, 2, F.w.w_ih0, 0, static_cast<long long>(G) * n.D, st));
    FT_TRY(launch_cast(w.lstm_w_hh0, 2, F.w.w_hh0, 0, static_cast<long long>(G) * H, st));
    FT_TRY(launch_cast(w.lstm_w_ih1, 2, F.w.w_ih1, 0, static_cast<long long>(G) * H, st));
    FT_TRY(launch_cast(w.lstm_w_hh1, 2, F.w.w_hh1, 0, static_cast<long long>(G) * H, st));
    FT_TRY(launch_cast(w.att_query, 2, F.w.wq, 0, static_cast<long long>(n.A) * H, st));
    FT_TRY(launch_cast(w.att_key, 2, F.w.wk, 0, static_cast<long long>(n.A) * n.E, st));
    FT_TRY(launch_cast(w.att_value, 2, F.w.wv, 0, static_cast<long long>(n.A) * n.E, st));
    FT_TRY(launch_cast(w.dense_w0, 2, F.w.w1, 0, static_cast<long long>(H) * H, st));
    FT_TRY(launch_cast(w.dense_w1, 2, F.w.w2, 0, static_cast<long long>(H) * H, st));
    FT_TRY(launch_cast(w.conv_w, 2, F.w.wc, 0, static_cast<long long>(2 * n.M) * H, st));

    // teacher-forcing shift (+ AR_Back_Step time reversal folded into the gather)
    FT_TRY(launch_prep_mel(mel, out_lens, n.T, n.B, n.M, d.reversed, S.mel_in16, S.mel_flow, st));
    const float* mel_flow = d.reversed ? S.mel_flow : mel;

    Streams* pp = get_streams(st);
    if (!pp) return ft_set_error("ar_step_fwd: could not create the pipeline streams");

    // Attention-LSTM / attention overlap (T >= kAttnChunk + 64): the attention LSTM runs as a 64-CTA recurrence in chunks of
    // kAttnChunk steps; as soon as a chunk's h is there, a second stream runs that chunk's query projection, fused attention,
    // gate logits and lstm layer 0's input projection on the SMs the 64-CTA recurrence leaves free, underneath the next
    // chunk's recurrence.  Only the last chunk's share of that work stays exposed.  The 64-CTA kernel has no room for the
    // folded 80-channel projection next to its 128 KB weight slice, so the projection is a per-chunk GEMM on a third stream,
    // one chunk ahead.  Short chunks lose: every chunk boundary costs a kernel drain + launch + 128 KB weight reload on 64 SMs.
    auto attention_rows = [&](cudaStream_t s2, int t0, int t1) -> int {      // Q projection, attention, gate logits of steps [t0, t1)
        const long long r0 = static_cast<long long>(t0) * n.B, rows = static_cast<long long>(t1 - t0) * n.B;
        FT_TRY(gemm_nt(s2, rows, n.A, H, S.d16 + r0 * n.D, n.D, F.w.wq, H, S.Q + r0 * n.A, n.A));
        AttnFwdArgs a;
        a.T = n.T; a.B = n.B; a.L = n.L; a.A = n.A;
        a.Q = S.Q; a.ldq = n.A; a.K = S.Kp; a.ldk = n.A; a.V = S.Vp; a.ldv = n.A; a.v = w.att_v;
        a.in_lens = in_lens; a.out_lens = out_lens; a.prior = d.has_prior ? prior : nullptr; a.reversed = d.reversed;
        a.temperature = d.temperature; a.attn = attn; a.logprob = logprob; a.p_save = S.p_save;
        a.ctx16 = S.d16 + H; a.ldc = n.D; a.ctx32 = F.ctx32; a.ldc32 = n.A;
        a.t_begin = t0; a.t_end = t1; a.rows = F.attn_rows;
        FT_TRY(launch_attn_fwd(a, s2));
        if (d.has_gate) FT_TRY(launch_gate_fwd_f32(F.hA32 + r0 * H, H, H, F.ctx32 + r0 * n.A, n.A, n.A, w.gate_w, w.gate_b, rows, gates + r0, s2));
        return 0;
    };
    auto kv_projections = [&](cudaStream_t s2) -> int {
        // First use of `text`: if the caller produced it on another stream it passed the event to wait for, so the encoder
        // ran underneath everything above.
        if (text_ready) {
            if (cudaStreamWaitEvent(s2, text_ready, 0) != cudaSuccess) return ft_set_error("ar_step_fwd: cudaStreamWaitEvent(text_ready) failed");
        }
        FT_TRY(launch_cast(text, 2, S.text16, 0, n.RL * n.E, s2));
        FT_TRY(gemm_nt(s2, n.RL, n.A, n.E, S.text16, n.E, F.w.wk, n.E, S.Kp, n.A));
        FT_TRY(gemm_nt(s2, n.RL, n.A, n.E, S.text16, n.E, F.w.wv, n.E, S.Vp, n.A));
        return 0;
    };
    if (n.T >= kAttnChunk + 64) {
        const int CH = kAttnChunk;
        auto xa = [&](cudaStream_t s2, int t0, int t1) {              // attention-LSTM input projection of steps [t0, t1) -> F.X1 rows
            const long long r0 = static_cast<long long>(t0) * n.B, rows = static_cast<long long>(t1 - t0) * n.B;
            return gemm_nt(s2, rows, G, n.M, S.mel_in16 + r0 * n.M, n.M, F.w.w_ih_a, n.M, F.X1 + r0 * G, G, nullptr, 0,
                           w.attn_lstm_b_ih, w.attn_lstm_b_hh);
        };
        cudaStream_t sr = pp->sA;                                    // the attention LSTM's stream
        FT_TRY(order(pp->ev0, st, {sr, pp->sB, pp->sC}));
        FT_TRY(kv_projections(pp->sC));
        FT_TRY(xa(sr, 0, CH < n.T ? CH : n.T));
        for (int t0 = 0; t0 < n.T; t0 += CH) {
            const int t1 = t0 + CH < n.T ? t0 + CH : n.T;
            if (t1 < n.T) FT_TRY(xa(pp->sB, t1, t1 + CH < n.T ? t1 + CH : n.T));   // next chunk's projection, one chunk ahead
            FT_TRY(launch_lstm_fwd_chunk(n.T, n.B, t0, t1, F.X1, F.w.w_hh_a, out_lens, S.d16, n.D, S.gatesA, S.cA, F.flags, sr, F.hA32, H));
            FT_TRY(order(pp->evA, sr, {pp->sC}));
            if (t1 < n.T) FT_TRY(order(pp->evB, pp->sB, {sr}));      // the next launch on sr needs its projection
            FT_TRY(attention_rows(pp->sC, t0, t1));
            const long long r0 = static_cast<long long>(t0) * n.B, rows = static_cast<long long>(t1 - t0) * n.B;
            FT_TRY(gemm_nt(pp->sC, rows, G, n.D, S.d16 + r0 * n.D, n.D, F.w.w_ih0, n.D, F.X + r0 * G, G, nullptr, 0, w.lstm_b_ih0,
                           w.lstm_b_hh0));
        }
        FT_TRY(order(pp->evG, pp->sC, {st}));
        FT_TRY(order(pp->evJ, sr, {st}));
    } else {
        // attention_lstm: the 80-channel input projection is folded into the persistent recurrence (no [R,4096] projection
        // tensor: one GEMM and 1 GB of HBM traffic less per flow); h lands in d16[:, 0:H].
        FT_TRY(launch_lstm_fwd_xin(n.T, n.B, S.mel_in16, n.M, n.M, F.w.w_ih_a, w.attn_lstm_b_ih, w.attn_lstm_b_hh, F.w.w_hh_a, out_lens,
                                   S.d16, n.D, S.gatesA, S.cA, F.hA32, H, F.flags, st));
        // attention: K/V/Q projections, fused score+softmax(+prior)+context; ctx lands in d16[:, H:H+A]
        FT_TRY(kv_projections(st));
        FT_TRY(attention_rows(st, 0, n.T));
        FT_TRY(gemm_nt(st, n.R, G, n.D, S.d16, n.D, F.w.w_ih0, n.D, F.X, G, nullptr, 0, w.lstm_b_ih0, w.lstm_b_hh0));
    }

    // 2-layer lstm: layer 1 at step t needs layer 0 only up to t, so the two recurrences run as two 64-CTA kernels one chunk
    // apart: sA = layer 0, sC = layer-1 input projection of a finished chunk, sB = layer 1.
    const int CH = layer_chunk(n.T);
    int* flagsA = F.flags;
    int* flagsB = F.flags + static_cast<size_t>(CH) * 16;
    cudaStream_t sr = pp->sA;                                    // layer 0's recurrence stream
    FT_TRY(order(pp->ev0, st, {sr, pp->sB, pp->sC}));
    for (int t0 = 0; t0 < n.T; t0 += CH) {
        const int t1 = t0 + CH < n.T ? t0 + CH : n.T;
        const long long r0 = static_cast<long long>(t0) * n.B, rows = static_cast<long long>(t1 - t0) * n.B;
        FT_TRY(launch_lstm_fwd_chunk(n.T, n.B, t0, t1, F.X, F.w.w_hh0, out_lens, S.h0_16, H, S.gates0, S.c0, flagsA, sr));
        FT_TRY(order(pp->evA, sr, {pp->sC}));
        FT_TRY(gemm_nt(pp->sC, rows, G, H, S.h0_16 + r0 * H, H, F.w.w_ih1, H, F.X1 + r0 * G, G, nullptr, 0, w.lstm_b_ih1, w.lstm_b_hh1));
        FT_TRY(order(pp->evG, pp->sC, {pp->sB}));
        FT_TRY(launch_lstm_fwd_chunk(n.T, n.B, t0, t1, F.X1, F.w.w_hh1, out_lens, S.h1_16, H, S.gates1, S.c1, flagsB, pp->sB));
    }
    FT_TRY(order(pp->evB, pp->sB, {st}));
    FT_TRY(order(pp->evJ, sr, {st}));

    // dense x2 (tanh fused in the GEMM epilogue), 1x1 conv, affine coupling
    FT_TRY(gemm_nt(st, n.R, H, H, S.h1_16, H, F.w.w1, H, nullptr, 0, S.y1_16, H, w.dense_b0, nullptr, 1));
    FT_TRY(gemm_nt(st, n.R, H, H, S.y1_16, H, F.w.w2, H, nullptr, 0, S.y2_16, H, w.dense_b1, nullptr, 1));
    FT_TRY(gemm_nt(st, n.R, 2 * n.M, H, S.y2_16, H, F.w.wc, H, S.o32, 2 * n.M, nullptr, 0, w.conv_b));
    FT_TRY(launch_affine_fwd(S.o32, mel_flow, out_lens, n.T, n.B, n.M, d.reversed, mel_out, log_s, st));
    return 0;
}

// =================================================================================================== backward
// The gradient of both LSTM biases is the column sum of dG: one column sum into whichever of the two is wanted, copied to
// the other when both are.
static int lstm_bias_grads(const uint16_t* dG, long long R, float* db_ih, float* db_hh, const float* iS, cudaStream_t st) {
    float* first = db_ih ? db_ih : db_hh;
    if (first) FT_TRY(launch_colsum(dG, 0, G, R, G, first, iS, st));
    if (db_ih && db_hh) FT_CU(cudaMemcpyAsync(db_hh, db_ih, sizeof(float) * G, cudaMemcpyDeviceToDevice, st), "ar_step");
    return 0;
}

// Main part: everything except the attention LSTM.  Outputs d_text and every parameter gradient but attention_lstm's; leaves
// dhA / dmel_flow / the loss scale in `carry` for ar_step_bwd_attn.  Runs the stages of bwd_plan only.
int ar_step_bwd_main(const FtArStepDesc& d, const FtArStepWeights& w, const float* mel, const int* in_lens, const int* out_lens,
                     const float* attn, const float* d_mel_out, const float* d_log_s, const float* d_gates, const float* d_attn,
                     const float* d_logprob, float* d_text, const FtArStepWeights& g, void* saved, void* scratch, void* carry,
                     cudaStream_t st) {
    FT_TRY(check_desc(d));
    const Dims n(d);
    const unsigned m = bwd_plan(d, g, d_text != nullptr, !d.no_d_mel);
    Workspace ps; ps.base = static_cast<uint8_t*>(saved);
    Saved S_; S_.plan(ps, d);
    Workspace pb; pb.base = static_cast<uint8_t*>(scratch);
    BwdScratch F; F.plan(pb, d);
    Workspace pc; pc.base = static_cast<uint8_t*>(carry);
    BwdCarry C; C.plan(pc, d);
    const float* mel_flow = d.reversed ? S_.mel_flow : mel;
    const long long R = n.R, RL = n.RL, Rm = n.R - n.B;     // Rm: rows with a predecessor step

    // fp16 operand copies: natural layouts for dgrad (B operand MN-major), transposed recurrent weights for BPTT
    if (m & FT_BWD_LSTM0) FT_TRY(launch_cast(w.lstm_w_ih0, 2, F.w.w_ih0, 0, static_cast<long long>(G) * n.D, st));
    if (m & FT_BWD_LSTM0) FT_TRY(launch_cast(w.lstm_w_ih1, 2, F.w.w_ih1, 0, static_cast<long long>(G) * H, st));
    if (m & FT_BWD_QUERY_DGRAD) FT_TRY(launch_cast(w.att_query, 2, F.w.wq, 0, static_cast<long long>(n.A) * H, st));
    if (m & FT_BWD_D_TEXT) FT_TRY(launch_cast(w.att_key, 2, F.w.wk, 0, static_cast<long long>(n.A) * n.E, st));
    if (m & FT_BWD_D_TEXT) FT_TRY(launch_cast(w.att_value, 2, F.w.wv, 0, static_cast<long long>(n.A) * n.E, st));
    if (m & FT_BWD_DENSE0_DGRAD) FT_TRY(launch_cast(w.dense_w0, 2, F.w.w1, 0, static_cast<long long>(H) * H, st));
    if (m & FT_BWD_DENSE1_DGRAD) FT_TRY(launch_cast(w.dense_w1, 2, F.w.w2, 0, static_cast<long long>(H) * H, st));
    if (m & FT_BWD_CONV_DGRAD) FT_TRY(launch_cast(w.conv_w, 2, F.w.wc, 0, static_cast<long long>(2 * n.M) * H, st));
    if (m & FT_BWD_LSTM0) FT_TRY(launch_transpose_cast_f16(w.lstm_w_hh0, F.w.w_hh0, G, H, st));
    if (m & FT_BWD_LSTM1) FT_TRY(launch_transpose_cast_f16(w.lstm_w_hh1, F.w.w_hh1, G, H, st));

    // 0. loss scale for this flow's backward: S = 2^k with S * max|incoming grad| ~ 64 (device-side, no host sync)
    const long long RM = R * n.M;
    const long long BTL = static_cast<long long>(n.B) * n.T * n.L;
    if (m & FT_BWD_COUPLING)
        FT_TRY(launch_grad_scale(d_mel_out, d_mel_out ? RM : 0, d_log_s, d_log_s ? RM : 0, d_gates, d_gates ? R : 0, 64.f, C.scale,
                                 st, d_attn, d_attn ? BTL : 0, d_logprob, d_logprob ? BTL : 0));
    const float* S = C.scale;            // S[0] = scale, S[1] = 1/scale
    const float* iS = C.scale + 1;

    Streams* pp = get_streams(st);
    if (!pp) return ft_set_error("ar_step_bwd: could not create the pipeline streams");
    const cudaStream_t ss = pp->side;

    // 1. affine coupling (scales the incoming gradients by S)
    if (m & FT_BWD_COUPLING)
        FT_TRY(launch_affine_bwd(d_mel_out, d_log_s, S_.o32, mel_flow, out_lens, n.T, n.B, n.M, d.reversed, F.do16, C.dmel_flow, S, st));

    // 2. 1x1 conv     (weight / bias gradients go to the side stream, the dgrad chain stays on `st`)
    FT_TRY(fork_side(pp, st));
    if (g.conv_w) FT_TRY(gemm_wgrad(ss, 2 * n.M, H, R, F.do16, 2 * n.M, S_.y2_16, H, g.conv_w, H, iS));
    if (g.conv_b) FT_TRY(launch_colsum(F.do16, 0, 2 * n.M, R, 2 * n.M, g.conv_b, iS, ss));
    if (m & FT_BWD_CONV_DGRAD)
        FT_TRY(gemm_dgrad(st, R, H, 2 * n.M, F.do16, 2 * n.M, F.w.wc, H, nullptr, 0, F.dy2, H, 0, nullptr, S_.y2_16, H));     // * (1 - y2^2)

    // 3. dense layer 1 (second linear)
    FT_TRY(fork_side(pp, st));
    if (g.dense_w1) FT_TRY(gemm_wgrad(ss, H, H, R, F.dy2, H, S_.y1_16, H, g.dense_w1, H, iS));
    if (g.dense_b1) FT_TRY(launch_colsum(F.dy2, 0, H, R, H, g.dense_b1, iS, ss));
    if (m & FT_BWD_DENSE1_DGRAD)
        FT_TRY(gemm_dgrad(st, R, H, H, F.dy2, H, F.w.w2, H, nullptr, 0, F.dy1, H, 0, nullptr, S_.y1_16, H));               // * (1 - y1^2)

    // 4. dense layer 0
    FT_TRY(fork_side(pp, st));
    if (g.dense_w0) FT_TRY(gemm_wgrad(ss, H, H, R, F.dy1, H, S_.h1_16, H, g.dense_w0, H, iS));
    if (g.dense_b0) FT_TRY(launch_colsum(F.dy1, 0, H, R, H, g.dense_b0, iS, ss));
    if (m & FT_BWD_DENSE0_DGRAD) FT_TRY(gemm_dgrad(st, R, H, H, F.dy1, H, F.w.w1, H, F.dh, H));

    if (m & FT_BWD_ATTN) {
        FT_CU(cudaMemsetAsync(F.dK, 0, sizeof(float) * RL * n.A, st), "ar_step");
        FT_CU(cudaMemsetAsync(F.dV, 0, sizeof(float) * RL * n.A, st), "ar_step");
    }
    if (g.att_v) FT_CU(cudaMemsetAsync(g.att_v, 0, sizeof(float) * n.A, st), "ar_step");
    if (m & FT_BWD_G_GATE) {
        if (g.gate_w) FT_CU(cudaMemsetAsync(g.gate_w, 0, sizeof(float) * n.D, st), "ar_step");
        if (g.gate_b) FT_CU(cudaMemsetAsync(g.gate_b, 0, sizeof(float), st), "ar_step");
    }
    // 5 + 6. lstm layers 1 and 0: BPTT of layer 1 (sA) and layer 0 (sB) one chunk apart; the layer-1 dgrad of a finished chunk
    // (sC) turns dG1 rows into layer 0's incoming dh rows (F.dh is reused row-disjointly: layer 1 only reads rows below the
    // chunk it has finished).  Highest chunk first.
    if (m & FT_BWD_LSTM1) {
        const bool l0 = (m & FT_BWD_LSTM0) != 0;
        const int CH = layer_chunk(n.T);
        int* flagsA = F.flags;
        int* flagsB = F.flags + static_cast<size_t>(CH) * 128;
        cudaStream_t sr = pp->sA;                                    // layer 1's BPTT stream
        FT_TRY(order(pp->ev0, st, {sr, pp->sB, pp->sC}));
        const int n_chunks = (n.T + CH - 1) / CH;
        for (int c = n_chunks - 1; c >= 0; --c) {
            const int t0 = c * CH, t1 = t0 + CH < n.T ? t0 + CH : n.T;
            const long long r0 = static_cast<long long>(t0) * n.B, rows = static_cast<long long>(t1 - t0) * n.B;
            FT_TRY(launch_lstm_bwd_chunk(n.T, n.B, t0, t1, F.dh, H, F.w.w_hh1, S_.gates1, S_.c1, out_lens, F.dG1, F.dcarry1, flagsA, F.xchg1, sr));
            if (!l0) continue;
            FT_TRY(order(pp->evA, sr, {pp->sC}));
            FT_TRY(gemm_dgrad(pp->sC, rows, H, G, F.dG1 + r0 * G, G, F.w.w_ih1, H, F.dh + r0 * H, H));
            FT_TRY(order(pp->evG, pp->sC, {pp->sB}));
            FT_TRY(launch_lstm_bwd_chunk(n.T, n.B, t0, t1, F.dh, H, F.w.w_hh0, S_.gates0, S_.c0, out_lens, F.dG0, F.dcarry0, flagsB, F.xchg0, pp->sB));
        }
        // layer-1 weight gradients run under the tail of layer 0 (side stream forks from st = all of layer 1 done)
        FT_TRY(order(pp->evJ, sr, {st}));
        FT_TRY(fork_side(pp, st));
        if (g.lstm_w_hh1) FT_TRY(gemm_wgrad(ss, G, H, Rm, F.dG1 + static_cast<size_t>(n.B) * G, G, S_.h1_16, H, g.lstm_w_hh1, H, iS));
        if (g.lstm_w_ih1) FT_TRY(gemm_wgrad(ss, G, H, R, F.dG1, G, S_.h0_16, H, g.lstm_w_ih1, H, iS));
        FT_TRY(lstm_bias_grads(F.dG1, R, g.lstm_b_ih1, g.lstm_b_hh1, iS, ss));
        if (l0) FT_TRY(order(pp->evB, pp->sB, {st}));
    }
    // (the weight gradients of lstm layer 0 and of the attention projections are launched by ar_step_bwd_attn, on the side
    //  stream underneath the attention LSTM's BPTT: dG0, dQ16, dK16, dV16 stay in the scratch area until then)
    // 6b. lstm layer 0's input gradient: dd = [dhA ; dctx]
    if (m & FT_BWD_LSTM0) FT_TRY(gemm_dgrad(st, R, n.D, G, F.dG0, G, F.w.w_ih0, n.D, C.dd, n.D));
    // 7. gate layer (last flow only): dd is in the scaled domain, the gate's own parameter gradients are not.  A frozen gate
    //    still adds its term to dd; with dd unused, only the parameter gradients are computed.
    if ((m & (FT_BWD_GATE_DD | FT_BWD_G_GATE)) && d_gates) {
        float* dwg = g.gate_w ? g.gate_w : F.sink + n.A;
        float* dbg = g.gate_b ? g.gate_b : F.sink + n.A + n.D;
        FT_TRY(launch_gate_bwd(S_.d16, n.D, n.D, w.gate_w, d_gates, R, (m & FT_BWD_GATE_DD) ? C.dd : nullptr, n.D, dwg, dbg,
                               (m & FT_BWD_GATE_DD) ? S : nullptr, st));
    }
    // 8. attention (score/softmax/context) with tanh recompute; dK / dV / dv accumulate
    if (m & FT_BWD_ATTN) {
        AttnBwdArgs a;
        a.T = n.T; a.B = n.B; a.L = n.L; a.A = n.A;
        a.Q = S_.Q; a.ldq = n.A; a.K = S_.Kp; a.ldk = n.A; a.V = S_.Vp; a.ldv = n.A; a.v = w.att_v;
        a.in_lens = in_lens; a.out_lens = out_lens; a.attn = attn; a.p_save = S_.p_save; a.temperature = d.temperature;
        a.dctx = C.dd + H; a.lddc = n.D; a.dattn_ext = d_attn; a.dlp_ext = d_logprob; a.scale = S;
        a.dQ = F.dQ; a.lddq = n.A; a.dK = F.dK; a.lddk = n.A; a.dV = F.dV; a.lddv = n.A; a.dv = g.att_v ? g.att_v : F.sink;
        a.t_begin = 0; a.t_end = n.T; a.rows = F.attn_rows;
        FT_TRY(launch_attn_bwd(a, st));
    }
    // 9a. query projection (d16 = [hA ; ctx] saved in fp16, row pitch D)
    if (m & (FT_BWD_QUERY_DGRAD | FT_BWD_G_QUERY)) FT_TRY(launch_cast(F.dQ, 2, F.dQ16, 0, R * n.A, st));
    if (m & FT_BWD_QUERY_DGRAD)
        FT_TRY(gemm_dgrad(st, R, H, n.A, F.dQ16, n.A, F.w.wq, H, C.dd, n.D, nullptr, 0, 1));   // dhA += dQ Wq

    // 9b. key / value projections -> d_text
    if (m & (FT_BWD_D_TEXT | FT_BWD_G_KEY)) FT_TRY(launch_cast(F.dK, 2, F.dK16, 0, RL * n.A, st));
    if (m & (FT_BWD_D_TEXT | FT_BWD_G_VALUE)) FT_TRY(launch_cast(F.dV, 2, F.dV16, 0, RL * n.A, st));
    if (m & FT_BWD_D_TEXT) {
        FT_TRY(gemm_dgrad(st, RL, n.E, n.A, F.dK16, n.A, F.w.wk, n.E, d_text, n.E, nullptr, 0, 0, iS));
        FT_TRY(gemm_dgrad(st, RL, n.E, n.A, F.dV16, n.A, F.w.wv, n.E, d_text, n.E, nullptr, 0, 1, iS));
    }

    return join_side(pp, st);            // everything this call launched is ordered before what the caller enqueues next
}

// Attention-LSTM part: BPTT over dhA (carry), its weight gradients, and the input gradient d_mel (coupling path from carry +
// the shifted attention-LSTM path, back to natural time, loss scale undone).  The stages it runs depend on `g` and
// d.no_d_mel only, so the plan matches the one ar_step_bwd_main ran whatever d_text was.
int ar_step_bwd_attn(const FtArStepDesc& d, const FtArStepWeights& w, const int* out_lens, float* d_mel, const FtArStepWeights& g,
                     void* saved, void* scratch, void* carry, cudaStream_t st) {
    FT_TRY(check_desc(d));
    const Dims n(d);
    const unsigned m = bwd_plan(d, g, false, !d.no_d_mel);
    Workspace ps; ps.base = static_cast<uint8_t*>(saved);
    Saved S_; S_.plan(ps, d);
    Workspace pb; pb.base = static_cast<uint8_t*>(scratch);
    BwdScratch F; F.plan(pb, d);
    Workspace pc; pc.base = static_cast<uint8_t*>(carry);
    BwdCarry C; C.plan(pc, d);
    const long long R = n.R, Rm = n.R - n.B;
    const float* iS = C.scale + 1;
    Streams* pp = get_streams(st);
    if (!pp) return ft_set_error("ar_step_bwd: could not create the pipeline streams");
    const cudaStream_t ss = pp->side;
    const long long RL = n.RL;
    if (m & FT_BWD_D_MEL) FT_TRY(launch_cast(w.attn_lstm_w_ih, 2, F.w.w_ih_a, 0, static_cast<long long>(G) * n.M, st));
    if (m & FT_BWD_ATTN_LSTM) FT_TRY(launch_transpose_cast_f16(w.attn_lstm_w_hh, F.w.w_hh_a, G, H, st));

    // deferred from ar_step_bwd_main: weight gradients of lstm layer 0 and of the attention projections, on the side stream,
    // underneath the BPTT kernel below (64 of the SMs)
    FT_TRY(fork_side(pp, st));
    if (g.lstm_w_hh0) FT_TRY(gemm_wgrad(ss, G, H, Rm, F.dG0 + static_cast<size_t>(n.B) * G, G, S_.h0_16, H, g.lstm_w_hh0, H, iS));
    if (g.lstm_w_ih0) FT_TRY(gemm_wgrad(ss, G, n.D, R, F.dG0, G, S_.d16, n.D, g.lstm_w_ih0, n.D, iS));
    FT_TRY(lstm_bias_grads(F.dG0, R, g.lstm_b_ih0, g.lstm_b_hh0, iS, ss));
    if (g.att_query) FT_TRY(gemm_wgrad(ss, n.A, H, R, F.dQ16, n.A, S_.d16, n.D, g.att_query, H, iS));
    if (g.att_key) FT_TRY(gemm_wgrad(ss, n.A, n.E, RL, F.dK16, n.A, S_.text16, n.E, g.att_key, n.E, iS));
    if (g.att_value) FT_TRY(gemm_wgrad(ss, n.A, n.E, RL, F.dV16, n.A, S_.text16, n.E, g.att_value, n.E, iS));

    // 10. attention_lstm  (dhA = C.dd[:, 0:H], pitch D)
    if (m & FT_BWD_ATTN_LSTM) FT_TRY(launch_lstm_bwd(n.T, n.B, C.dd, n.D, F.w.w_hh_a, S_.gatesA, S_.cA, out_lens, F.dGa, F.flags, st));
    FT_TRY(fork_side(pp, st));
    if (g.attn_lstm_w_hh)
        FT_TRY(gemm_wgrad(ss, G, H, Rm, F.dGa + static_cast<size_t>(n.B) * G, G, S_.d16, n.D, g.attn_lstm_w_hh, H, iS));
    if (g.attn_lstm_w_ih) FT_TRY(gemm_wgrad(ss, G, n.M, R, F.dGa, G, S_.mel_in16, n.M, g.attn_lstm_w_ih, n.M, iS));
    FT_TRY(lstm_bias_grads(F.dGa, R, g.attn_lstm_b_ih, g.attn_lstm_b_hh, iS, ss));
    if (m & FT_BWD_D_MEL) FT_TRY(gemm_dgrad(st, R, n.M, G, F.dGa, G, F.w.w_ih_a, n.M, F.dmel_in, n.M));

    // 11. input gradient: coupling path + (shifted) attention_lstm path, back to natural time, loss scale undone
    if ((m & FT_BWD_D_MEL) && d_mel)
        FT_TRY(launch_combine_dmel(C.dmel_flow, F.dmel_in, out_lens, n.T, n.B, n.M, d.reversed, d_mel, iS, st));
    return join_side(pp, st);            // everything this call launched is ordered before what the caller enqueues next
}

}  // namespace ft

// =================================================================================================== C ABI
extern "C" {

size_t ft_ar_step_saved_bytes(const FtArStepDesc* d) {
    ft::Workspace p; ft::Saved s; s.plan(p, *d);
    return p.off + 256;
}
size_t ft_ar_step_bwd_carry_bytes(const FtArStepDesc* d) {
    ft::Workspace pc; ft::BwdCarry c; c.plan(pc, *d);
    return pc.off + 256;
}
size_t ft_ar_step_scratch_bytes(const FtArStepDesc* d) {
    ft::Workspace pf; ft::FwdScratch f; f.plan(pf, *d);
    ft::Workspace pb; ft::BwdScratch b; b.plan(pb, *d);
    // the one-call backward (ft_ar_step_bwd) places its carry area behind the backward scratch
    const size_t bwd = ((pb.off + 255) & ~static_cast<size_t>(255)) + ft_ar_step_bwd_carry_bytes(d);
    return (pf.off > bwd ? pf.off : bwd) + 256;
}
int ft_ar_step_saved_lookup(const FtArStepDesc* d, const char* name, size_t* offset, size_t* bytes) {
    std::vector<ft::Region> regs;
    ft::Workspace p; p.regs = &regs;
    ft::Saved s; s.plan(p, *d);
    for (const auto& r : regs)
        if (std::strcmp(r.name, name) == 0) { *offset = r.off; *bytes = r.bytes; return 0; }
    return ft::ft_set_error("ft_ar_step_saved_lookup: unknown region");
}

int ft_ar_step_fwd(const FtArStepDesc* d, const FtArStepWeights* w, const float* mel, const float* text,
                   const int* in_lens, const int* out_lens, const float* attn_prior, float* mel_out, float* log_s,
                   float* gates, float* attn, float* attn_logprob, void* saved, void* scratch, void* text_ready_event,
                   void* stream) {
    if (!d || !w || !mel || !text || !mel_out || !log_s || !attn || !attn_logprob || !saved || !scratch)
        return ft::ft_set_error("ft_ar_step_fwd: NULL argument");
    return ft::ar_step_fwd(*d, *w, mel, text, in_lens, out_lens, attn_prior, mel_out, log_s, gates, attn, attn_logprob,
                           saved, scratch, static_cast<cudaEvent_t>(text_ready_event), static_cast<cudaStream_t>(stream));
}

int ft_ar_step_bwd(const FtArStepDesc* d, const FtArStepWeights* w, const float* mel, const int* in_lens,
                   const int* out_lens, const float* attn, const float* d_mel_out, const float* d_log_s,
                   const float* d_gates, const float* d_attn, const float* d_attn_logprob, float* d_mel, float* d_text,
                   const FtArStepWeights* g, void* saved, void* scratch, void* stream) {
    if (!d || !w || !mel || !attn || !g || !saved || !scratch) return ft::ft_set_error("ft_ar_step_bwd: NULL argument");
    ft::Workspace pb; ft::BwdScratch b; b.plan(pb, *d);
    void* carry = static_cast<uint8_t*>(scratch) + ((pb.off + 255) & ~static_cast<size_t>(255));
    FtArStepDesc dd = *d;
    if (!d_mel) dd.no_d_mel = 1;
    if (ft::ar_step_bwd_main(dd, *w, mel, in_lens, out_lens, attn, d_mel_out, d_log_s, d_gates, d_attn, d_attn_logprob, d_text, *g,
                             saved, scratch, carry, static_cast<cudaStream_t>(stream)) != 0) return -1;
    return ft::ar_step_bwd_attn(dd, *w, out_lens, d_mel, *g, saved, scratch, carry, static_cast<cudaStream_t>(stream));
}

int ft_ar_step_bwd_main(const FtArStepDesc* d, const FtArStepWeights* w, const float* mel, const int* in_lens,
                        const int* out_lens, const float* attn, const float* d_mel_out, const float* d_log_s,
                        const float* d_gates, const float* d_attn, const float* d_attn_logprob, float* d_text,
                        const FtArStepWeights* g, void* saved, void* scratch, void* carry, void* stream) {
    if (!d || !w || !mel || !attn || !g || !saved || !scratch || !carry) return ft::ft_set_error("ft_ar_step_bwd_main: NULL argument");
    return ft::ar_step_bwd_main(*d, *w, mel, in_lens, out_lens, attn, d_mel_out, d_log_s, d_gates, d_attn, d_attn_logprob, d_text,
                                *g, saved, scratch, carry, static_cast<cudaStream_t>(stream));
}

int ft_ar_step_bwd_attn_lstm(const FtArStepDesc* d, const FtArStepWeights* w, const int* out_lens, float* d_mel,
                             const FtArStepWeights* g, void* saved, void* scratch, void* carry, void* stream) {
    if (!d || !w || !g || !saved || !scratch || !carry) return ft::ft_set_error("ft_ar_step_bwd_attn_lstm: NULL argument");
    return ft::ar_step_bwd_attn(*d, *w, out_lens, d_mel, *g, saved, scratch, carry, static_cast<cudaStream_t>(stream));
}

int ft_ar_step_bwd_plan(const FtArStepDesc* d, const FtArStepWeights* grads, int want_d_text, int want_d_mel, unsigned* stages) {
    if (!d || !grads || !stages) return ft::ft_set_error("ft_ar_step_bwd_plan: NULL argument");
    *stages = ft::bwd_plan(*d, *grads, want_d_text != 0, want_d_mel != 0);
    return 0;
}

int ft_nll_reduce(const float* z, const float* const* log_s_list, int n_flows, const float* gate,
                  const float* gate_target, const int* out_lens, int T, int B, int M, float* sums, void* stream) {
    return ft::launch_nll_reduce(z, log_s_list, n_flows, gate, gate_target, out_lens, T, B, M, sums,
                                 static_cast<cudaStream_t>(stream));
}
int ft_nll_rows(const float* z, const float* const* log_s_list, int n_flows, const float* gate,
                const float* gate_target, const int* out_lens, int T, int B, int M, float* rows_out, void* stream) {
    return ft::launch_nll_rows(z, log_s_list, n_flows, gate, gate_target, out_lens, T, B, M, rows_out,
                               static_cast<cudaStream_t>(stream));
}
int ft_nll_grad(const float* z, const float* gate, const float* gate_target, const int* out_lens, int T, int B, int M,
                float sigma, const float* sums, const float* g_nll, const float* g_gate, float* dz, float* dlog_s,
                float* dgate, void* stream) {
    return ft::launch_nll_grad(z, gate, gate_target, out_lens, T, B, M, sigma, sums, g_nll, g_gate, dz, dlog_s, dgate,
                               static_cast<cudaStream_t>(stream));
}

}  // extern "C"
