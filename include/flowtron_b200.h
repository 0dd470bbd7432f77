/* flowtron_b200 — C ABI of the H100-native Flowtron hot path (libflowtron_b200.so).
 *
 * The reference (NVIDIA/flowtron) has no FFI: the hot path sits behind Python nn.Modules.  These entry
 * points are what a binding for that path replaces; each cites the reference interface it stands for.
 * Conventions: all pointers are DEVICE pointers owned by the caller (torch's allocator in the shipped
 * host layer); no entry point allocates, synchronises the stream, or touches the default stream unless
 * `stream` is 0; return 0 on success, negative on error (message in ft_last_error()).  Weights are
 * passed in PyTorch's native layouts ([4H, in], gate order i,f,g,o) so checkpoints need no conversion.
 */
#ifndef FLOWTRON_B200_H
#define FLOWTRON_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* element formats */
#define FT_F16 0
#define FT_BF16 1
#define FT_TF32 2   /* fp32 storage, tf32 tensor-core math */

/* Longest text (tokens, the padded L of FtArStepDesc) the flow-step kernels take, training and inference.  Texts of up to
 * 256 tokens run the short-text kernel variants; longer ones the long-text variants (DESIGN.md 4.16).  The Python layer
 * mirrors it as flowtron_b200._lib.MAX_TEXT_LEN; ft_max_text_len() returns it. */
#define FT_MAX_TEXT_LEN 1024

int ft_version(void);
int ft_max_text_len(void);
const char* ft_last_error(void);
/* 0 = ok; non-zero = code written by a device-side watchdog (a bounded spin-wait expired). Synchronises. */
int ft_device_status(void);
/* Optional per-kernel device timing with CUDA events on the launching stream (bench.py roofline leg). */
void ft_timing_enable(int on);
void ft_timing_reset(void);
int ft_timing_report(char* buf, int cap);   /* synchronises; "name m n k count total_ms" per line */
/* number of kernels this library has launched (bench.py's gpu_launches) */
long long ft_launch_count(void);
void ft_reset_launch_count(void);

/* C[M,N] = act(alpha * A[M,K] B[N,K]^T + bias + bias2) (+ C32 if beta).  wgmma/TMA GEMM.
 * a_mn / b_mn = 1: operand is given MN-major, i.e. A points at a row-major [K, M] tensor.
 * Replaces: nn.Linear / Conv1d(k=1) / LSTM input projections (flowtron.py:278-288, 651, 654-655) and
 * their autograd dgrad / wgrad. */
int ft_gemm(int M, int N, int K, const void* A, long long lda, int a_fmt, int a_mn, const void* B, long long ldb,
            int b_fmt, int b_mn, const float* bias, const float* bias2, int act, int beta, float alpha, float* C32,
            long long ldc32, void* C16, long long ldc16, int c16_fmt, void* stream);

/* One nn.LSTM layer recurrence, hidden size 1024 (flowtron.py:654-655 `lstm` / `attention_lstm`, run via
 * run_padded_sequence :671-695).  xproj = W_ih x + b_ih + b_hh for all T*B rows (row = t*B + b), fp32
 * [T*B, 4096], gate order i,f,g,o.  whh16: fp16 copy of weight_hh [4096,1024].  Writes h (fp16, zero at
 * t >= lens[b]) to hseq16 [T*B, ldh] and, when non-null, the post-activation gates (fp16 [T*B,4096]) and
 * cell state (fp32 [T*B,1024]) needed by ft_lstm_bwd.  flags: int scratch [T*16].  B <= 32.  Runs the 64-CTA
 * recurrence kernel (16 hidden units per CTA). */
int ft_lstm_fwd(int T, int B, const float* xproj, const void* whh16, const int* lens, void* hseq16, long long ldh,
                void* gates16, float* cstate, float* h32, long long ldh32, int* flags, void* stream);

/* debug/profiling: device buffer [T][16] that receives clock64 stamps of CTA 0 of later ft_lstm_fwd launches */
void ft_debug_set_lstm_trace(long long* buf);
/* same for ft_ar_step_infer: [T][32] stamps of CTA 0 (phase boundaries, tools/trace_infer.py) */
void ft_debug_set_infer_trace(long long* buf);
/* debug: 4-CTA clusters of the BPTT cluster kernel that fit on the device at once, at its launch configuration for
 * batch B (cudaOccupancyMaxActiveClusters); -1 on error */
int ft_debug_lstm_bwd_max_clusters(int B);
/* debug: steps [t0, t1) of one BPTT chunk of the layer pipeline (B <= 32), resuming dc*f from / handing it on through
 * dc_carry [B,1024] fp32 and dG_{t1} from dG16.  xchg non-NULL: the flat kernel the pipeline runs (flags [(t1-t0)*128],
 * xchg [2*16*4*B*64] fp32); NULL: the 4-CTA cluster kernel (flags [(t1-t0)*64]).  Both give bit-identical results. */
int ft_debug_lstm_bwd_chunk(int T, int B, int t0, int t1, const float* dh_ext, long long ldd, const void* whhT16,
                            const void* gates16, const float* cstate, const int* lens, void* dG16, float* dc_carry, int* flags,
                            float* xchg, void* stream);

/* ft_gemm tile policy: 0 (default) = one CTA per 128 x 256 tile always; 1 = CTA pairs (2-CTA clusters sharing B by TMA multicast, 256 x 256 tiles) for
 * contractions >= 1e11 FLOP; 2 = CTA pairs whenever the output is wide and has >= SMs/2 such tiles. */
void ft_set_gemm_pair_mode(int mode);

/* BPTT of the same layer (autograd of nn.LSTM).  dh_ext: gradient w.r.t. the layer outputs, fp32
 * [T*B, ldd] (ignored at t >= lens[b]; the caller may pre-multiply it by a power-of-two loss scale).  whhT16:
 * fp16 copy of weight_hh^T [1024,4096].  Writes dG (fp16 [T*B,4096], saturating), the gradient w.r.t. the gate
 * pre-activations; dW_ih, dW_hh, db and dx are GEMMs / column sums over dG done by the caller.
 * flags: int scratch [T*64].  B <= 32. */
int ft_lstm_bwd(int T, int B, const float* dh_ext, long long ldd, const void* whhT16, const void* gates16,
                const float* cstate, const int* lens, void* dG16, int* flags, void* stream);

/* ------------------------------------------------------------------------------------------------------
 * AR_Step / AR_Back_Step (flowtron.py:595-828): one autoregressive flow step, training direction.
 * ---------------------------------------------------------------------------------------------------- */
typedef struct {
    int T, B, L;        /* mel frames (padded max), batch, text tokens (padded max, <= FT_MAX_TEXT_LEN) */
                        /* B <= 32 per training call (ft_ar_step_infer: <= 16)      */
    int n_mel;          /* 80  (n_mel_channels, <= 128)                             */
    int n_hidden;       /* 1024 (must be 1024 in this build)                        */
    int n_attn;         /* 640 (n_attn_channels)                                    */
    int n_text;         /* 640 = n_text_dim + n_speaker_dim                         */
    int reversed;       /* 1 = AR_Back_Step semantics (flowtron.py:605-627)         */
    int has_gate;       /* flow owns gate_layer (last flow only, flowtron.py:854)   */
    int has_prior;      /* attn_prior given                                         */
    float temperature;  /* Attention.temperature (flowtron.py:532, 573)             */
    int no_d_mel;       /* backward: the caller will not read d_mel (ft_ar_step_bwd_plan); ignored by ft_ar_step_infer */
} FtArStepDesc;

/* fp32 device pointers in PyTorch's native layouts == the state_dict entries of one AR_Step
 * (SURVEY.md 8a row 15).  The same struct type carries the parameter gradients in ft_ar_step_bwd. */
typedef struct {
    float *attn_lstm_w_ih, *attn_lstm_w_hh, *attn_lstm_b_ih, *attn_lstm_b_hh;   /* attention_lstm.*_l0  [4H,M] [4H,H] [4H] [4H] */
    float *lstm_w_ih0, *lstm_w_hh0, *lstm_b_ih0, *lstm_b_hh0;                   /* lstm.*_l0            [4H,H+A] [4H,H] ...      */
    float *lstm_w_ih1, *lstm_w_hh1, *lstm_b_ih1, *lstm_b_hh1;                   /* lstm.*_l1            [4H,H] [4H,H] ...        */
    float *att_query, *att_key, *att_value, *att_v;                            /* attention_layer.{query,key,value,v}.linear_layer.weight */
    float *dense_w0, *dense_b0, *dense_w1, *dense_b1;                          /* dense_layer.layers.{0,1}.linear_layer.{weight,bias}     */
    float *conv_w, *conv_b;                                                     /* conv.weight [2M,H,1], conv.bias [2M]                    */
    float *gate_w, *gate_b;                                                     /* gate_layer.linear_layer.{weight,bias} or NULL           */
} FtArStepWeights;

/* Bytes of the two caller-owned work areas: `saved` persists from ft_ar_step_fwd to ft_ar_step_bwd of the
 * same flow; `scratch` is transient and may be shared by all flows on a stream. */
size_t ft_ar_step_saved_bytes(const FtArStepDesc* d);
size_t ft_ar_step_scratch_bytes(const FtArStepDesc* d);
/* Byte offset / size of a named intermediate inside `saved` (debug + tests): returns 0 on success. */
int ft_ar_step_saved_lookup(const FtArStepDesc* d, const char* name, size_t* offset, size_t* bytes);

/* AR_Step.forward / AR_Back_Step.forward (flowtron.py:725-773, 605-627).
 *   mel [T,B,M] f32, text [L,B,E] f32 (encoder outputs), in_lens/out_lens int32 [B] (NULL = no padding),
 *   attn_prior [B,T,L] f32 or NULL  ->  mel_out [T,B,M], log_s [T,B,M], gates [T,B] (NULL if !has_gate),
 *   attn [B,T,L], attn_logprob [B,T,L].  For reversed flows log_s/gates/attn are in flipped time exactly as
 *   the reference returns them.
 *   text_ready_event: a cudaEvent_t recorded on whatever stream produced `text`, or NULL.  The call waits for it right
 *   before it first reads `text` -- i.e. after the attention LSTM, which depends on mel only -- so the caller can run
 *   the text encoder (flowtron.py:871-880) concurrently with the first third of the flow instead of in front of it. */
int ft_ar_step_fwd(const FtArStepDesc* d, const FtArStepWeights* w, const float* mel, const float* text,
                   const int* in_lens, const int* out_lens, const float* attn_prior, float* mel_out, float* log_s,
                   float* gates, float* attn, float* attn_logprob, void* saved, void* scratch, void* text_ready_event,
                   void* stream);

/* Autograd of the above.  Incoming gradients (any may be NULL = zero): d_mel_out, d_log_s [T,B,M], d_gates [T,B],
 * d_attn, d_attn_logprob [B,T,L].  Outputs: d_mel [T,B,M], d_text [L,B,E] (overwritten), parameter gradients
 * into `g` (overwritten; same layouts as the weights).  Every output may be NULL = not wanted: the backward then runs only
 * the stages that a wanted output depends on (ft_ar_step_bwd_plan below); a NULL d_mel here counts as d->no_d_mel. */
int ft_ar_step_bwd(const FtArStepDesc* d, const FtArStepWeights* w, const float* mel, const int* in_lens,
                   const int* out_lens, const float* attn, const float* d_mel_out, const float* d_log_s,
                   const float* d_gates, const float* d_attn, const float* d_attn_logprob, float* d_mel, float* d_text,
                   const FtArStepWeights* g, void* saved, void* scratch, void* stream);

/* The same backward as two calls, so that the caller's autograd can overlap work that depends only on d_text (the text
 * encoder's backward) with the attention LSTM's BPTT (a 64-SM kernel):
 *   ft_ar_step_bwd_main      : everything but the attention LSTM.  Writes d_text and the gradients of conv, dense_layer,
 *                              lstm layer 1 and the gate; leaves dhA / the coupling-path input gradient / the loss scale in
 *                              `carry` (ft_ar_step_bwd_carry_bytes, caller-owned, must survive until the second call) and
 *                              dG0 / dQ / dK / dV in `scratch` (nothing else may use `scratch` in between).
 *   ft_ar_step_bwd_attn_lstm : attention-LSTM BPTT; writes d_mel and the gradients of attention_lstm, lstm layer 0 and the
 *                              attention query / key / value projections (their GEMMs run underneath the BPTT kernel).
 * ft_ar_step_bwd == the two back to back.  ft_ar_step_bwd_main must know whether d_mel will be read before the second call
 * runs: d->no_d_mel = 1 says it will not (ft_ar_step_bwd_attn_lstm then skips the input gradient even for a non-NULL d_mel).
 * d_text and any entry of `g` may be NULL, as for ft_ar_step_bwd. */
size_t ft_ar_step_bwd_carry_bytes(const FtArStepDesc* d);
int ft_ar_step_bwd_main(const FtArStepDesc* d, const FtArStepWeights* w, const float* mel, const int* in_lens,
                        const int* out_lens, const float* attn, const float* d_mel_out, const float* d_log_s,
                        const float* d_gates, const float* d_attn, const float* d_attn_logprob, float* d_text,
                        const FtArStepWeights* g, void* saved, void* scratch, void* carry, void* stream);
int ft_ar_step_bwd_attn_lstm(const FtArStepDesc* d, const FtArStepWeights* w, const int* out_lens, float* d_mel,
                             const FtArStepWeights* g, void* saved, void* scratch, void* carry, void* stream);

/* Which stages of a flow step's backward run, for the wanted outputs: a NULL entry of `grads` is a parameter gradient
 * nobody wants, want_d_text / want_d_mel say whether d_text / d_mel are.  A stage runs when something downstream of it is
 * wanted (FT_BWD_G_* name the weight-gradient work of one parameter group; within a group only the non-NULL entries are
 * computed):
 *   D_MEL                the attention-LSTM dgrad to the input and combine_dmel:   d_mel wanted
 *   ATTN_LSTM            attention-LSTM BPTT:                  D_MEL or G_ATTN_LSTM
 *   QUERY_DGRAD          dhA += dQ Wq:                         ATTN_LSTM
 *   D_TEXT               d_text = dK Wk + dV Wv:               d_text wanted
 *   ATTN                 zero dK / dV, attention backward:     QUERY_DGRAD, D_TEXT, G_QUERY, G_KEY, G_VALUE or G_V
 *   GATE_DD              the gate's term of dd (gated flow):   ATTN or ATTN_LSTM (both read dd)
 *   LSTM0                layer-1 per-chunk dgrad, layer 0 BPTT, dd = dG0 W_ih0:   ATTN, ATTN_LSTM or G_LSTM0
 *   LSTM1                layer 1 BPTT:                         LSTM0 or G_LSTM1
 *   DENSE0_DGRAD         dense layer 0 dgrad (-> layer 1):     LSTM1
 *   DENSE1_DGRAD         dense layer 1 dgrad:                  DENSE0_DGRAD or G_DENSE0
 *   CONV_DGRAD           1x1 conv dgrad:                       DENSE1_DGRAD or G_DENSE1
 *   COUPLING             loss scale + affine coupling backward:   CONV_DGRAD, G_CONV or D_MEL
 *   G_GATE               the gate's parameter gradients (gated flow): a gate entry of `grads` non-NULL.  With GATE_DD off
 *                        it is the whole backward of a gate-only step: one launch, no loss scale.
 * With every gradient, d_text and d_mel wanted all stages run, in the order of the full backward.  The two backward calls
 * branch on this mask and nothing else.  Returns 0, or -1 for a NULL argument. */
enum {
    FT_BWD_COUPLING = 1u << 0, FT_BWD_CONV_DGRAD = 1u << 1, FT_BWD_DENSE1_DGRAD = 1u << 2, FT_BWD_DENSE0_DGRAD = 1u << 3,
    FT_BWD_LSTM1 = 1u << 4, FT_BWD_LSTM0 = 1u << 5, FT_BWD_GATE_DD = 1u << 6, FT_BWD_ATTN = 1u << 7,
    FT_BWD_QUERY_DGRAD = 1u << 8, FT_BWD_D_TEXT = 1u << 9, FT_BWD_ATTN_LSTM = 1u << 10, FT_BWD_D_MEL = 1u << 11,
    FT_BWD_G_CONV = 1u << 16, FT_BWD_G_DENSE1 = 1u << 17, FT_BWD_G_DENSE0 = 1u << 18, FT_BWD_G_LSTM1 = 1u << 19,
    FT_BWD_G_LSTM0 = 1u << 20, FT_BWD_G_QUERY = 1u << 21, FT_BWD_G_KEY = 1u << 22, FT_BWD_G_VALUE = 1u << 23,
    FT_BWD_G_V = 1u << 24, FT_BWD_G_ATTN_LSTM = 1u << 25, FT_BWD_G_GATE = 1u << 26
};
int ft_ar_step_bwd_plan(const FtArStepDesc* d, const FtArStepWeights* grads, int want_d_text, int want_d_mel,
                        unsigned* stages);

/* FlowtronLoss default branch (flowtron.py:205-243): sums[0]=sum (z m)^2, [1]=sum_flows sum log_s m,
 * [2]=sum m BCEWithLogits(gate m, target), [3]=n=sum m.  log_s_list: HOST array of n_flows (<= 16) device pointers (passed
 * to the kernel by value: no upload, so the call can be captured in a CUDA graph). */
int ft_nll_reduce(const float* z, const float* const* log_s_list, int n_flows, const float* gate,
                  const float* gate_target, const int* out_lens, int T, int B, int M, float* sums, void* stream);
/* The same sums per utterance (Flowtron.score): rows_out [B, 4] fp32, row b = {sum z^2, sum_flows sum log_s,
 * sum BCEWithLogits(gate, target), n} over its n = min(out_lens[b], T) frames (gate NULL: entry 2 is 0).  z / log_s
 * [T, B, M], gate [T, B] or NULL, gate_target [B, T].  One CTA per row, fixed summation order, no atomics: a row's values
 * do not depend on B, on the other rows or on T beyond its own length, and replays are bit-identical.  log_s_list as for
 * ft_nll_reduce (host array of device pointers). */
int ft_nll_rows(const float* z, const float* const* log_s_list, int n_flows, const float* gate,
                const float* gate_target, const int* out_lens, int T, int B, int M, float* rows_out, void* stream);
/* Gradients of g_nll*nll + g_gate*gate_loss w.r.t. z, every log_s (identical tensor), gate logits. */
int ft_nll_grad(const float* z, const float* gate, const float* gate_target, const int* out_lens, int T, int B, int M,
                float sigma, const float* sums, const float* g_nll, const float* g_gate, float* dz, float* dlog_s,
                float* dgate, void* stream);

/* Optimizer step of the training loop around the hot path (SURVEY.md 8f "next"): torch.nn.utils.clip_grad_norm_
 * (train.py:324-329) followed by RAdam.step (radam.py:44-122), on flat fp32 device buffers, no host sync.
 *   ft_sumsq_partials: partials[0..1023] = per-block sums of x[i]^2 over x[0..n) (one call per contiguous gradient
 *     segment, each into its own 1024 floats);
 *   ft_clip_coef: norm_coef[0] = sqrt(sum partials) (the total gradient norm clip_grad_norm_ returns),
 *     norm_coef[1] = min(1, max_norm / (norm + 1e-6)) (the factor it multiplies every gradient by);
 *   ft_radam_step: p, m (exp_avg), v (exp_avg_sq) updated in place from g * grad_coef[0] (grad_coef NULL = 1):
 *     v = beta2 v + (1-beta2) g^2; m = beta1 m + (1-beta1) g; p -= weight_decay_lr p (weight_decay*lr, radam.py:109);
 *     use_denom (N_sma >= 5, radam.py:115): p -= step_size m / (sqrt(v) + eps), else p -= step_size m.
 *     N_sma / step_size are the host scalars of radam.py:87-107. */
int ft_sumsq_partials(const float* x, long long n, float* partials, void* stream);
int ft_clip_coef(const float* partials, int n_partials, float max_norm, float* norm_coef, void* stream);
int ft_radam_step(float* p, const float* g, float* m, float* v, long long n, double beta1, double beta2, double eps,
                  double weight_decay_lr, double step_size, int use_denom, const float* grad_coef, void* stream);
/* CUDA-graph-capturable form: the step count lives on the device (step_dev[0] = updates done so far); the kernel derives
 * N_sma / step_size from step_dev[0] + 1 itself (fp64), so a captured step replays with the right schedule.  Call
 * ft_step_increment once after all segments of an optimizer step. */
int ft_radam_step_dev(float* p, const float* g, float* m, float* v, long long n, double beta1, double beta2, double eps,
                      double weight_decay, double lr, const int* step_dev, const float* grad_coef, void* stream);
int ft_step_increment(int* step_dev, void* stream);

/* AR_Step.infer / AR_Back_Step.infer (flowtron.py:775-828, 629-642): sequential inverse of one flow for a padded batch,
 * all T frames in ONE persistent launch.  Row b equals its own B == 1 run on its unpadded inputs.
 *   residual [T,B,M] f32 in NATURAL time order, text [L,B,E] f32; scratch: ft_ar_step_infer_scratch_bytes(d).
 *   in_lens [B] int32 device or NULL (all L): text length of row b; keys l >= in_lens[b] take no part in the softmax and get
 *     attention weight 0.
 *   frame_lens [B] int32 device or NULL (all T): frame budget of row b; row b generates while i < frame_lens[b] and its gate
 *     has not fired; residual rows t >= frame_lens[b] are never read.
 *   d->reversed = 1 (AR_Back_Step): frame i reads residual[frame_lens[b] - 1 - i], and the emitted frames come back flipped
 *     within the row's own n_frames[b], so `out` is in natural time order too.
 *   attn_prior [B,T,L] f32 or NULL (used when d->has_prior): row i is used at generation step i; for a back step the
 *     caller flips it (the reference's torch.flip(attn_prior, (1,))).
 *   attn_forced [B,Ta,L] f32 or NULL: forced alignments (the `attns` argument, flowtron.py:585-588, 797).  Row (b, i) holds
 *     the weights of GENERATION STEP i of utterance b: with d->reversed = 1, step i produces natural frame
 *     frame_lens[b] - 1 - i, the order in which AR_Back_Step.forward returns its attention, so a flow's forward attention
 *     feeds the same flow's inverse with no transpose or flip.  Scoring, softmax and the prior are skipped; context =
 *     weights . V.  Ta >= max frame_lens[b] (>= d->T when frame_lens is NULL); only keys l < in_lens[b] of rows
 *     i < frame_lens[b] are read, every other weight is 0 whatever the buffer holds.
 *   out [T,B,M]: zero at t >= n_frames[b]; attn_out [T,B,L]: the weights used, in generation order, zero at i >= n_frames[b]
 *     and l >= in_lens[b]; n_frames [B] int32 = min(gate stop (the frame that trips the gate is emitted), frame_lens[b]);
 *     a gate_threshold >= 1 disables stopping.
 *   Lengths must satisfy 1 <= in_lens[b] <= L and 1 <= frame_lens[b] <= T; they are read on the device only.
 *   B <= 16, L <= FT_MAX_TEXT_LEN (texts over 256 tokens run the long-text kernel variant, which stages the row of scores in
 *   shared memory).  With B == 1 this is exactly the reference's loop-with-break; B > 1 with a gate is the per-row-stop
 *   extension (the reference raises there, SURVEY.md 3.2).
 *   Two launches (the persistent kernel, then a small per-row flip / attention clear), no allocation, no host
 *   synchronisation: CUDA-graph capturable. */
size_t ft_ar_step_infer_scratch_bytes(const FtArStepDesc* d);
int ft_ar_step_infer(const FtArStepDesc* d, const FtArStepWeights* w, const float* residual, const float* text, const int* in_lens,
                     const int* frame_lens, const float* attn_prior, const float* attn_forced, int Ta, float gate_threshold,
                     float* out, float* attn_out, int* n_frames, void* scratch, void* stream);

/* TacotronSTFT.mel_spectrogram (audio_processing.py:117-134) for a ragged batch.  wav: concatenated utterances
 * (f32 in [-1,1]); sample_offsets / frame_offsets: device int64 [n_utt+1] prefix sums (frames of utterance u =
 * 1 + N_u / hop); window [n_fft] (periodic Hann, centre-padded); mel_basis [n_mel, n_fft/2+1] with its non-zero
 * column range [band_lo[m], band_hi[m]) per row.  mel_out: per-utterance [n_mel, F_u] blocks, concatenated
 * (== [B, n_mel, F] for equal lengths).  scratch: ft_mel_scratch_bytes(n_fft, chunk_frames). */
size_t ft_mel_scratch_bytes(int n_fft, long long chunk_frames);
int ft_mel_spectrogram(const float* wav, const long long* sample_offsets, const long long* frame_offsets, int n_utt,
                       long long total_frames, const float* window, const float* mel_basis, const int* band_lo,
                       const int* band_hi, int n_mel, int n_fft, int hop, float clip, float* mel_out, void* scratch,
                       long long chunk_frames, void* stream);

/* Fused form for n_fft == 1024 (the shipped configuration, config.json:31-33): ONE kernel -- reflect pad + window on the
 * load, a 1024-point real FFT per warp in shared memory, |X|, sparse filterbank, log -- reads the waveform once and writes
 * the mel once (no frames / spectrum round trip, no scratch).  wav_fmt: 0 = f32 in [-1,1], 1 = int16 PCM scaled by
 * 1/32768 on load (data.py:150 `audio / max_wav_value`).  Same output layout as ft_mel_spectrogram. */
int ft_mel_spectrogram_fused(const void* wav, int wav_fmt, const long long* sample_offsets, const long long* frame_offsets,
                             int n_utt, long long total_frames, const float* window, const float* mel_basis, const int* band_lo,
                             const int* band_hi, int n_mel, int n_fft, int hop, float clip, float* mel_out, void* stream);

/* STFT.transform (audio_processing.py:207-235), n_fft == 1024: magnitude and phase (atan2(imag, real)) as per-utterance
 * [n_fft/2+1, F_u] blocks (== [B, 513, F] for equal lengths), same kernel as above without the filterbank.  total_frames
 * is a host upper bound that sizes the grid; the kernel reads the true total from frame_offsets[n_utt] in device memory,
 * so offsets planned on the device (ft_stft_pack_rows) need no host round trip. */
int ft_stft_transform(const float* wav, const long long* sample_offsets, const long long* frame_offsets, int n_utt,
                      long long total_frames, const float* window, int n_fft, int hop, float* magnitude, float* phase,
                      void* stream);

/* Packs the rows of a padded batch audio [B, N] fp32 into the layout ft_stft_transform reads, from per-row sample counts
 * in device memory (lengths int64 [B]): row b's first min(lengths[b], N) samples go to packed[sample_offsets[b]], and
 * sample_offsets / frame_offsets (int64 [B + 1] each, written) are their prefix sums and those of 1 + n / hop frames.  A
 * row of at most n_fft / 2 samples (the reflect padding) is empty: no samples, no frames.  packed holds at most B * N
 * floats and the frames total at most B * (1 + N / hop).  One launch, no host synchronisation. */
int ft_stft_pack_rows(const float* audio, int B, long long N, const long long* lengths, int n_fft, int hop, float* packed,
                      long long* sample_offsets, long long* frame_offsets, void* stream);

/* STFT.inverse (audio_processing.py:237-265), n_fft == 1024, hop in {128, 256, 512}: magnitude / phase as per-utterance
 * [513, F_u] blocks at frame_offsets[u] (prefix sums, n_utt + 1 entries, the layout ft_stft_transform writes) ->
 * (F_u - 1) * hop samples per utterance written at out[out_offsets[u]] (n_utt entries read: prefix sums for a packed
 * output, row starts for a padded one).  Frames are irfft'd, windowed with `window` (the zero-padded analysis window,
 * 1024 floats), overlap-added, divided by the window's sum-square envelope where it exceeds FLT_MIN, and 512 samples
 * are dropped at each end.  bias (513 floats, optional): the magnitude becomes max(m - strength * bias[k], 0) on load
 * (tacotron2/waveglow/denoiser.py), so transform + inverse is the whole Denoiser.  One launch, deterministic (each
 * sample sums its frames in utterance-local order: ragged rows equal B = 1 runs), no host sync.  total_frames is a host
 * upper bound, the true total is frame_offsets[n_utt], as for ft_stft_transform. */
int ft_stft_inverse(const float* magnitude, const float* phase, const long long* frame_offsets, const long long* out_offsets,
                    int n_utt, long long total_frames, const float* window, int n_fft, int hop, const float* bias,
                    float strength, float* out, void* stream);

/* Data layer on the device (SURVEY.md 8f row 1).
 * ft_attn_prior: beta_binomial_prior_distribution (data.py:31-41) for a whole batch directly in DataCollate's zero-padded
 *   [B,T,L] layout (data.py:222-243): prior[b,i-1,k] = BetaBinomial(k; n=in_lens[b]-1, a=s*i, b=s*(out_lens[b]+1-i)) for
 *   i <= out_lens[b], k < in_lens[b], else 0; values < threshold are zeroed when threshold > 0 (data.py:137-139).
 *   fp64 log-gamma evaluation, fp32 output.
 * ft_collate_mel: DataCollate's mel / gate padding (data.py:214-236) from ft_mel_spectrogram's packed output: row i of
 *   mel_padded [B,n_mel,T] is utterance order[i]; gate_padded [B,T] = 1 from its last frame on; out_lens[i] = its frames. */
int ft_attn_prior(const int* in_lens, const int* out_lens, int B, int T, int L, float scaling, float threshold, float* prior,
                  void* stream);
int ft_collate_mel(const float* mel_packed, const long long* frame_offsets, const int* order, int B, int n_mel, int T,
                   float* mel_padded, float* gate_padded, int* out_lens, void* stream);

/* AttentionCTCLoss (flowtron.py:155-182) for a whole batch, with its gradient, in one launch (SURVEY.md 8f row 4; the
 * reference loops over utterances in Python).  attn_logprob [B,T,L] f32 of ONE flow; classes = blank (constant logit
 * blank_logprob) + the utterance's in_lens[b] tokens, log_softmax over them, CTC against the target 1..in_lens[b] over
 * out_lens[b] frames, reduction 'mean' (nll / in_lens[b]), zero_infinity.  time_reversed = 1: the tensor is in an
 * AR_Back_Step's flipped time (flowtron.py:250-256).  cost [B]; d_attn_logprob [B,T,L] = d cost[b] / d attn_logprob (zeros
 * outside the utterance's frames / tokens).  scratch: ft_attn_ctc_scratch_bytes(B, T, L). */
size_t ft_attn_ctc_scratch_bytes(int B, int T, int L);
int ft_attn_ctc_loss(const float* attn_logprob, const int* in_lens, const int* out_lens, int B, int T, int L, int time_reversed,
                     float blank_logprob, float* cost, float* d_attn_logprob, void* scratch, void* stream);


/* ------------------------------------------------------------------------------------------------------
 * Text Encoder (flowtron.py:467-525): 3 x [Conv1d(512, 512, k=5) -> MaskedInstanceNorm1d(affine) -> relu -> dropout(0.5)],
 * then a packed bidirectional LSTM(512 -> 2 x 256); forward + backward (SURVEY.md 8a row 13 / 8f row 2).
 * Replaces Encoder.forward (masked = 1: tokens at l >= in_lens[b] are zeroed before every convolution, statistics run over
 * the utterance's own tokens, the BiLSTM behaves as on a packed sequence, outputs are zero at l >= in_lens[b]) and
 * Encoder.infer / the B == 1 case (masked = 0: no lengths).  Weights in PyTorch layouts; index 1 of the LSTM arrays is the
 * `_reverse` direction.
 * ---------------------------------------------------------------------------------------------------- */
typedef struct {
    int B, L;           /* utterances (1..64), padded text length                               */
    int C;              /* 512 (encoder_embedding_dim; must be 512 in this build)               */
    int n_convs, ksize; /* 3, 5                                                                 */
    int masked;         /* 1: use in_lens (Encoder.forward, B > 1); 0: every token valid        */
    float dropout_p;    /* 0 (eval) or the training probability (flowtron.py:502 hard-codes 0.5) */
    float eps;          /* instance-norm eps (1e-5)                                             */
} FtEncoderDesc;

typedef struct {
    const float* conv_w[3]; const float* conv_b[3];    /* [512,512,5], [512] */
    const float* norm_w[3]; const float* norm_b[3];    /* [512]              */
    const float* w_ih[2]; const float* w_hh[2];        /* [1024,512], [1024,256] */
    const float* b_ih[2]; const float* b_hh[2];        /* [1024]             */
} FtEncoderWeights;

typedef struct {                                       /* gradients, same shapes, OVERWRITTEN */
    float* d_conv_w[3]; float* d_conv_b[3];
    float* d_norm_w[3]; float* d_norm_b[3];
    float* d_w_ih[2]; float* d_w_hh[2];
    float* d_b_ih[2]; float* d_b_hh[2];
} FtEncoderGrads;

size_t ft_encoder_saved_bytes(const FtEncoderDesc* d);          /* forward -> backward tensors */
size_t ft_encoder_fwd_scratch_bytes(const FtEncoderDesc* d);
size_t ft_encoder_bwd_scratch_bytes(const FtEncoderDesc* d);
/* x [B, 512, L] fp32 (embedding output, channels first, as Encoder.forward receives it); in_lens int32 [B] (masked only);
 * rng_state: device uint64[2] = {seed, call counter} for the dropout masks (advanced by the call; NULL when dropout_p == 0);
 * out: fp32, element (b, l, c) at out[b * out_stride_b + l * out_stride_l + c], c < 512 (forward direction first) -- lets the
 * caller write straight into the [L, B, 640] text tensor the flows read. */
int ft_encoder_fwd(const FtEncoderDesc* d, const FtEncoderWeights* w, const float* x, const int* in_lens,
                   unsigned long long* rng_state, float* out, long long out_stride_b, long long out_stride_l, void* saved,
                   void* scratch, void* stream);
/* Token form: the nn.Embedding lookup in front of the encoder (flowtron.py:873 `self.embedding(text).transpose(1, 2)`) fused into
 * the first kernel (tokens int64 [B, L], emb_weight fp32 [n_text, 512]); the backward scatters into d_emb_weight (overwritten). */
int ft_encoder_fwd_tokens(const FtEncoderDesc* d, const FtEncoderWeights* w, const long long* tokens, const float* emb_weight,
                          int n_text, const int* in_lens, unsigned long long* rng_state, float* out, long long out_stride_b,
                          long long out_stride_l, void* saved, void* scratch, void* stream);
int ft_encoder_bwd_tokens(const FtEncoderDesc* d, const FtEncoderWeights* w, const float* d_out, long long d_stride_b,
                          long long d_stride_l, const void* saved, const long long* tokens, int n_text, float* d_emb_weight,
                          const FtEncoderGrads* grads, void* scratch, void* stream);
/* d_out: dense [B, L, 512] fp32; d_x [B, 512, L] fp32 (may be NULL). */
int ft_encoder_bwd(const FtEncoderDesc* d, const FtEncoderWeights* w, const float* d_out, long long d_stride_b,
                   long long d_stride_l, const void* saved, float* d_x, const FtEncoderGrads* grads, void* scratch, void* stream);

/* ------------------------------------------------------------------------------------------------------
 * MelEncoder of the Gaussian-mixture prior (flowtron.py:416-439): 2 x [conv k=3 (80 -> 512, 512 -> 512) -> masked instance
 * norm (affine) -> relu -> dropout], packed BiLSTM 512 -> 2 x 256, mean over time.  Same conventions as the text encoder.
 * ---------------------------------------------------------------------------------------------------- */
#define FT_MEL_ENC_MAX_BATCH 64

typedef struct {
    int B, T;                 /* utterances in this call (1..64), padded frames (any T: limited by memory only) */
    float eps, dropout_p;     /* instance-norm eps; dropout probability (0: eval)                                 */
} FtMelEncoderDesc;

typedef struct {
    const float* conv_w[2]; const float* conv_b[2];    /* [512,80,3] / [512,512,3], [512] */
    const float* norm_w[2]; const float* norm_b[2];    /* [512]                           */
    const float* w_ih[2]; const float* w_hh[2];        /* [1024,512], [1024,256]          */
    const float* b_ih[2]; const float* b_hh[2];        /* [1024]                          */
} FtMelEncoderWeights;

typedef struct {                                       /* gradients, same shapes, OVERWRITTEN */
    float* d_conv_w[2]; float* d_conv_b[2];
    float* d_norm_w[2]; float* d_norm_b[2];
    float* d_w_ih[2]; float* d_w_hh[2];
    float* d_b_ih[2]; float* d_b_hh[2];
} FtMelEncoderGrads;

size_t ft_mel_encoder_saved_bytes(const FtMelEncoderDesc* d);
size_t ft_mel_encoder_fwd_scratch_bytes(const FtMelEncoderDesc* d);
size_t ft_mel_encoder_bwd_scratch_bytes(const FtMelEncoderDesc* d);
/* mel [B, 80, T] fp32 (read only; frames at t >= out_lens[b] are never read); out_lens int32 [B], every length in [1, T];
 * all_lens int32 [n_all]: the lengths of the whole batch this call is a slice of, whose maximum divides the time sum (the
 * reference's torch.mean over the padded LSTM output); rng_state as for ft_encoder_fwd; emb [B, 512] fp32. */
int ft_mel_encoder_fwd(const FtMelEncoderDesc* d, const FtMelEncoderWeights* w, const float* mel, const int* out_lens,
                       const int* all_lens, int n_all, unsigned long long* rng_state, float* emb, void* saved, void* scratch,
                       void* stream);
/* d_emb [B, 512] fp32; weight gradients only (no gradient w.r.t. the mel). */
int ft_mel_encoder_bwd(const FtMelEncoderDesc* d, const FtMelEncoderWeights* w, const float* d_emb, const void* saved,
                       const FtMelEncoderGrads* grads, void* scratch, void* stream);

/* ------------------------------------------------------------------------------------------------------
 * Gaussian-mixture NLL (FlowtronLoss gm_loss=True, flowtron.py:217-235):
 *   nll = -sum_{t < out_lens[b], b, m} logsumexp_k [log prob_bk - log_var_bmk / 2 - (z_tbm - mean_bmk)^2 / (2 exp log_var_bmk)]
 * z [T, B, M] fp32; mean / log_var [B, M, K] (per_row = 1) or [1, M, K] (per_row = 0); prob [B, K].  K <= 32, M <= 80.
 * Fixed summation order, no atomics: replays are bit-identical.
 * ---------------------------------------------------------------------------------------------------- */
#define FT_GMM_MAX_COMPONENTS 32

typedef struct { int T, B, M, K, per_row; } FtGmmDesc;

size_t ft_gmm_nll_scratch_bytes(const FtGmmDesc* d);
/* sums[0] = nll, sums[1] = number of valid frames */
int ft_gmm_nll_reduce(const FtGmmDesc* d, const float* z, const int* out_lens, const float* mean, const float* log_var,
                      const float* prob, float* sums, void* scratch, void* stream);
/* The same NLL per utterance (Flowtron.score): rows_out [B] fp32, row b = -sum_{t < out_lens[b], m} logsumexp_k a_k.  Same
 * scratch as ft_gmm_nll_reduce.  Each row is summed from its own partials in a fixed order: it does not depend on the other
 * rows' data or on B (the mixture parameters themselves come from the caller). */
int ft_gmm_nll_rows(const FtGmmDesc* d, const float* z, const int* out_lens, const float* mean, const float* log_var,
                    const float* prob, float* rows_out, void* scratch, void* stream);
/* gradients of g_nll[0] * nll: dz [T, B, M] (zero past the lengths), dprob [B, K], and dmean / dlog_var [B, M, K] (both NULL
 * when the Gaussians are shared buffers: per_row must then be 0 or they are ignored) -- all overwritten. */
int ft_gmm_nll_grad(const FtGmmDesc* d, const float* z, const int* out_lens, const float* mean, const float* log_var,
                    const float* prob, const float* g_nll, float* dz, float* dmean, float* dlog_var, float* dprob, void* scratch,
                    void* stream);

/* Sampling from the mixture (csrc/gmm_sample.cu).  d->T is z's padded frame count; mean / log_var / prob as above.
 * z [B, M, T] fp32, overwritten: for t < min(n_frames[b], T) element (c, t) takes component k -- component[b] when that lies
 * in [0, K), otherwise drawn from prob[b] (non-negative weights with a positive sum; they need not be normalised) -- and is
 * mean[b|0, c, k] + sigma exp(log_var[b|0, c, k] / 2) eps with eps ~ N(0, 1); every other element is 0.  component may be
 * NULL (draw every element).  rng_state: device uint64 {seed, counter}.  The draws of element (b, c, t) depend only on
 * (seed, counter, b, c, t); a one-thread launch behind the sampler adds 1 to the counter, so each call (and each replay of a
 * captured graph) draws new values.  Two launches, no allocation, no host synchronisation. */
int ft_gmm_sample(const FtGmmDesc* d, const float* mean, const float* log_var, const float* prob, const int* n_frames,
                  const int* component, float sigma, unsigned long long* rng_state, float* z, void* stream);
/* Component responsibilities: resp [B, K] fp32, resp[b, k] = mean over t < out_lens[b] (clamped to T) and all M channels of
 * prob_k N_k(z) / sum_j prob_j N_j(z), in log space with the NLL's max shift.  z [T, B, M] as ft_gmm_nll_reduce reads it;
 * scratch: ft_gmm_nll_scratch_bytes(d) bytes.  Each row is summed from its own partials in a fixed order with no atomics, so
 * it equals the row's B = 1 call bit for bit. */
int ft_gmm_responsibilities(const FtGmmDesc* d, const float* z, const int* out_lens, const float* mean, const float* log_var,
                            const float* prob, float* resp, void* scratch, void* stream);

/* ------------------------------------------------------------------------------------------------------
 * WaveGlow vocoder, inference direction (tacotron2/waveglow/glow.py:251-293 WaveGlow.infer): log-mel -> audio.
 * Built for n_mel 80, n_group 8, WN n_channels 256, kernel_size 3; n_flows <= 16, n_layers <= 8.
 * ---------------------------------------------------------------------------------------------------- */
#define FT_WG_MAX_FLOWS 16
#define FT_WG_MAX_LAYERS 8

typedef struct {
    int n_mel, n_flows, n_group, n_early_every, n_early_size;   /* 80, 12, 8, 4, 2 (waveglow config.json)        */
    int n_layers, n_channels, kernel_size;                      /* WN_config: 8, 256, 3                           */
    int B;                                                      /* utterances (1..128)                            */
    int F_max;                                                  /* padded mel frames of `mel`                     */
    const int* frames;                                          /* host int[B]: frames of utterance b (1..F_max), */
                                                                /* or NULL for ft_waveglow_infer_dev              */
} FtWaveGlowDesc;

/* Device pointers to the packed weights of WaveGlow (flowtron_b200/waveglow.py packs them once per weight version):
 *   up_w   fp16 [20480, 384]: the ConvTranspose1d(80, 80, 1024, stride 256) as one GEMM over frames f-3..f (4 x 96 K, mel
 *          channels zero-padded to 96); column n = g*640 + c*8 + j is sample 8g + j of channel c within the frame; up_b [20480]
 *   in_w   fp16 [512, 1408] per (flow, layer): [tap0 | tap1 | tap2 | cond_layer slice] of the weight-norm-folded in_layer and
 *          cond_layer, rows interleaved (2c = tanh channel c, 2c+1 = sigmoid channel c); in_b [512] = in_layer + cond bias
 *   rs_w   fp16 [512 (256 for the last layer), 256]: res_skip_layer; rs_b fp32
 *   start_w fp32 [256, n_half], start_b [256]; end_w fp32 [2 n_half, 256], end_b [2 n_half]; inv_w fp32 [c, c] = convinv^-1 */
typedef struct {
    const void* up_w; const float* up_b;
    const void* in_w[FT_WG_MAX_FLOWS][FT_WG_MAX_LAYERS]; const float* in_b[FT_WG_MAX_FLOWS][FT_WG_MAX_LAYERS];
    const void* rs_w[FT_WG_MAX_FLOWS][FT_WG_MAX_LAYERS]; const float* rs_b[FT_WG_MAX_FLOWS][FT_WG_MAX_LAYERS];
    const float* start_w[FT_WG_MAX_FLOWS]; const float* start_b[FT_WG_MAX_FLOWS];
    const float* end_w[FT_WG_MAX_FLOWS]; const float* end_b[FT_WG_MAX_FLOWS];
    const float* inv_w[FT_WG_MAX_FLOWS];
} FtWaveGlowWeights;

/* Bytes of the caller-owned scratch of ft_waveglow_infer (0 if the descriptor is rejected).  With d->frames == NULL: the
 * scratch of ft_waveglow_infer_dev, sized for every utterance at F_max. */
size_t ft_waveglow_scratch_bytes(const FtWaveGlowDesc* d);
/* mel fp32 [B, 80, F_max]; noise fp32 [B, 8, 32 F_max]: channels of WaveGlow.forward's z -- the first flow's draw on the
 * highest channels (4:8 for the shipped config), each early injection on the channels just below (2:4 after flow 8, 0:2
 * after flow 4); it is multiplied by sigma.  audio fp32 [B, 256 F_max]: utterance b fills its first 256 frames[b] samples,
 * the rest is zero.  A planner kernel lays the batch out in scratch from the frame counts (passed to it by value), and the
 * other kernels read that layout from device memory.  n_flows * (2 n_layers + 1) + 4 launches, no host synchronisation
 * (CUDA-graph capturable). */
int ft_waveglow_infer(const FtWaveGlowDesc* d, const FtWaveGlowWeights* w, const float* mel, const float* noise, float sigma,
                      float* audio, void* scratch, void* stream);
/* ft_waveglow_infer with the frame counts in device memory: frames_dev int32 [B], read only by the planner kernel, so a
 * CUDA graph captured once replays with whatever counts the buffer holds.  d->frames must be NULL and the scratch is
 * ft_waveglow_scratch_bytes(d) for that descriptor.  Grids and GEMM rows are sized for every utterance at F_max; tiles and
 * rows past the planned layout exit at once.  Each count is clamped to 1..F_max, so no value makes a kernel address past
 * mel, noise, audio or the scratch; counts outside 1..F_max give an unspecified row.  Rows equal ft_waveglow_infer's with
 * the same counts bit for bit.  Same launches, no host synchronisation. */
int ft_waveglow_infer_dev(const FtWaveGlowDesc* d, const FtWaveGlowWeights* w, const float* mel, const float* noise, float sigma,
                          const int* frames_dev, float* audio, void* scratch, void* stream);

/* ------------------------------------------------------------------------------------------------------
 * WaveGlow training (glow.py:196-245 WaveGlow.forward, the z direction) and its backward, same configurations as infer.
 * ---------------------------------------------------------------------------------------------------- */
typedef struct {
    int n_mel, n_flows, n_group, n_early_every, n_early_size;   /* as FtWaveGlowDesc                               */
    int n_layers, n_channels, kernel_size;
    int B;                                                      /* utterances (1..128), all of N samples           */
    int F;                                                      /* mel frames of `mel`                             */
    int N;                                                      /* audio samples: a multiple of 8, N <= 256 F      */
} FtWaveGlowTrainDesc;

/* Packed weights as in FtWaveGlowWeights (up_w, in_w, rs_w fp16; the rest fp32), plus the backward's transposed copies and
 * the forward 1x1 convolutions:
 *   in_wT  fp16 [256, 1536]: in_wT[c, 512 t + j] = in_w[j, 256 t + c], t = 0..2 (the dilated taps, transposed)
 *   rs_wT  fp16 [256, 512 (256 for the last layer)] = rs_w^T
 *   conv_w fp32 [c, c]: convinv weight of flow k */
typedef struct {
    const void* up_w; const float* up_b;
    const void* in_w[FT_WG_MAX_FLOWS][FT_WG_MAX_LAYERS]; const float* in_b[FT_WG_MAX_FLOWS][FT_WG_MAX_LAYERS];
    const void* rs_w[FT_WG_MAX_FLOWS][FT_WG_MAX_LAYERS]; const float* rs_b[FT_WG_MAX_FLOWS][FT_WG_MAX_LAYERS];
    const void* in_wT[FT_WG_MAX_FLOWS][FT_WG_MAX_LAYERS]; const void* rs_wT[FT_WG_MAX_FLOWS][FT_WG_MAX_LAYERS];
    const float* start_w[FT_WG_MAX_FLOWS]; const float* start_b[FT_WG_MAX_FLOWS];
    const float* end_w[FT_WG_MAX_FLOWS]; const float* end_b[FT_WG_MAX_FLOWS];
    const float* conv_w[FT_WG_MAX_FLOWS];
} FtWaveGlowTrainWeights;

/* fp32 gradients of the packed (effective, weight-norm-folded) weights, all overwritten: up_w [20480, 384], up_b [20480];
 * in_w[k][i][t] [512, 256] for tap t = 0..2 and in_w[k][i][3] [512, 640] (the cond_layer slice), in_b [512]; rs_w / rs_b;
 * start_w [256, n_half], start_b [256], end_w [2 n_half, 256], end_b, conv_w [c, c] (without the log-determinant term). */
typedef struct {
    float* up_w; float* up_b;
    float* in_w[FT_WG_MAX_FLOWS][FT_WG_MAX_LAYERS][4]; float* in_b[FT_WG_MAX_FLOWS][FT_WG_MAX_LAYERS];
    float* rs_w[FT_WG_MAX_FLOWS][FT_WG_MAX_LAYERS]; float* rs_b[FT_WG_MAX_FLOWS][FT_WG_MAX_LAYERS];
    float* start_w[FT_WG_MAX_FLOWS]; float* start_b[FT_WG_MAX_FLOWS];
    float* end_w[FT_WG_MAX_FLOWS]; float* end_b[FT_WG_MAX_FLOWS];
    float* conv_w[FT_WG_MAX_FLOWS];
} FtWaveGlowTrainGrads;

/* Caller-owned areas (0 if the descriptor is rejected): `saved` lives from ft_waveglow_train_fwd to ft_waveglow_train_bwd,
 * `scratch` only during one call. */
size_t ft_waveglow_train_saved_bytes(const FtWaveGlowTrainDesc* d);
size_t ft_waveglow_train_scratch_bytes(const FtWaveGlowTrainDesc* d);
/* mel fp32 [B, 80, F], audio fp32 [B, N] -> z fp32 [B, 8, N/8] (the reference's channel order: early outputs first) and
 * log_s[k] fp32 [B, n_half_k, N/8] (HOST array of n_flows device pointers).  No allocation, no host synchronisation. */
int ft_waveglow_train_fwd(const FtWaveGlowTrainDesc* d, const FtWaveGlowTrainWeights* w, const float* mel, const float* audio,
                          float* z, float* const* log_s, void* saved, void* scratch, void* stream);
/* Upstream gradients d_z [B, 8, N/8] and d_log_s[k] [B, n_half_k, N/8] (d_z, d_log_s or any entry may be NULL = zero)
 * -> the packed-weight gradients.  No allocation, no host synchronisation. */
int ft_waveglow_train_bwd(const FtWaveGlowTrainDesc* d, const FtWaveGlowTrainWeights* w, const float* d_z,
                          const float* const* d_log_s, const void* saved, const FtWaveGlowTrainGrads* g, void* scratch,
                          void* stream);

/* ------------------------------------------------------------------------------------------------------
 * Style transfer by posterior sampling (the reference's inference_style_transfer.ipynb): the posterior mean of the z of
 * B reference utterances (csrc/style.cu).
 * ---------------------------------------------------------------------------------------------------- */
/* z fp32 [T, B, M] (Flowtron.forward's flow layout, row t*B + b), M <= 128; out_lens int32 [B] on the device, each in
 * [1, T] (not checked);  mode 0 ('batch'): out fp32 [M, n_frames],
 *   out[m, t] = scale * (1/B) sum_b z[t mod out_lens[b], b, m]                      (each z repeated in time to n_frames);
 * mode 1 ('time_and_batch'): out fp32 [M],
 *   out[m] = scale * (1/B) sum_b (1/out_lens[b]) sum_{t < out_lens[b]} z[t, b, m].
 * scale = ratio / (ratio + 1) with ratio = B / lambda.  One launch, fp32 sums in a fixed order (no atomics: replays are
 * bit-identical), no allocation, no host synchronisation.  Rejects B < 1, T < 1, n_frames < 1 and M > 128. */
int ft_posterior_mean(const float* z, int T, int B, int M, const int* out_lens, int n_frames, int mode, float scale,
                      float* out, void* stream);

/* ------------------------------------------------------------------------------------------------------
 * Hard alignments (csrc/align.cu): monotonic alignment search over one flow's attention log-probabilities, and the
 * one-hot maps of per-token durations.
 * ---------------------------------------------------------------------------------------------------- */
/* logp fp32 [B, T, L] (a flow's attn_logprob), in_lens / out_lens int32 [B] on the device, L <= FT_MAX_TEXT_LEN, any T.
 * Row b (Tb = out_lens[b], Lb = in_lens[b]), s[t][l] = logp[b, t', l] with t' = t, or Tb-1-t when time_reversed (an
 * AR_Back_Step's flipped time):  Q[0][0] = s[0][0], Q[0][l > 0] = -inf, Q[t][l] = s[t][l] + max(Q[t-1][l], Q[t-1][l-1])
 * (Q[t-1][-1] = -inf), fp32 adds without contraction.  The path ends at (Tb-1, Lb-1) and, walked back, moves to l-1 only
 * where Q[t-1][l-1] > Q[t-1][l] (ties stay on the token).  token_of_frame int32 [B, T] (natural time): the path's token at
 * frame t < Tb, -1 from Tb on; durations int32 [B, L]: frames per token (each >= 1, summing to Tb), 0 from Lb on.  A row
 * with Tb < Lb (or Lb = 0) has no path: all-zero durations, -1 everywhere.  Only t < Tb, l < Lb are read.  scratch:
 * ft_mas_align_scratch_bytes(B, T, L) (the backpointer bits, T * ceil(L/32) words per row).  One launch, no allocation, no
 * host synchronisation (CUDA-graph capturable). */
size_t ft_mas_align_scratch_bytes(int B, int T, int L);
int ft_mas_align(const float* logp, const int* in_lens, const int* out_lens, int B, int T, int L, int time_reversed,
                 int* durations, int* token_of_frame, void* scratch, void* stream);
/* durations int32 [B, L] (tokens at l >= in_lens[b] and negative values count as 0), in_lens int32 [B] on the device ->
 * out fp32 [B, Ta, L], one-hot: with n_b = sum_l durations[b, l], row (b, i) for i < n_b is generation step i -- natural
 * frame i, or n_b-1-i when time_reversed -- and holds a 1 at the token that frame belongs to; every other entry is 0.
 * The prefix sums are computed on the device.  One launch, no allocation, no host synchronisation. */
int ft_durations_to_attn(const int* durations, const int* in_lens, int B, int L, int Ta, int time_reversed, float* out,
                         void* stream);

/* ------------------------------------------------------------------------------------------------------
 * Attention (flowtron.py:528-592) as a module of its own (csrc/attention_module.cu): the Q / K / V projections, the fused
 * score / softmax / prior / context kernels the flow step runs, and the forced-weights branch, forward and backward.
 * ---------------------------------------------------------------------------------------------------- */
typedef struct {
    int T, B, L;        /* queries (frames), batch, keys (text tokens, <= FT_MAX_TEXT_LEN)                        */
    int Dq, E, A;       /* query channels, key / value channels, attention channels: each a multiple of 8        */
    int has_prior;      /* attn_prior given (ignored when attn_given)                                              */
    int attn_given;     /* 1: `attn` is the caller's forced weights [B, T, L]; only the value projection runs       */
    float temperature;  /* Attention.temperature (> 0)                                                             */
} FtAttentionDesc;

typedef struct {                                     /* fp32, PyTorch layouts                                       */
    const float *query, *key, *value, *v;            /* [A, Dq], [A, E], [A, E], [A] (v.linear_layer.weight [1, A])  */
} FtAttentionWeights;
typedef struct {                                     /* gradients, same shapes, OVERWRITTEN; each may be NULL        */
    float *query, *key, *value, *v;
} FtAttentionGrads;

/* `saved` persists from ft_attention_fwd to ft_attention_bwd; `scratch` is transient.  0 for a descriptor the kernels do
 * not take (ft_last_error says why). */
size_t ft_attention_saved_bytes(const FtAttentionDesc* d);
size_t ft_attention_scratch_bytes(const FtAttentionDesc* d);
/* queries fp32 [T, B, Dq], keys / values fp32 [L, B, E] (may be different tensors), in_lens int32 [B] valid keys per row on the
 * device (NULL: all L; trusted: a row needs at least one), attn_prior fp32 [B, T, L] or NULL.
 * Writes output fp32 [B, A, T] = bmm(attn, value(values)).transpose(1, 2), attn fp32 [B, T, L] (masked keys exactly 0) and
 * attn_logprob fp32 [B, T, L] (log(attn + 1e-8), or the pre-mask posterior with a prior).  With attn_given, `attn` is read,
 * queries / keys / in_lens / attn_prior / attn_logprob are not used, and one batched tensor-core kernel forms the context.
 * No allocation, no host synchronisation (CUDA-graph capturable). */
int ft_attention_fwd(const FtAttentionDesc* d, const FtAttentionWeights* w, const float* queries, const float* keys,
                     const float* values, const int* in_lens, const float* attn_prior, float* output, float* attn,
                     float* attn_logprob, void* saved, void* scratch, void* stream);
/* Gradients of the forward above given the upstream gradients d_output [B, A, T], d_attn and d_attn_logprob [B, T, L], each
 * NULL when absent (d_attn_logprob must be NULL with attn_given).  `attn` is the forward's attn.  Every output pointer may be
 * NULL and skips its work: d_queries [T, B, Dq], d_keys / d_values [L, B, E], g (weight gradients) and, with attn_given only,
 * d_attn_given [B, T, L] = d_attn + the context's gradient w.r.t. the forced weights. */
int ft_attention_bwd(const FtAttentionDesc* d, const FtAttentionWeights* w, const float* queries, const float* keys,
                     const float* values, const int* in_lens, const float* attn, const float* d_output, const float* d_attn,
                     const float* d_attn_logprob, float* d_queries, float* d_keys, float* d_values, float* d_attn_given,
                     const FtAttentionGrads* g, void* saved, void* scratch, void* stream);

#ifdef __cplusplus
}
#endif
#endif
