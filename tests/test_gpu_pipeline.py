"""GPU: the chunked schedules of a flow step (csrc/ar_step.cu, DESIGN.md 4.2).  lstm layers 0/1 run as two 64-CTA
recurrences one 100-step chunk apart at every T (forward and BPTT); from T = 320 on the attention LSTM runs in 256-step
chunks with the attention of each finished chunk underneath the next one.  Gradients at these shapes are checked against
the CPU oracle in test_gpu_flowtron_train.py::test_chunked_schedules_match_oracle."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _step_and_inputs(T, B=5, L=12):
    """A gated AR_Step (the last flow of a one-flow model) with a prior, and inputs for T frames."""
    from flowtron_b200 import synth
    from flowtron_b200.flowtron import Flowtron
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=1)
    model = Flowtron(**cfg)
    model.load_state_dict(synth.synth_params(cfg, 5), strict=True)
    step = model.flows[0].cuda()
    assert hasattr(step, "gate_layer")
    batch = synth.synth_batch(B, T, L, cfg, 9, out_lens=[T] * B, in_lens=[L, L, 9, 6, 3], with_prior=True)
    E = cfg["n_text_dim"] + cfg["n_speaker_dim"]
    mel = batch["mel"].permute(2, 0, 1).contiguous().cuda()
    text = (0.5 * torch.randn(L, B, E, generator=torch.Generator().manual_seed(11))).cuda()
    mask = ~(torch.arange(L)[None, :] < batch["in_lens"][:, None])[..., None]
    return step, mel, text, mask.cuda(), batch["attn_prior"].cuda()


def _forward(step, mel, text, mask, prior, T):
    """The step on the first T frames, every utterance T frames long: (z, log_s, gate, attention)."""
    from flowtron_b200 import _lib
    out_lens = torch.full((mel.shape[1],), T, dtype=torch.long, device="cuda")
    with torch.no_grad():
        z, log_s, gate, attn, _ = step(mel[:T].contiguous(), text, mask, out_lens, prior[:, :T].contiguous())
    torch.cuda.synchronize()
    assert _lib.device_status() == 0
    return z, log_s, gate, attn


def test_layer_chunk_boundaries_leave_the_forward_unchanged():
    """At T = 250 lstm layers 0/1 run as three chunks with a ragged 50-step tail; the first 78 frames alone are one chunk.
    Every forward kernel is per step or per row, so the 78 frames come out bit-identical.  The cut is even because the
    attention kernel scores query rows in pairs that share one reciprocal (csrc/attention.cu, score_chunk): after an odd
    cut the last row would be paired with a padding row and differ in the last bit."""
    step, mel, text, mask, prior = _step_and_inputs(250)
    a = _forward(step, mel, text, mask, prior, 250)
    b = _forward(step, mel, text, mask, prior, 78)
    for x, y in zip(a[:3], b[:3]):
        assert torch.equal(x[:78], y)
    assert torch.equal(a[3][:, :78], b[3])


def test_attention_overlap_equals_folded_attention_lstm():
    """T = 347 runs the attention overlap (chunks of 256 + 91 steps); T = 256 runs the attention LSTM as one recurrence with
    the 80-channel input projection folded into its MMA chain.  Not bit-equal: the overlap adds the projection as a GEMM
    result in the epilogue, so the two differ by fp16 operand rounding of the recurrent state.  Both are within the 1e-3
    bar of the fp32 reference; the first 256 frames must agree to that bar."""
    def rel(x, y):
        return (x - y).abs().max().item() / max(y.abs().max().item(), 1e-12)
    step, mel, text, mask, prior = _step_and_inputs(347)
    a = _forward(step, mel, text, mask, prior, 347)
    b = _forward(step, mel, text, mask, prior, 256)
    for x, y in zip(a[:3], b[:3]):
        assert rel(x[:256], y) < 1e-3


def test_one_call_backward_equals_main_then_attention_lstm():
    """ft_ar_step_bwd is ft_ar_step_bwd_main followed by ft_ar_step_bwd_attn_lstm: one flow with a prior and a gate, run
    forward once per backward form, must give the same d_mel, d_text and parameter gradients up to the order of fp32
    atomics (split-K weight gradients, attention reductions)."""
    from flowtron_b200 import _lib, synth
    from flowtron_b200.flowtron import Flowtron
    B, T, L = 6, 300, 40
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=1)
    model = Flowtron(**cfg)
    model.load_state_dict(synth.synth_params(cfg, 5), strict=True)
    step = model.flows[0].cuda()
    assert hasattr(step, "gate_layer")
    batch = synth.synth_batch(B, T, L, cfg, 9, with_prior=True)
    g = torch.Generator().manual_seed(11)
    M, E = cfg["n_mel_channels"], cfg["n_text_dim"] + cfg["n_speaker_dim"]
    mel = batch["mel"].permute(2, 0, 1).contiguous().cuda()
    text = (0.5 * torch.randn(L, B, E, generator=g)).cuda()
    in_lens, out_lens = batch["in_lens"].to(torch.int32).cuda(), batch["out_lens"].to(torch.int32).cuda()
    prior = batch["attn_prior"].cuda()
    d_mel_out, d_log_s = torch.randn(T, B, M, generator=g).cuda(), torch.randn(T, B, M, generator=g).cuda()
    d_gates = torch.randn(T, B, 1, generator=g).cuda()
    d_attn, d_lp = (1e-2 * torch.randn(B, T, L, generator=g)).cuda(), (1e-2 * torch.randn(B, T, L, generator=g)).cuda()
    plist = [p.detach() for p in step._param_list()]
    desc = _lib.FtArStepDesc(T, B, L, M, 1024, cfg["n_attn_channels"], E, 0, 1, 1, 1.0)
    saved_bytes, scratch_bytes = _lib.ar_step_sizes(desc)

    def run(one_call):
        saved = torch.empty(saved_bytes, dtype=torch.uint8, device="cuda")
        scratch = torch.empty(scratch_bytes, dtype=torch.uint8, device="cuda")
        outs = [torch.empty(T, B, M, device="cuda"), torch.empty(T, B, M, device="cuda"), torch.empty(T, B, 1, device="cuda"),
                torch.empty(B, T, L, device="cuda"), torch.empty(B, T, L, device="cuda")]
        _lib.ar_step_fwd(desc, _lib.make_weights(plist), mel, text, in_lens, out_lens, prior, *outs, saved, scratch)
        d_mel, d_text = torch.full_like(mel, float("nan")), torch.full_like(text, float("nan"))
        grads = [torch.full_like(p, float("nan")) for p in plist]
        w, gw = _lib.make_weights(plist), _lib.make_weights(grads)
        if one_call:
            _lib.ar_step_bwd(desc, w, mel, in_lens, out_lens, outs[3], d_mel_out, d_log_s, d_gates, d_attn, d_lp, d_mel, d_text,
                             gw, saved, scratch)
        else:
            carry = torch.empty(_lib.ar_step_bwd_carry_bytes(desc), dtype=torch.uint8, device="cuda")
            _lib.ar_step_bwd_main(desc, w, mel, in_lens, out_lens, outs[3], d_mel_out, d_log_s, d_gates, d_attn, d_lp, d_text,
                                  gw, saved, scratch, carry)
            _lib.ar_step_bwd_attn_lstm(desc, w, out_lens, d_mel, gw, saved, scratch, carry)
        torch.cuda.synchronize()
        assert _lib.device_status() == 0
        return [o.cpu() for o in outs], [d_mel.cpu(), d_text.cpu()] + [x.cpu() for x in grads]

    fa, a = run(False)
    fb, b = run(True)
    for x, y in zip(fa, fb):
        assert torch.equal(x, y)                               # the forward is deterministic
    gmax = max(x.norm().item() for x in a)
    for i, (x, y) in enumerate(zip(a, b)):
        assert torch.isfinite(x).all(), i
        d = (x - y).norm().item()
        assert d <= 1e-3 * (x.norm().item() + 1e-4 * gmax), (i, d)
