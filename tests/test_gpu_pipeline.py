"""GPU: the chunk-pipelined forward and BPTT of lstm layers 0/1 (FT_PIPE_FWD=1 / FT_PIPE_BWD=1, DESIGN.md 4.2: two 64-CTA
recurrences one chunk apart) must reproduce the one-launch-per-layer schedule bit for bit -- same kernel, same arithmetic,
different step ranges per launch.  The switch is read once per process by the library, so each run is a child process."""
import os
import subprocess
import sys

import pytest
import torch

from conftest import ROOT

pytestmark = pytest.mark.gpu

CHILD = r'''
import sys, torch
sys.path.insert(0, sys.argv[1])
from flowtron_b200 import synth
from flowtron_b200.flowtron import Flowtron
cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=2)
model = Flowtron(**cfg); model.load_state_dict(synth.synth_params(cfg, 5), strict=True); model = model.cuda()
b = synth.synth_batch(5, 77, 12, cfg, 9, with_prior=True)
d = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in b.items()}
from flowtron_b200.flowtron import FlowtronLoss
model.train(); model.encoder.p_dropout = 0.0
torch.backends.cudnn.allow_tf32 = False
out = model(d["mel"], d["speaker_ids"], d["text"], d["in_lens"], d["out_lens"], d["attn_prior"])
nll, gl, _ = FlowtronLoss()(out, d["gate_target"], d["in_lens"], d["out_lens"])
(nll + gl).sum().backward()
torch.cuda.synchronize()
torch.save({"z": out[0].detach().cpu(), "log_s": [x.detach().cpu() for x in out[1]], "gate": out[2].detach().cpu(),
            "grads": {n: p.grad.cpu() for n, p in model.named_parameters()}}, sys.argv[2])
'''


def _run(tmp_path, name, env):
    out = tmp_path / f"{name}.pt"
    e = dict(os.environ, **env)
    r = subprocess.run([sys.executable, "-c", CHILD, ROOT, str(out)], env=e, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    return torch.load(out)


def test_pipelined_layers_equal_default_schedule(tmp_path):
    a = _run(tmp_path, "default", {"FT_PIPE_FWD": "0", "FT_PIPE_BWD": "0"})
    b = _run(tmp_path, "pipe", {"FT_PIPE_FWD": "1", "FT_PIPE_BWD": "1", "FT_PIPE_CHUNK": "16"})   # 77 steps -> 5 chunks, ragged tail
    assert torch.equal(a["z"], b["z"]) and torch.equal(a["gate"], b["gate"])
    for x, y in zip(a["log_s"], b["log_s"]):
        assert torch.equal(x, y)
    gmax = max(v.norm().item() for v in a["grads"].values())
    for k in a["grads"]:
        d = (a["grads"][k] - b["grads"][k]).norm().item()
        assert d <= 1e-3 * (a["grads"][k].norm().item() + 1e-4 * gmax), (k, d)     # fp32 atomics / split-K order only


CHILD_LONG = CHILD.replace("synth.synth_batch(5, 77, 12, cfg, 9, with_prior=True)", "synth.synth_batch(6, 300, 40, cfg, 9, with_prior=True)")


def test_attention_overlap_equals_serial_schedule(tmp_path):
    """FT_ATT_OVERLAP (attention LSTM in 64-step chunks with the query projection / attention / gate / layer-0 projection of
    each finished chunk on a second stream) against the serial schedule.  Not bit-equal: the serial schedule folds the 80-channel
    input projection into the recurrence's MMA chain, the chunked one adds a GEMM result in the epilogue."""
    def run(name, env):
        out = tmp_path / f"{name}.pt"
        e = dict(os.environ, **env)
        r = subprocess.run([sys.executable, "-c", CHILD_LONG, ROOT, str(out)], env=e, capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stderr[-2000:]
        return torch.load(out)
    a = run("serial", {"FT_ATT_OVERLAP": "0"})
    b = run("overlap", {"FT_ATT_OVERLAP": "64"})              # 300 steps -> 5 chunks, ragged tail (44 steps)
    # third schedule: the same overlap under 64-step layer-pipeline chunks
    c = run("overlap_pipe64", {"FT_ATT_OVERLAP": "64", "FT_PIPE_CHUNK": "64"})

    def rel(x, y):
        return (x - y).abs().max().item() / max(y.abs().max().item(), 1e-12)
    gm = max(v.norm().item() for v in a["grads"].values())
    for k in a["grads"]:
        dd = (a["grads"][k] - c["grads"][k]).norm().item()
        assert dd <= 1e-2 * (a["grads"][k].norm().item() + 1e-4 * gm), ("overlap_pipe64", k, dd)
    # both schedules are within the 1e-3 bar of the fp32 reference; between themselves they differ by fp16 operand rounding of
    # the recurrent state (measured 4.8e-4 on z)
    assert rel(b["z"], a["z"]) < 1e-3 and rel(b["gate"], a["gate"]) < 1e-3
    for x, y in zip(b["log_s"], a["log_s"]):
        assert rel(x, y) < 1e-3
    gmax = max(v.norm().item() for v in a["grads"].values())
    for k in a["grads"]:
        d = (a["grads"][k] - b["grads"][k]).norm().item()
        assert d <= 1e-2 * (a["grads"][k].norm().item() + 1e-4 * gmax), (k, d)


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
