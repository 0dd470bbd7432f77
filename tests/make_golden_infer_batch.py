#!/usr/bin/env python
"""Generate tests/golden/infer_ragged_{f2,f3,t400}.npz by running the UNMODIFIED reference on CPU fp32: one B = 1
Flowtron.infer (flowtron.py:901-930) per row, on that row's unpadded text and residual.  Writes these new files only; the
other fixtures are left as they are.

Run where the reference tree exists (FLOWTRON_REFERENCE, default /root/reference):
    python tests/make_golden_infer_batch.py
Weights come from flowtron_b200.synth.synth_params(cfg, seed) with the gate layer's weight scaled by `gate_scale` and its
bias set to `gate_bias`: the synthetic gate weight is small, so the gate logit barely moves from frame to frame; scaled up,
each stop decision is far from the threshold (the chosen lengths do not change when the bias moves by +-0.1), which an fp16
kernel must reproduce exactly.  Text padding holds random tokens and the residual past each budget random values: they
must not matter.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from flowtron_b200 import synth  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")

# tag -> n_flows, n_speakers, seed, T, L, in_lens, max_frames, gate_scale, gate_bias, (min gate stops, min budget runs)
CASES = {
    # 2 flows: the gated AR_Back_Step runs first
    "f2": (2, 1, 61, 48, 20, [20, 7, 13, 20, 9, 16], [44, 30, 40, 36, 46, 32], 40.0, -0.3, (2, 2)),
    # 3 flows: a gated forward AR_Step runs first; three speakers
    "f3": (3, 3, 62, 48, 20, [11, 20, 6, 17, 20, 14], [47, 33, 41, 28, 45, 38], 40.0, -6.0, (2, 2)),
    # BASELINE-like shapes, the gate never fires: fixed work
    "t400": (2, 1, 63, 400, 100, [100, 61, 83, 40], [400, 250, 330, 170], 1.0, -10.0, (0, 4)),
}


def case_inputs(n_flows, n_speakers, seed, T, L, in_lens, gate_scale, gate_bias):
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=n_flows, n_speakers=n_speakers)
    params = synth.synth_params(cfg, seed)
    kb = [k for k in params if k.endswith("gate_layer.linear_layer.bias")][0]
    kw = [k for k in params if k.endswith("gate_layer.linear_layer.weight")][0]
    params[kb] = torch.full_like(params[kb], gate_bias)
    params[kw] = params[kw] * gate_scale
    g = torch.Generator().manual_seed(seed)
    B = len(in_lens)
    residual = torch.randn(B, 80, T, generator=g) * 0.5
    text = torch.randint(0, cfg["n_text"], (B, L), generator=g)
    spk = torch.randint(0, n_speakers, (B,), generator=g)
    return cfg, params, residual, text, spk


def infer_batch_case(tag):
    from oracle import ref_shims
    n_flows, n_speakers, seed, T, L, in_lens, max_frames, gate_scale, gate_bias, (n_gate, n_budget) = CASES[tag]
    cfg, params, residual, text, spk = case_inputs(n_flows, n_speakers, seed, T, L, in_lens, gate_scale, gate_bias)
    _, model = ref_shims.reference_model(cfg, params)
    B = len(in_lens)
    mel = torch.zeros(B, 80, T)
    lens = np.zeros(B, dtype=np.int64)
    with torch.no_grad():
        for b in range(B):
            out, _ = model.infer(residual[b:b + 1, :, :max_frames[b]], spk[b:b + 1], text[b:b + 1, :in_lens[b]],
                                 temperature=1.0, gate_threshold=0.5)
            lens[b] = out.shape[-1]
            mel[b, :, :lens[b]] = out[0]
    stopped = int(sum(int(n) < m for n, m in zip(lens, max_frames)))
    print(f"infer_ragged_{tag}: in_lens {in_lens} max_frames {max_frames} -> mel_lens {lens.tolist()} "
          f"({stopped} gate stops, {B - stopped} at budget)")
    assert stopped >= n_gate and B - stopped >= n_budget, "the case no longer covers gate stops and budget runs"
    rec = dict(cfg_n_flows=n_flows, n_speakers=n_speakers, seed=seed, T=T, L=L, gate_scale=np.float32(gate_scale),
               gate_bias=np.float32(gate_bias), residual=residual.numpy(), text=text.numpy(), speaker_ids=spk.numpy(),
               in_lens=np.array(in_lens, dtype=np.int64), max_frames=np.array(max_frames, dtype=np.int64),
               mel=mel.numpy(), mel_lens=lens)
    np.savez_compressed(os.path.join(OUT, f"infer_ragged_{tag}.npz"), **rec)


def main():
    from oracle import ref_shims
    assert ref_shims.available(), "the reference tree is needed to generate fixtures"
    torch.set_num_threads(os.cpu_count() or 1)
    for tag in (sys.argv[1:] or CASES):
        infer_batch_case(tag)


if __name__ == "__main__":
    main()
