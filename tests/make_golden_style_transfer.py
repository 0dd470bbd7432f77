#!/usr/bin/env python
"""Generate tests/golden/style_{encode,posterior}.npz by running the UNMODIFIED reference on CPU fp32, the way its style-transfer
notebook (inference_style_transfer.ipynb) uses it.  Writes these new files only; the other fixtures are left as they are.

Run where the reference tree exists (FLOWTRON_REFERENCE, default /root/reference):
    python tests/make_golden_style_transfer.py

* style_encode.npz: K = 5 reference utterances with ragged text and frame lengths, each forwarded at B = 1 on its unpadded
  inputs (Flowtron.forward, flowtron.py:867-899); z[k, :, :out_lens[k]] holds that call's z.permute(1, 2, 0), the rest
  is zero.  The padded mel and text hold random values past each length: they must not matter.
* style_posterior.npz: both aggregations at n_frames 30, 120 and 300 (below, at and above the lengths) and at two lambd,
  restated in float64 from the stored z; then the reference Flowtron.infer (flowtron.py:901-930) of a new text from the
  residual mu + sigma * noise ('batch', 120 frames), with the noise stored.  The gate bias is -10, so the gate never fires
  and the output keeps all 120 frames.
Weights come from flowtron_b200.synth.synth_params(cfg, SEED): 2 flows, the last with the gate.
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

SEED = 71
GATE_BIAS = -10.0
IN_LENS = [23, 11, 30, 17, 26]
OUT_LENS = [97, 40, 120, 63, 81]
N_FRAMES = (30, 120, 300)
LAMBDS = (1e-4, 2.0)
INFER_TEXT_LEN, INFER_FRAMES, INFER_SIGMA = 25, 120, 0.5


def model_params():
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=2)
    params = synth.synth_params(cfg, SEED)
    key = [k for k in params if k.endswith("gate_layer.linear_layer.bias")][0]
    params[key] = torch.full_like(params[key], GATE_BIAS)
    return cfg, params


def inputs(cfg):
    g = torch.Generator().manual_seed(SEED)
    K, T, L = len(OUT_LENS), max(OUT_LENS), max(IN_LENS)
    mel = (torch.randn(K, 80, T, generator=g) * 2.0 - 5.5).clamp_(-11.5, 2.0)
    text = torch.randint(0, cfg["n_text"], (K, L), generator=g)
    spk = torch.zeros(K, dtype=torch.long)
    return mel, text, spk


def posterior_mean_f64(z, out_lens, n_frames, lambd, aggregation):
    """The notebook's arithmetic restated: z [K, 80, T] (row k valid in [0, out_lens[k])) -> [80, n_frames] or [80, 1]."""
    K = len(out_lens)
    rows = [z[k, :, :n].astype(np.float64) for k, n in enumerate(out_lens)]
    if aggregation == "batch":
        mean = np.mean([r[:, np.arange(n_frames) % r.shape[1]] for r in rows], axis=0)
    else:
        mean = np.mean([r.mean(axis=1) for r in rows], axis=0)[:, None]
    ratio = K / lambd
    return ratio * mean / (ratio + 1.0)


def main():
    from oracle import ref_shims
    assert ref_shims.available(), "the reference tree is needed to generate fixtures"
    torch.set_num_threads(os.cpu_count() or 1)
    cfg, params = model_params()
    _, model = ref_shims.reference_model(cfg, params)
    mel, text, spk = inputs(cfg)
    K, T = len(OUT_LENS), mel.shape[-1]
    z = np.zeros((K, 80, T), dtype=np.float32)
    with torch.no_grad():
        for k, (nl, nt) in enumerate(zip(IN_LENS, OUT_LENS)):
            zk = model(mel[k:k + 1, :, :nt], spk[k:k + 1], text[k:k + 1, :nl], torch.LongTensor([nl]),
                       torch.LongTensor([nt]))[0]
            z[k, :, :nt] = zk.permute(1, 2, 0)[0].numpy()
    np.savez_compressed(os.path.join(OUT, "style_encode.npz"), seed=SEED, gate_bias=np.float32(GATE_BIAS),
                        mel=mel.numpy(), text=text.numpy(), speaker_ids=spk.numpy(),
                        in_lens=np.array(IN_LENS, dtype=np.int64), out_lens=np.array(OUT_LENS, dtype=np.int64), z=z)
    print(f"style_encode: K {K}, in_lens {IN_LENS}, out_lens {OUT_LENS}, max|z| {np.abs(z).max():.3f}")

    rec = dict(n_frames=np.array(N_FRAMES, dtype=np.int64), lambds=np.array(LAMBDS, dtype=np.float64))
    for li, lambd in enumerate(LAMBDS):
        for n in N_FRAMES:
            for agg in ("batch", "time_and_batch"):
                rec[f"mu_{agg}_n{n}_l{li}"] = posterior_mean_f64(z, OUT_LENS, n, lambd, agg)
    g = torch.Generator().manual_seed(SEED + 1)
    noise = torch.randn(1, 80, INFER_FRAMES, generator=g)
    infer_text = torch.randint(0, cfg["n_text"], (1, INFER_TEXT_LEN), generator=g)
    mu = torch.from_numpy(rec[f"mu_batch_n{INFER_FRAMES}_l0"]).float()[None]
    residual = mu + INFER_SIGMA * noise
    with torch.no_grad():
        mel_out, _ = model.infer(residual, torch.zeros(1, dtype=torch.long), infer_text, temperature=1.0, gate_threshold=0.5)
    assert mel_out.shape[-1] == INFER_FRAMES, mel_out.shape
    rec.update(infer_sigma=np.float32(INFER_SIGMA), infer_noise=noise.numpy(), infer_text=infer_text.numpy(),
               infer_residual=residual.numpy(), infer_mel=mel_out.numpy())
    np.savez_compressed(os.path.join(OUT, "style_posterior.npz"), **rec)
    print(f"style_posterior: n_frames {N_FRAMES}, lambd {LAMBDS}; infer {tuple(mel_out.shape)}")


if __name__ == "__main__":
    main()
