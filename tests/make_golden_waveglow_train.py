#!/usr/bin/env python
"""Generate tests/golden/waveglow_train.npz by running the UNMODIFIED reference WaveGlow.forward and WaveGlowLoss
(tacotron2/waveglow/glow.py) and its autograd on CPU fp32, on synth.synth_waveglow_params weights.  Writes a new file only.

Run where the reference tree exists (FLOWTRON_REFERENCE, default /root/reference):
    python tests/make_golden_waveglow_train.py
  fwd_*   the shipped config at B = 2, N = 2048: z, every log_s, every log_det_W and the loss (sigma 0.7)
  grad_*  a reduced config (4 flows, early output every 2, 3 layers) at B = 2, N = 1024: every parameter's gradient of the
          loss, as its L2 norm and a seeded sample of GRAD_SAMPLES entries (flat indices and values)
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
REF = os.environ.get("FLOWTRON_REFERENCE", "/root/reference")
SIGMA = 0.7
GRAD_SAMPLES = 64
REDUCED_CONFIG = dict(synth.DEFAULT_WAVEGLOW_CONFIG, n_flows=4, n_early_every=2,
                      WN_config=dict(n_layers=3, n_channels=256, kernel_size=3))


def inputs(B, N, seed):
    """spect [B, 80, 1 + N // 256] and audio [B, N] (Mel2Samp-like segment lengths) from a seed."""
    spect = synth.synth_waveglow_mel(B, 1 + N // 256, seed)
    audio = (0.3 * torch.randn(B, N, generator=torch.Generator().manual_seed(seed + 17))).clamp(-1, 1)
    return spect, audio


def sample_index(name, numel):
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    return torch.randint(0, numel, (min(GRAD_SAMPLES, numel),), generator=g)


def main():
    torch.set_num_threads(os.cpu_count() or 1)
    sys.path.insert(0, os.path.join(REF, "tacotron2", "waveglow"))
    import glow  # noqa: the reference module
    rec = {"sigma": np.float32(SIGMA)}
    cfg = synth.DEFAULT_WAVEGLOW_CONFIG
    torch.manual_seed(0)                       # Invertible1x1Conv's QR init; overwritten by the state_dict
    m = glow.WaveGlow(**cfg)
    m.load_state_dict(synth.synth_waveglow_params(cfg, 201), strict=True)
    spect, audio = inputs(2, 2048, 202)
    with torch.no_grad():
        z, log_s, log_det = m((spect, audio))
        loss = glow.WaveGlowLoss(SIGMA)((z, log_s, log_det))
    rec.update(fwd_seed=201, fwd_input_seed=202, fwd_B=2, fwd_N=2048, fwd_z=z.numpy(), fwd_loss=np.float32(loss),
               fwd_log_det_W=np.array([float(t) for t in log_det], dtype=np.float32))
    for k, t in enumerate(log_s):
        rec[f"fwd_log_s_{k}"] = t.numpy()
    torch.manual_seed(0)
    m = glow.WaveGlow(**REDUCED_CONFIG)
    m.load_state_dict(synth.synth_waveglow_params(REDUCED_CONFIG, 203), strict=True)
    spect, audio = inputs(2, 1024, 204)
    loss = glow.WaveGlowLoss(SIGMA)(m((spect, audio)))
    loss.backward()
    rec.update(grad_seed=203, grad_input_seed=204, grad_B=2, grad_N=1024, grad_loss=np.float32(loss.item()))
    names = []
    for name, p in m.named_parameters():
        idx = sample_index(name, p.numel())
        names.append(name)
        rec[f"grad_norm/{name}"] = np.float32(p.grad.norm())
        rec[f"grad_idx/{name}"] = idx.numpy().astype(np.int64)
        rec[f"grad_val/{name}"] = p.grad.flatten()[idx].numpy()
    rec["grad_names"] = np.array(names)
    np.savez_compressed(os.path.join(OUT, "waveglow_train.npz"), **rec)
    print("loss", float(rec["fwd_loss"]), "reduced loss", float(rec["grad_loss"]), len(names), "parameters")


if __name__ == "__main__":
    main()
