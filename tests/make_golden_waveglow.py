#!/usr/bin/env python
"""Generate tests/golden/waveglow_*.npz and waveglow_keys.json by running the UNMODIFIED reference WaveGlow
(tacotron2/waveglow/glow.py) on CPU fp32.  Writes new files only; the other fixtures are left as they are.

Run where the reference tree exists (FLOWTRON_REFERENCE, default /root/reference):
    python tests/make_golden_waveglow.py
Weights, mel inputs and noise are functions of a seed (flowtron_b200.synth), so the fixtures store outputs and seeds only.
WaveGlow.infer draws its noise with torch.cuda.FloatTensor(...).normal_(); the shim below hands out the fixture's noise
instead, in draw order (the first flow's channels, then each early injection), so the reference runs on the host.
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from flowtron_b200 import synth  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
REF = os.environ.get("FLOWTRON_REFERENCE", "/root/reference")
SIGMA = 0.6


class _NoiseFeed:
    """Stands in for torch.cuda.FloatTensor(B, c, T): returns the next slice of the fixture noise; normal_() is a no-op."""
    queue: list = []

    def __init__(self, *size):
        t = self.queue.pop(0)
        assert tuple(t.shape) == tuple(size), (t.shape, size)
        self.t = t

    def normal_(self):
        return self.t


def import_glow():
    sys.path.insert(0, os.path.join(REF, "tacotron2", "waveglow"))
    import glow  # noqa: the reference module
    torch.cuda.FloatTensor = _NoiseFeed
    return glow


def reference_model(glow, cfg, sd):
    torch.manual_seed(0)                      # Invertible1x1Conv's QR init; overwritten by the state_dict
    m = glow.WaveGlow(**cfg)
    m.load_state_dict(sd, strict=True)
    return m.eval()


def run_reference(model, mel, noise, cfg):
    chans = synth.waveglow_channels(cfg)
    B, Tg = noise.shape[0], noise.shape[2]
    c = chans[-1][0]
    q = [noise[:, 8 - c:].clone()]
    for k in reversed(range(cfg["n_flows"])):
        if k % cfg["n_early_every"] == 0 and k > 0:
            ck, e = chans[k][0], cfg["n_early_size"]
            q.append(noise[:, 8 - ck - e: 8 - ck].clone())
    _NoiseFeed.queue = q
    with torch.no_grad():
        audio = model.infer(mel, sigma=SIGMA)
    assert not _NoiseFeed.queue
    assert audio.shape == (B, Tg * 8)
    return audio


def case(glow, tag, B, Fr, seed, lengths=None):
    cfg = synth.DEFAULT_WAVEGLOW_CONFIG
    sd = synth.synth_waveglow_params(cfg, seed)
    model = reference_model(glow, cfg, sd)
    mel = synth.synth_waveglow_mel(B, Fr, seed)
    noise = synth.synth_waveglow_noise(B, Fr, seed)
    if lengths is None:
        audio = run_reference(model, mel, noise, cfg)
    else:                                                    # each row is its own B=1 reference run
        audio = torch.zeros(B, 256 * Fr)
        for b, n in enumerate(lengths):
            audio[b, :256 * n] = run_reference(model, mel[b:b + 1, :, :n].contiguous(), noise[b:b + 1, :, :32 * n].contiguous(),
                                               cfg)[0]
    rec = dict(seed=seed, B=B, F=Fr, sigma=np.float32(SIGMA), audio=audio.numpy().astype(np.float32))
    if lengths is not None:
        rec["lengths"] = np.asarray(lengths, dtype=np.int64)
    np.savez_compressed(os.path.join(OUT, f"waveglow_{tag}.npz"), **rec)
    print(tag, audio.shape, float(audio.abs().max()))


def keys_case(glow):
    cfg = synth.DEFAULT_WAVEGLOW_CONFIG
    m = reference_model(glow, cfg, synth.synth_waveglow_params(cfg, 1))
    wn_form = {k: list(v.shape) for k, v in m.state_dict().items()}
    m = glow.WaveGlow.remove_weightnorm(m)
    plain = {k: list(v.shape) for k, v in m.state_dict().items()}
    with open(os.path.join(OUT, "waveglow_keys.json"), "w") as f:
        json.dump({"weight_norm": wn_form, "plain": plain}, f, indent=0)
        f.write("\n")


def main():
    torch.set_num_threads(os.cpu_count() or 1)
    glow = import_glow()
    keys_case(glow)
    case(glow, "b1", 1, 32, 101)
    case(glow, "b2", 2, 24, 102)
    case(glow, "f96", 1, 96, 103)
    case(glow, "ragged", 2, 32, 104, lengths=[32, 19])


if __name__ == "__main__":
    main()
