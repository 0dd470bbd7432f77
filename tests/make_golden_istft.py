#!/usr/bin/env python
"""Generate tests/golden/istft.npz, griffin_lim.npz and denoiser.npz by running the UNMODIFIED reference on CPU fp32:
STFT.inverse and griffin_lim of audio_processing.py, and the Denoiser of tacotron2/waveglow/denoiser.py on the reference
WaveGlow.  Writes these new files only; the other fixtures are left as they are.

Run where the reference tree exists (FLOWTRON_REFERENCE, default /root/reference):
    python tests/make_golden_istft.py
Inputs are functions of a seed (flowtron_b200.synth) or committed fixtures, so the files store outputs and seeds only.
Shims: the librosa stub of oracle.ref_shims; WaveGlow's noise draws fed zeros through make_golden_waveglow's _NoiseFeed
(the Denoiser runs WaveGlow at sigma 0); Module.cuda / Tensor.cuda as identities so the Denoiser runs on the host.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
from flowtron_b200 import synth  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")

# tag -> (kind, seed, B, N samples (audio) or F frames (spectrum), hop, win_length)
ISTFT_CASES = {
    "audio_h256": ("audio", 31, 2, 6000, 256, 1024),
    "random_h256": ("spectrum", 32, 2, 24, 256, 1024),
    "audio_h128_w800": ("audio", 33, 1, 5000, 128, 800),
    "random_h512": ("spectrum", 34, 2, 20, 512, 1024),
}
GL = dict(seed=41, B=1, N=8192, hop=256, np_seed=1234, iters=(8, 30))
DENOISER = dict(wg_seed=102, input="waveglow_b2.npz", strengths=(0.1, 0.5))


def istft_input(AP, kind, seed, B, n, hop, win):
    """(magnitude, phase) for a case: the reference transform of seeded audio, or a random inconsistent pair."""
    if kind == "audio":
        return AP.STFT(1024, hop, win).transform(synth.synth_istft_audio(B, n, seed))
    return synth.synth_istft_spectrum(B, n, seed)


def istft_cases(AP):
    rec = {}
    for tag, (kind, seed, B, n, hop, win) in ISTFT_CASES.items():
        with torch.no_grad():
            mag, phase = istft_input(AP, kind, seed, B, n, hop, win)
            out = AP.STFT(1024, hop, win).inverse(mag, phase)
        rec[f"{tag}_out"] = out.numpy().astype(np.float32)
        print(tag, tuple(out.shape), float(out.abs().max()))
    np.savez_compressed(os.path.join(OUT, "istft.npz"), **rec)


def griffin_lim_case(AP):
    stft = AP.STFT(1024, GL["hop"], 1024)
    with torch.no_grad():
        mag, _ = stft.transform(synth.synth_istft_audio(GL["B"], GL["N"], GL["seed"]))
        rec = {}
        for n in GL["iters"]:
            np.random.seed(GL["np_seed"])
            rec[f"out_{n}"] = AP.griffin_lim(mag, stft, n_iters=n).numpy().astype(np.float32)
            print("griffin_lim", n, rec[f"out_{n}"].shape, float(np.abs(rec[f"out_{n}"]).max()))
    np.savez_compressed(os.path.join(OUT, "griffin_lim.npz"), **rec)


def denoiser_case():
    import make_golden_waveglow as mgw
    from oracle import ref_shims
    glow = mgw.import_glow()
    sys.path.insert(0, os.path.join(ref_shims.REF, "tacotron2"))
    torch.nn.Module.cuda = lambda self, *a, **k: self
    torch.Tensor.cuda = lambda self, *a, **k: self
    import denoiser as D  # noqa: the reference module (tacotron2/waveglow/denoiser.py)
    cfg = synth.DEFAULT_WAVEGLOW_CONFIG
    wg = mgw.reference_model(glow, cfg, synth.synth_waveglow_params(cfg, DENOISER["wg_seed"]))
    Tg = 88 * 256 // cfg["n_group"]
    c_last = synth.waveglow_channels(cfg)[-1][0]
    n_early = sum(1 for k in range(cfg["n_flows"]) if k % cfg["n_early_every"] == 0 and k > 0)
    mgw._NoiseFeed.queue = [torch.zeros(1, c_last, Tg)] + [torch.zeros(1, cfg["n_early_size"], Tg)] * n_early
    den = D.Denoiser(wg)
    assert not mgw._NoiseFeed.queue
    audio = torch.from_numpy(np.load(os.path.join(OUT, DENOISER["input"]))["audio"])
    rec = {"bias_spec": den.bias_spec.numpy().astype(np.float32)}
    sd = den.state_dict()
    rec["state_keys"] = np.array(list(sd.keys()))
    rec["state_shapes"] = np.array([list(v.shape) + [0] * (3 - v.dim()) for v in sd.values()], dtype=np.int64)
    with torch.no_grad():
        for s in DENOISER["strengths"]:
            rec[f"out_{s}"] = den(audio, s).numpy().astype(np.float32)
            print("denoiser", s, rec[f"out_{s}"].shape, float(np.abs(rec[f"out_{s}"]).max()))
    np.savez_compressed(os.path.join(OUT, "denoiser.npz"), **rec)


def main():
    from oracle import ref_shims
    assert ref_shims.available(), "the reference tree is needed to generate fixtures"
    torch.set_num_threads(os.cpu_count() or 1)
    AP = ref_shims.import_audio_processing()
    istft_cases(AP)
    griffin_lim_case(AP)
    denoiser_case()


if __name__ == "__main__":
    main()
