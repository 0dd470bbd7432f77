#!/usr/bin/env python
"""Generate tests/golden/convert_{f2,f3,long}.npz by running the UNMODIFIED reference on CPU fp32: voice conversion with the
alignments of the recording kept.  Writes these new files only; the other fixtures are left as they are.

Run where the reference tree exists (FLOWTRON_REFERENCE, default /root/reference):
    python tests/make_golden_convert.py
Every utterance k is processed on its own, at B = 1, on its unpadded inputs:
  1. Flowtron.forward (flowtron.py:870-899) with the SOURCE speaker -> z and the flows' attention maps (``attns_list``: an
     AR_Back_Step returns its map in its own, flipped, time order);
  2. Flowtron.infer (flowtron.py:901-930) of that z with the TARGET speaker and ``attns=`` those maps -> the converted mel.
     ``infer`` indexes ``reversed(attns)`` (:925), which a plain list does not allow; the maps are handed over in a list
     whose ``__reversed__`` returns a list, so flow f gets attns[f] and the reference code runs as it is.
The files hold the padded batch (random mel frames and text tokens past each length: they must not matter), z, the maps
(zero outside each row's lengths) and the converted mels.  convert_f2 also holds a rhythm transfer: the same call with z
replaced by fresh noise (``noise`` -> ``mel_rhythm``).  Lengths come in no particular order, both speakers are sources and
targets, and convert_long has texts over 256 tokens (few frames, to keep the file small).  The gate bias is -10: the gate
never fires, every row keeps its frames.
Weights come from flowtron_b200.synth.synth_params(cfg, seed).
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
GATE_BIAS = -10.0

# tag -> n_flows, n_speakers, seed, in_lens, out_lens, source speakers, target speakers, with rhythm transfer
CASES = {
    "f2": (2, 2, 81, [17, 9, 23, 12], [52, 31, 60, 44], [0, 1, 1, 0], [1, 0, 0, 1], True),
    "f3": (3, 3, 82, [14, 21, 8, 19], [38, 57, 26, 49], [2, 0, 1, 1], [0, 1, 2, 0], False),
    "long": (2, 2, 83, [290, 352], [12, 9], [0, 1], [1, 0], False),
}


class _FlowIndexed(list):
    """Per-flow alignments for the reference's ``reversed(attns)[i]``."""

    def __reversed__(self):
        return list(self)[::-1]


def model_params(n_flows, n_speakers, seed):
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=n_flows, n_speakers=n_speakers)
    params = synth.synth_params(cfg, seed)
    key = [k for k in params if k.endswith("gate_layer.linear_layer.bias")][0]
    params[key] = torch.full_like(params[key], GATE_BIAS)
    return cfg, params


def convert_case(tag):
    from oracle import ref_shims
    n_flows, n_speakers, seed, in_lens, out_lens, src, dst, rhythm = CASES[tag]
    cfg, params = model_params(n_flows, n_speakers, seed)
    _, model = ref_shims.reference_model(cfg, params)
    g = torch.Generator().manual_seed(seed)
    K, T, L = len(in_lens), max(out_lens), max(in_lens)
    mel = (torch.randn(K, 80, T, generator=g) * 2.0 - 5.5).clamp_(-11.5, 2.0)
    text = torch.randint(0, cfg["n_text"], (K, L), generator=g)
    noise = torch.randn(K, 80, T, generator=g) * 0.5
    src_t, dst_t = torch.tensor(src), torch.tensor(dst)
    z = np.zeros((K, 80, T), dtype=np.float32)
    attns = [np.zeros((K, T, L), dtype=np.float32) for _ in range(n_flows)]
    conv = np.zeros((K, 80, T), dtype=np.float32)
    rhy = np.zeros((K, 80, T), dtype=np.float32)
    with torch.no_grad():
        for k, (nl, nt) in enumerate(zip(in_lens, out_lens)):
            txt = text[k:k + 1, :nl]
            out = model(mel[k:k + 1, :, :nt], src_t[k:k + 1], txt, torch.LongTensor([nl]), torch.LongTensor([nt]))
            zk = out[0].permute(1, 2, 0)
            z[k, :, :nt] = zk[0].numpy()
            forced = _FlowIndexed(a[0] for a in out[3])                    # [nt, nl] per flow
            for f, a in enumerate(forced):
                assert tuple(a.shape) == (nt, nl)
                attns[f][k, :nt, :nl] = a.numpy()
            m, _ = model.infer(zk, dst_t[k:k + 1], txt, temperature=1.0, gate_threshold=0.5, attns=forced)
            assert m.shape[-1] == nt, (tag, k, m.shape)
            conv[k, :, :nt] = m[0].numpy()
            if rhythm:
                m, _ = model.infer(noise[k:k + 1, :, :nt], dst_t[k:k + 1], txt, temperature=1.0, gate_threshold=0.5,
                                   attns=forced)
                assert m.shape[-1] == nt, (tag, k, m.shape)
                rhy[k, :, :nt] = m[0].numpy()
    rec = dict(cfg_n_flows=n_flows, n_speakers=n_speakers, seed=seed, gate_bias=np.float32(GATE_BIAS), mel=mel.numpy(),
               text=text.numpy(), speaker_ids=src_t.numpy(), target_speaker_ids=dst_t.numpy(),
               in_lens=np.array(in_lens, dtype=np.int64), out_lens=np.array(out_lens, dtype=np.int64), z=z,
               mel_converted=conv)
    for f, a in enumerate(attns):
        rec[f"attn_{f}"] = a
    if rhythm:
        rec.update(noise=noise.numpy(), mel_rhythm=rhy)
    np.savez_compressed(os.path.join(OUT, f"convert_{tag}.npz"), **rec)
    print(f"convert_{tag}: in_lens {in_lens} out_lens {out_lens} speakers {src} -> {dst}; max|z| {np.abs(z).max():.3f}, "
          f"max|mel - converted| {np.abs(conv - np.where(conv != 0, mel.numpy(), 0)).max():.3f}")


def main():
    from oracle import ref_shims
    assert ref_shims.available(), "the reference tree is needed to generate fixtures"
    torch.set_num_threads(os.cpu_count() or 1)
    for tag in (sys.argv[1:] or CASES):
        convert_case(tag)


if __name__ == "__main__":
    main()
