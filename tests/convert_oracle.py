"""CPU restatement of Flowtron.convert / Flowtron.infer_aligned (TEST INFRASTRUCTURE), built on the B = 1 ``flowtron_forward``
and ``flowtron_infer`` of oracle/flowtron_oracle.py: every row of the padded batch equals its own B = 1 run on its unpadded
inputs, zero-padded to T.  Pinned against the reference-generated fixtures of tests/make_golden_convert.py by
tests/test_convert_host.py.
"""
from __future__ import annotations

import torch

from oracle.flowtron_oracle import flowtron_forward, flowtron_infer


def flowtron_encode_attns(p, mel, speaker_ids, text, in_lens, out_lens):
    """One B = 1 ``flowtron_forward`` per row -> (z [B, M, T], [attn [B, T, L]] per flow), zero outside each row's lengths;
    a back step's map is in its own (flipped) time order, as forward returns it."""
    B, M, T = mel.shape
    L = text.shape[1]
    z = mel.new_zeros(B, M, T)
    attns = None
    for b in range(B):
        nl, nt = int(in_lens[b]), int(out_lens[b])
        out = flowtron_forward(p, mel[b:b + 1, :, :nt], speaker_ids[b:b + 1], text[b:b + 1, :nl], torch.tensor([nl]),
                               torch.tensor([nt]))
        z[b, :, :nt] = out[0].permute(1, 2, 0)[0]
        if attns is None:
            attns = [mel.new_zeros(B, T, L) for _ in out[3]]
        for a, o in zip(attns, out[3]):
            a[b, :nt, :nl] = o[0]
    return z, attns


def flowtron_infer_aligned(p, residual, speaker_ids, text, in_lens, attns, n_frames):
    """One B = 1 ``flowtron_infer(attns=)`` per row, the gate off -> mel [B, M, T], zero past n_frames[b]."""
    B, M, T = residual.shape
    mel = residual.new_zeros(B, M, T)
    for b in range(B):
        nl, nt = int(in_lens[b]), int(n_frames[b])
        out, _ = flowtron_infer(p, residual[b:b + 1, :, :nt], speaker_ids[b:b + 1], text[b:b + 1, :nl], gate_threshold=1.0,
                                attns=[a[b, :nt, :nl] for a in attns])
        assert out.shape[-1] == nt
        mel[b, :, :nt] = out[0]
    return mel


def flowtron_convert(p, mel, speaker_ids, target_speaker_ids, text, in_lens, out_lens):
    z, attns = flowtron_encode_attns(p, mel, speaker_ids, text, in_lens, out_lens)
    return flowtron_infer_aligned(p, z, target_speaker_ids, text, in_lens, attns, out_lens), z, attns
