"""CPU restatement of Flowtron.infer_batch (TEST INFRASTRUCTURE), built on the B = 1 ``flowtron_infer`` of
oracle/flowtron_oracle.py: the contract of the ragged-batch entry point is that every row equals its own B = 1 inference
on its unpadded text and residual, zero-padded to the residual's T.  Pinned against the reference-generated fixtures of
tests/make_golden_infer_batch.py by tests/test_infer_batch_host.py.
"""
from __future__ import annotations

import torch

from oracle.flowtron_oracle import flowtron_infer


def flowtron_infer_batch(p, residual, speaker_ids, text, in_lens, temperature=1.0, gate_threshold=0.5, max_frames=None):
    """One B = 1 ``flowtron_infer`` per row on ``text[b, :in_lens[b]]`` and ``residual[b, :, :max_frames[b]]`` (default T),
    each output zero-padded to T.  -> (mel [B, M, T], mel_lens int64 [B])."""
    B, M, T = residual.shape
    in_lens = [int(v) for v in in_lens]
    max_frames = [T] * B if max_frames is None else [int(v) for v in max_frames]
    mel = residual.new_zeros(B, M, T)
    lens = torch.zeros(B, dtype=torch.long)
    for b in range(B):
        out, _ = flowtron_infer(p, residual[b:b + 1, :, :max_frames[b]], speaker_ids[b:b + 1], text[b:b + 1, :in_lens[b]],
                                temperature, gate_threshold)
        n = out.shape[-1]
        mel[b, :, :n] = out[0]
        lens[b] = n
    return mel, lens
