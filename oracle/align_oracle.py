"""CPU restatement of the monotonic alignment search (MAS) and of one-hot maps from durations (TEST INFRASTRUCTURE),
written from the definition in include/flowtron_b200.h (ft_mas_align / ft_durations_to_attn) in float32 numpy, so the
recursion rounds exactly as the kernel's fp32 adds do and the tests can demand identical paths."""
from __future__ import annotations

import numpy as np


def mas_row(s):
    """One utterance: s float32 [Tb, Lb] in natural time, Tb >= Lb >= 1 -> token_of_frame int64 [Tb].

    Q[0][0] = s[0][0], Q[0][l > 0] = -inf; Q[t][l] = s[t][l] + max(Q[t-1][l], Q[t-1][l-1]) with Q[t-1][-1] = -inf.  The
    path ends at (Tb-1, Lb-1) and, walked back, moves to l-1 only where Q[t-1][l-1] > Q[t-1][l] (ties stay)."""
    s = np.asarray(s, dtype=np.float32)
    Tb, Lb = s.shape
    neg = np.float32(-np.inf)
    q = np.full(Lb, neg, dtype=np.float32)
    q[0] = s[0, 0]
    move = np.zeros((Tb, Lb), dtype=bool)
    for t in range(1, Tb):
        up = np.concatenate([[neg], q[:-1]]).astype(np.float32)
        mv = up > q
        move[t] = mv
        q = (s[t] + np.where(mv, up, q)).astype(np.float32)
    tok = np.empty(Tb, dtype=np.int64)
    l = Lb - 1
    for t in range(Tb - 1, -1, -1):
        tok[t] = l
        if t > 0 and move[t, l]:
            l -= 1
    return tok


def mas(logp, in_lens, out_lens, time_reversed=False):
    """logp [B, T, L], lengths [B] -> (durations int64 [B, L], token_of_frame int64 [B, T]) as ft_mas_align defines them.

    time_reversed: row b's first out_lens[b] rows are in flipped time (row q holds natural frame out_lens[b]-1-q), the order
    in which an AR_Back_Step's forward returns its maps; token_of_frame stays in natural time."""
    logp = np.asarray(logp, dtype=np.float32)
    B, T, L = logp.shape
    durations = np.zeros((B, L), dtype=np.int64)
    token_of_frame = np.full((B, T), -1, dtype=np.int64)
    for b in range(B):
        Tb, Lb = int(out_lens[b]), int(in_lens[b])
        if Lb < 1 or Tb < Lb:
            continue
        s = logp[b, :Tb, :Lb]
        tok = mas_row(s[::-1] if time_reversed else s)
        token_of_frame[b, :Tb] = tok
        durations[b, :Lb] = np.bincount(tok, minlength=Lb)
    return durations, token_of_frame


def hard_attention(durations, in_lens, n_frames_max, time_reversed=False):
    """One-hot [B, n_frames_max, L] float32: row (b, i) is generation step i -- natural frame i, or n_b-1-i when
    time_reversed, n_b = sum of row b's durations over its in_lens[b] tokens -- with a 1 at that frame's token."""
    durations = np.asarray(durations)
    B, L = durations.shape
    out = np.zeros((B, n_frames_max, L), dtype=np.float32)
    for b in range(B):
        d = np.clip(durations[b, :int(in_lens[b])], 0, None)
        tok = np.repeat(np.arange(d.size), d)
        n = tok.size
        for i in range(min(n, n_frames_max)):
            out[b, i, tok[n - 1 - i] if time_reversed else tok[i]] = 1.0
    return out
