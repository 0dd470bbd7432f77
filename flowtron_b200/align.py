"""Hard alignments and duration-controlled synthesis on the sm_90a kernels (csrc/align.cu).

``mas`` turns a flow's attention log-probabilities into a hard alignment by monotonic alignment search (MAS, the Viterbi
step of "One TTS Alignment to Rule Them All"): which token each frame belongs to and how many frames each token lasts.
``hard_attention`` turns a row of per-token durations back into the one-hot maps ``Flowtron.infer_aligned`` reads.

Per-phoneme durations of a dataset, and the utterances whose alignment failed::

    durations, token_of_frame = model.align(mel, speaker_ids, text, in_lens, out_lens, attn_prior)   # [B, L], [B, T]

Changing the timing of a synthesis -- here, slowing token k of row b down to twice its length::

    durations, _ = model.align(mel, speaker_ids, text, in_lens, out_lens)      # or durations from any other source
    durations[b, k] *= 2                                                       # each row must still fit in T frames
    residual = sigma * torch.randn(B, 80, T, device=durations.device)
    mel_out, mel_lens = model.infer_durations(residual, speaker_ids, text, in_lens, durations)
    audio = waveglow.infer(mel_out, sigma=0.75, lengths=mel_lens)

``infer_durations`` builds one map per flow with ``hard_attention`` (back to front for an AR_Back_Step) and calls
``infer_aligned``; row b then lasts ``durations[b].sum()`` frames.
"""
from __future__ import annotations

import torch
from torch import Tensor

from . import _lib
from ._lib import FlowtronB200Error, check_frames_cover_tokens, ragged_lengths


def mas(logp: Tensor, in_lens, out_lens, time_reversed: bool = False):
    """Monotonic alignment search over a padded batch of attention log-probabilities.

    logp [B, T, L] f32 CUDA (a flow's ``attn_logprob``), in_lens [B] (tokens), out_lens [B] (frames) -> (durations int64
    [B, L], token_of_frame int64 [B, T]).  Row b's path runs from (0, 0) to (out_lens[b]-1, in_lens[b]-1), one token step at
    most per frame, and maximises the sum of the log-probabilities it visits; where two predecessors tie it stays on the
    token.  ``token_of_frame[b, t]`` is the path's token at frame t (natural time) and -1 from out_lens[b] on;
    ``durations[b, l]`` counts the frames of token l (each >= 1, summing to out_lens[b]) and is 0 from in_lens[b] on.
    ``time_reversed``: the rows are in an AR_Back_Step's flipped time (row q holds natural frame out_lens[b]-1-q), as its
    ``forward`` returns them.  Only t < out_lens[b] and l < in_lens[b] are read.

    Adding a per-frame constant to the log-probabilities does not change a path, so the attention, its log or its
    posterior under a prior give the same alignment.  One kernel launch (``ft_mas_align``), fp32 adds and strict compares,
    bit-for-bit the float32 restatement in ``oracle/align_oracle.py``.  Host lengths are checked (ValueError unless
    1 <= in_lens[b] <= L, 1 <= out_lens[b] <= T and out_lens[b] >= in_lens[b]); CUDA length tensors are trusted, a row with
    fewer frames than tokens then gets zero durations and -1 everywhere, and the call makes no host synchronisation, so it
    can be captured in a CUDA graph.  L <= _lib.MAX_TEXT_LEN (1024); any T.  CPU tensors raise FlowtronB200Error."""
    if not torch.is_tensor(logp) or logp.dim() != 3 or not logp.is_floating_point():
        raise ValueError(f"logp must be a float tensor [B, T, L], got "
                         f"{tuple(logp.shape) if torch.is_tensor(logp) else type(logp).__name__}")
    B, T, L = logp.shape
    if B < 1 or T < 1 or L < 1:
        raise ValueError(f"logp is empty: {tuple(logp.shape)}")
    _lib.check_text_len(L, "mas")
    in_lens = ragged_lengths(in_lens, B, L, "in_lens")
    out_lens = ragged_lengths(out_lens, B, T, "out_lens")
    check_frames_cover_tokens(in_lens, out_lens)
    if not logp.is_cuda:
        raise FlowtronB200Error("mas needs CUDA tensors: the sm_90a kernel is the only implementation")
    dev = logp.device
    in_i32 = in_lens.to(device=dev, dtype=torch.int32).contiguous()
    out_i32 = out_lens.to(device=dev, dtype=torch.int32).contiguous()
    durations = torch.empty(B, L, dtype=torch.int32, device=dev)
    token_of_frame = torch.empty(B, T, dtype=torch.int32, device=dev)
    _lib.mas_align(logp.detach().float().contiguous(), in_i32, out_i32, time_reversed, durations, token_of_frame)
    return durations.long(), token_of_frame.long()


def hard_attention(durations: Tensor, in_lens, n_frames_max: int, time_reversed: bool = False) -> Tensor:
    """One-hot attention maps from per-token durations, in the layout ``Flowtron.infer_aligned`` reads.

    durations [B, L] integer CUDA, in_lens [B] -> [B, n_frames_max, L] f32.  With n_b = durations[b, :in_lens[b]].sum(),
    row (b, i) for i < n_b is generation step i -- natural frame i, or n_b-1-i with ``time_reversed`` (an AR_Back_Step's
    order) -- and holds a 1 at the token that frame belongs to (token l lasts durations[b, l] frames, in order); every other
    entry is 0, frames past n_frames_max are cut.  Durations at l >= in_lens[b] are ignored.  One kernel launch
    (``ft_durations_to_attn``), prefix sums on the device, no host synchronisation.  Host in_lens are checked (ValueError
    unless 1 <= in_lens[b] <= L); host checks of the durations themselves are the caller's (``Flowtron.infer_durations``
    makes them).  CPU durations raise FlowtronB200Error."""
    if not torch.is_tensor(durations) or durations.dim() != 2 or durations.is_floating_point() or durations.dtype == torch.bool:
        raise ValueError(f"durations must be an integer tensor [B, L], got "
                         f"{tuple(durations.shape) if torch.is_tensor(durations) else type(durations).__name__}")
    B, L = durations.shape
    if B < 1 or L < 1:
        raise ValueError(f"durations is empty: {tuple(durations.shape)}")
    _lib.check_text_len(L, "hard_attention")
    if isinstance(n_frames_max, bool) or int(n_frames_max) != n_frames_max or n_frames_max < 1:
        raise ValueError(f"n_frames_max must be a positive integer, got {n_frames_max}")
    in_lens = ragged_lengths(in_lens, B, L, "in_lens")
    if not durations.is_cuda:
        raise FlowtronB200Error("hard_attention needs CUDA tensors: the sm_90a kernel is the only implementation")
    dev = durations.device
    out = torch.empty(B, int(n_frames_max), L, dtype=torch.float32, device=dev)
    _lib.durations_to_attn(durations.to(torch.int32).contiguous(), in_lens.to(device=dev, dtype=torch.int32).contiguous(),
                           time_reversed, out)
    return out
