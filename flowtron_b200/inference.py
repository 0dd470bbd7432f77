"""Host side of AR_Step.infer / AR_Back_Step.infer (flowtron.py:775-828, 629-642) over ft_ar_step_infer."""
from __future__ import annotations

import torch

from . import _lib
from ._lib import FlowtronB200Error


def ar_step_infer(step, residual, text, reversed_flag, in_lens=None, frame_lens=None, attns=None, attn_prior=None):
    """Per-row inverse of one flow: row b equals its own B == 1 run on ``residual[:frame_lens[b], b]`` and
    ``text[:in_lens[b], b]``.

    residual [T,B,M] in natural time order (AR_Back_Step's reversal happens per row inside the kernel), text [L,B,E],
    in_lens / frame_lens [B] (None: L / T for every row; CUDA tensors are trusted and never read on the host),
    attns f32 CUDA [B, Ta, L] or None: row (b, i) holds the forced weights of generation step i of utterance b -- the layout
    and, for a back step, the flipped per-row time order in which the flow's ``forward`` returns its attention; weights at
    keys >= in_lens[b] or steps >= frame_lens[b] are never read.  attn_prior [B, >= T, L] or None, in natural time order
    (a back step flips it, as the reference does).
    -> (out [T,B,M] zero past n_frames[b], attention [T,B,L] in generation order and zero past n_frames[b], n_frames int32
    CUDA [B]).  No host synchronisation; batches above 16 run as slices of 16 (the kernel's limit: one mma M tile).

    L <= _lib.MAX_TEXT_LEN (1024): texts of up to 256 tokens run the short-text kernel, longer ones the long-text kernel."""
    _lib.check_text_len(text.size(0), "AR_Step.infer")
    T, B, M = residual.shape
    L, _, E = text.shape
    if attns is not None:
        if attns.dim() != 3 or attns.size(0) != B or attns.size(2) != L or attns.size(1) < 1:
            raise ValueError(f"attns must be [B, Ta, L] = ({B}, Ta, {L}), got {tuple(attns.shape)}")
        if frame_lens is None and attns.size(1) < T:
            raise ValueError(f"attns covers {attns.size(1)} frames, residual has {T}")
    if attn_prior is not None:
        if attn_prior.dim() != 3 or attn_prior.size(0) != B or attn_prior.size(1) < T or attn_prior.size(2) != L:
            raise ValueError(f"attn_prior must be [B, >= T, L] = ({B}, >= {T}, {L}), got {tuple(attn_prior.shape)}")
        # row i is used at generation step i: first T rows, so the kernel's row stride T holds for every utterance
        attn_prior = (torch.flip(attn_prior, (1,)) if reversed_flag else attn_prior)[:, :T]
    if not (residual.is_cuda and text.is_cuda and all(t is None or t.is_cuda for t in (attns, attn_prior))):
        raise FlowtronB200Error("AR_Step.infer needs CUDA tensors: the sm_90a kernel is the only implementation")
    dev = residual.device
    in_lens, frame_lens = [None if t is None else t.to(device=dev, dtype=torch.int32) for t in (in_lens, frame_lens)]
    has_gate = hasattr(step, 'gate_layer')
    plist = [None if p is None else p.detach().contiguous() for p in step._param_list()]
    weights = _lib.make_weights(plist)
    thr = float(getattr(step, 'gate_threshold', 0.5))
    parts = []
    for b0 in range(0, B, 16):
        sl = slice(b0, min(B, b0 + 16))
        rows = lambda t: None if t is None else t[sl].detach().float().contiguous()
        Bs = sl.stop - sl.start
        desc = _lib.FtArStepDesc(T, Bs, L, M, step.lstm.hidden_size, step.attention_layer.query.linear_layer.out_features, E,
                                 int(reversed_flag), int(has_gate), int(attn_prior is not None),
                                 float(step.attention_layer.temperature))
        out = torch.empty(T, Bs, M, device=dev)
        attn_out = torch.empty(T, Bs, L, device=dev)
        n_frames = torch.empty(Bs, dtype=torch.int32, device=dev)
        _lib.ar_step_infer(desc, weights, residual[:, sl].detach().float().contiguous(),
                           text[:, sl].detach().float().contiguous(), None if in_lens is None else in_lens[sl].contiguous(),
                           None if frame_lens is None else frame_lens[sl].contiguous(), rows(attn_prior), rows(attns), thr,
                           out, attn_out, n_frames)
        parts.append((out, attn_out, n_frames))
    if len(parts) == 1:
        return parts[0]
    return tuple(torch.cat([p[k] for p in parts], 0 if k == 2 else 1) for k in range(3))


def batch_major(attns, B, L):
    """Forced alignments of one flow as ``Flowtron.infer`` / ``AR_Step.infer`` take them -- a [T, L] tensor (B == 1, the
    reference's ``attns[i][None, None]``), a [T, B, L] tensor, or the list of T per-frame weights ``infer`` returns
    ([B, 1, L] each) -- as the [B, T, L] layout of ``ar_step_infer``."""
    if isinstance(attns, (list, tuple)):
        attns = torch.stack([a.reshape(B, L) for a in attns], 0)
    return attns.detach().float().reshape(-1, B, L).transpose(0, 1).contiguous()


def ar_step_infer_trimmed(step, residual, text, attns, attn_prior, reversed_flag):
    """AR_Step.infer's reference API: residual [T,B,M] -> (total_output [T',B,M], [attention_weight [B,1,L]] * T').

    T' is the longest row: B == 1 stops where the gate fired (the reference's ``break``); at B > 1 each row stops at its own
    gate and emits zeros after it (the reference raises there).  ``attns``: see ``batch_major``; like the reference, a back
    step consumes them in its own (flipped) time order."""
    forced = None if attns is None else batch_major(attns, residual.size(1), text.size(0)).to(residual.device)
    out, attn, n_frames = ar_step_infer(step, residual, text, reversed_flag, attns=forced, attn_prior=attn_prior)
    n = int(n_frames.max().item())                      # one host sync per flow (the reference syncs every frame)
    if hasattr(step, 'gate_layer') and n < residual.size(0):
        print("Hitting gate limit")
    return out[:n], [a.unsqueeze(1) for a in attn[:n]]
