"""Host side of AR_Step.infer / AR_Back_Step.infer (flowtron.py:775-828, 629-642) over ft_ar_step_infer."""
from __future__ import annotations

import torch

from . import _lib
from ._lib import FlowtronB200Error


def ar_step_infer(step, residual, text, attns, attn_prior=None, reversed_flag=False):
    """residual [T,B,M], text [L,B,E] -> (total_output [T',B,M], [attention_weight [B,1,L]] * T').

    B == 1: T' is where the gate fired (the reference's `break`); B > 1: per-sample stop (rows emit zeros after
    their own gate fires), T' = the longest row.  AR_Back_Step flips time on the way in and out (:629-642).

    ``attns`` (forced alignments, flowtron.py:585-588, 797): frame i uses ``attns[i]`` instead of scoring -- a [T, L] tensor
    (B == 1, the reference's ``attns[i][None, None]``), a [T, B, L] tensor, or the list of T per-frame weights this
    function returns ([B, 1, L] each).  Like the reference, a back step consumes them in its own (flipped) time order.

    L <= _lib.MAX_TEXT_LEN (1024): texts of up to 256 tokens run the short-text kernel, longer ones the long-text kernel."""
    _lib.check_text_len(text.size(0), "AR_Step.infer")
    if not residual.is_cuda:
        raise FlowtronB200Error("AR_Step.infer needs CUDA tensors: the sm_90a kernel is the only implementation")
    T, B, M = residual.shape
    L, _, E = text.shape
    dev = residual.device
    if B > 16:                                            # the kernel takes up to 16 utterances (one mma M tile): run slices
        outs, attns_o = [], []
        for b0 in range(0, B, 16):
            sl = slice(b0, min(B, b0 + 16))
            a_sl = attns
            if attns is not None:
                a_sl = torch.stack([a.reshape(B, L) for a in attns], 0)[:, sl] if isinstance(attns, (list, tuple)) \
                    else attns.reshape(-1, B, L)[:, sl]
            o, a = ar_step_infer(step, residual[:, sl], text[:, sl], a_sl, None if attn_prior is None else attn_prior[sl], reversed_flag)
            outs.append(o)
            attns_o.append(torch.stack(a, 0) if a else residual.new_zeros(0, sl.stop - sl.start, 1, L))
        n = max(o.size(0) for o in outs)
        pad = lambda t: t if t.size(0) == n else torch.cat([t, t.new_zeros(n - t.size(0), *t.shape[1:])], 0)
        if reversed_flag:       # slices that stopped earlier are left-padded in the flipped-back time order
            pad = lambda t: t if t.size(0) == n else torch.cat([t.new_zeros(n - t.size(0), *t.shape[1:]), t], 0)
        out = torch.cat([pad(o) for o in outs], 1)
        att = torch.cat([t if t.size(0) == n else torch.cat([t, t.new_zeros(n - t.size(0), *t.shape[1:])], 0) for t in attns_o], 1)
        return out, [a for a in att]
    res = residual.detach().float()
    prior = None if attn_prior is None else attn_prior.detach().float()
    if reversed_flag:
        res = torch.flip(res, (0,))
        if prior is not None:
            prior = torch.flip(prior, (1,))
    res = res.contiguous()
    prior = None if prior is None else prior.contiguous()
    has_gate = hasattr(step, 'gate_layer')
    desc = _lib.FtArStepDesc(T, B, L, M, step.lstm.hidden_size, step.attention_layer.query.linear_layer.out_features, E, 0,
                             int(has_gate), int(prior is not None), float(step.attention_layer.temperature))
    forced = None
    if attns is not None:
        if isinstance(attns, (list, tuple)):
            attns = torch.stack([a.reshape(B, L) for a in attns], 0)
        forced = attns.detach().float().reshape(-1, B, L)
        if forced.size(0) < T:
            raise ValueError(f"attns covers {forced.size(0)} frames, residual has {T}")
        forced = forced[:T].contiguous().to(dev)
    plist = [None if p is None else p.detach().contiguous() for p in step._param_list()]
    weights = _lib.make_weights(plist)
    out = torch.empty(T, B, M, device=dev)
    attn_out = torch.empty(T, B, L, device=dev)
    n_frames = torch.empty(B, dtype=torch.int32, device=dev)
    thr = float(getattr(step, 'gate_threshold', 0.5))
    _lib.ar_step_infer(desc, weights, res, text.detach().float().contiguous(), prior, forced, thr, out, attn_out, n_frames)
    n = int(n_frames.max().item())                      # one host sync per flow (the reference syncs every frame)
    if has_gate and n < T:
        print("Hitting gate limit")
    out, attn_out = out[:n], attn_out[:n]
    if reversed_flag:
        out = torch.flip(out, (0,))
    return out, [a.unsqueeze(1) for a in attn_out]


def ar_step_infer_ragged(step, residual, text, in_lens, frame_lens, reversed_flag=False):
    """Ragged-batch inverse of one flow over ft_ar_step_infer_ragged: row b equals its own B == 1 ``ar_step_infer`` on
    ``residual[:frame_lens[b], b]`` and ``text[:in_lens[b], b]``.

    residual [T,B,M] in natural time order (AR_Back_Step's reversal happens per row inside the C call), text [L,B,E],
    in_lens / frame_lens int32 CUDA [B] -> (out [T,B,M] zero past n_frames[b], attention [T,B,L] in generation order,
    n_frames int32 CUDA [B]).  No host synchronisation; batches above 16 run as slices of 16 that carry their lengths."""
    return _infer_ragged(step, residual, text, in_lens, frame_lens, None, reversed_flag, "AR_Step.infer_ragged")


def ar_step_infer_aligned(step, residual, text, in_lens, frame_lens, attns, reversed_flag=False):
    """``ar_step_infer_ragged`` with forced alignments, over ft_ar_step_infer_aligned: row b equals its own B == 1
    ``ar_step_infer(..., attns=attns[b, :frame_lens[b], :in_lens[b]])``.

    attns f32 CUDA [B, Ta, L], Ta >= max frame_lens: row (b, i) holds the weights of generation step i of utterance b -- the
    layout and, for an AR_Back_Step, the flipped per-row time order in which the flow's ``forward`` returns its attention,
    so that tensor is read where it lies.  Weights at keys >= in_lens[b] or steps >= frame_lens[b] are never read.  The
    returned attention [T,B,L] is the weights used."""
    _lib.check_text_len(text.size(0), "AR_Step.infer_aligned")
    B = residual.size(1)
    if attns.dim() != 3 or attns.size(0) != B or attns.size(2) != text.size(0) or attns.size(1) < 1:
        raise ValueError(f"attns must be [B, Ta, L] = ({B}, Ta, {text.size(0)}), got {tuple(attns.shape)}")
    if not attns.is_cuda:
        raise FlowtronB200Error("AR_Step.infer_aligned needs CUDA tensors: the sm_90a kernel is the only implementation")
    return _infer_ragged(step, residual, text, in_lens, frame_lens, attns, reversed_flag, "AR_Step.infer_aligned")


def _infer_ragged(step, residual, text, in_lens, frame_lens, attns, reversed_flag, where):
    if not residual.is_cuda:
        raise FlowtronB200Error(f"{where} needs CUDA tensors: the sm_90a kernel is the only implementation")
    T, B, M = residual.shape
    L, _, E = text.shape
    if B > 16:
        parts = [_infer_ragged(step, residual[:, b0:b0 + 16], text[:, b0:b0 + 16], in_lens[b0:b0 + 16], frame_lens[b0:b0 + 16],
                               None if attns is None else attns[b0:b0 + 16], reversed_flag, where) for b0 in range(0, B, 16)]
        return (torch.cat([p[0] for p in parts], 1), torch.cat([p[1] for p in parts], 1),
                torch.cat([p[2] for p in parts], 0))
    dev = residual.device
    has_gate = hasattr(step, 'gate_layer')
    desc = _lib.FtArStepDesc(T, B, L, M, step.lstm.hidden_size, step.attention_layer.query.linear_layer.out_features, E,
                             int(reversed_flag), int(has_gate), 0, float(step.attention_layer.temperature))
    plist = [None if p is None else p.detach().contiguous() for p in step._param_list()]
    weights = _lib.make_weights(plist)
    out = torch.empty(T, B, M, device=dev)
    attn_out = torch.empty(T, B, L, device=dev)
    n_frames = torch.empty(B, dtype=torch.int32, device=dev)
    thr = float(getattr(step, 'gate_threshold', 0.5))
    args = (desc, weights, residual.detach().float().contiguous(), text.detach().float().contiguous(),
            in_lens.to(device=dev, dtype=torch.int32).contiguous(), frame_lens.to(device=dev, dtype=torch.int32).contiguous())
    if attns is None:
        _lib.ar_step_infer_ragged(*args, thr, out, attn_out, n_frames)
    else:
        _lib.ar_step_infer_aligned(*args, attns.detach().float().contiguous(), thr, out, attn_out, n_frames)
    return out, attn_out, n_frames
