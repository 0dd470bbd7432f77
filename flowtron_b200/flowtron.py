"""Host-side mirror of the reference's model API for the AR-flow hot path.

Same class names, constructor signatures, attribute names and ``state_dict`` layout as
/root/reference/flowtron.py (Flowtron :831-961, AR_Step :645-828, AR_Back_Step :595-642,
Attention :528-592, DenseLayer :453-464, LinearNorm :278-288, Encoder :467-525, FlowtronLoss :185-275), so a
reference checkpoint loads with ``strict=True`` and callers switch by changing the import.

The text encoder (with the text-embedding lookup fused in), the flow steps, the NLL/gate loss and inference run on
hand-written sm_90a kernels through the C ABI (include/flowtron_b200.h).  There is NO torch/CPU fallback: CPU tensors
raise, and sizes the kernels are not built for raise NotImplementedError at construction.  The speaker embedding and
the [text ; speaker] concatenation stay ordinary PyTorch.
"""
from __future__ import annotations

import math
from typing import Optional

import numpy as np
import torch
from torch import nn, Tensor
from torch.nn import functional as F

from . import _lib
from ._lib import FlowtronB200Error
from .align import hard_attention, mas
from .inference import ar_step_infer, ar_step_infer_trimmed, batch_major


def get_mask_from_lengths(lengths: Tensor) -> Tensor:
    """flowtron.py:39-50 (device-agnostic: the reference hard-codes torch.cuda.LongTensor)."""
    max_len = int(torch.max(lengths).item())
    ids = torch.arange(0, max_len, device=lengths.device, dtype=lengths.dtype)
    return (ids < lengths.unsqueeze(1)).bool()


get_gate_mask_from_lengths = get_mask_from_lengths


# --------------------------------------------------------------------------------------------- encoder
def masked_instance_norm(input, mask, weight, bias, eps: float = 1e-5):
    """flowtron.py:53-92 with use_input_stats=True, no running stats."""
    lengths = mask.sum((-1,))
    mean = (input * mask).sum((-1,)) / lengths
    var = (((input - mean[..., None]) * mask) ** 2).sum((-1,)) / lengths
    out = (input - mean[..., None]) / torch.sqrt(var[..., None] + eps)
    return out * weight[None, :, None] + bias[None, :, None]


class MaskedInstanceNorm1d(nn.InstanceNorm1d):
    def __init__(self, num_features, eps=1e-5, momentum=0.1, affine=False, track_running_stats=False):
        super().__init__(num_features, eps, momentum, affine, track_running_stats)

    def forward(self, input, mask=None):
        if mask is None:
            return F.instance_norm(input, self.running_mean, self.running_var, self.weight, self.bias,
                                   self.training or not self.track_running_stats, self.momentum, self.eps)
        return masked_instance_norm(input, mask.to(input.dtype), self.weight, self.bias, self.eps)


class LinearNorm(nn.Module):
    def __init__(self, in_dim, out_dim, bias=True, w_init_gain='linear'):
        super().__init__()
        self.linear_layer = nn.Linear(in_dim, out_dim, bias=bias)
        nn.init.xavier_uniform_(self.linear_layer.weight, gain=nn.init.calculate_gain(w_init_gain))

    def forward(self, x):
        return self.linear_layer(x)


class ConvNorm(nn.Module):
    def __init__(self, in_channels, out_channels, kernel_size=1, stride=1, padding=None, dilation=1, bias=True,
                 w_init_gain='linear'):
        super().__init__()
        if padding is None:
            assert kernel_size % 2 == 1
            padding = int(dilation * (kernel_size - 1) / 2)
        self.conv = nn.Conv1d(in_channels, out_channels, kernel_size=kernel_size, stride=stride, padding=padding,
                              dilation=dilation, bias=bias)
        nn.init.xavier_uniform_(self.conv.weight, gain=nn.init.calculate_gain(w_init_gain))

    def forward(self, signal):
        return self.conv(signal)


class DenseLayer(nn.Module):
    def __init__(self, in_dim=1024, sizes=[1024, 1024]):
        super().__init__()
        in_sizes = [in_dim] + sizes[:-1]
        self.layers = nn.ModuleList([LinearNorm(i, o, bias=True) for (i, o) in zip(in_sizes, sizes)])

    def forward(self, x):
        for linear in self.layers:
            x = torch.tanh(linear(x))
        return x


_enc_streams = {}


def _encoder_overlap_stream(device):
    key = ("overlap", device.type, device.index)
    if key not in _enc_streams:
        _enc_streams[key] = torch.cuda.Stream(device=device)
    return _enc_streams[key]


def _mel_encoder_stream(device):
    key = ("mel", device.type, device.index)
    if key not in _enc_streams:
        _enc_streams[key] = torch.cuda.Stream(device=device)
    return _enc_streams[key]


def _kernel_params(enc):
    """Encoder / MelEncoder parameters in ENC_PARAM_FIELDS / MEL_ENC_PARAM_FIELDS order."""
    cs = enc.convolutions
    flat = [c[0].conv.weight for c in cs] + [c[0].conv.bias for c in cs] + [c[1].weight for c in cs] + [c[1].bias for c in cs]
    for n in ("weight_ih_l0", "weight_hh_l0", "bias_ih_l0", "bias_hh_l0"):
        flat += [getattr(enc.lstm, n), getattr(enc.lstm, n + "_reverse")]
    return flat


def _unflatten_params(fields, flat_params):
    """flat parameters (the _kernel_params order) -> dict name -> list of detached contiguous tensors."""
    params, i = {}, 0
    for n, k in fields:
        params[n] = [t.detach().contiguous() for t in flat_params[i:i + k]]
        i += k
    return params


def _flatten_grads(fields, grads):
    return [t for n, _ in fields for t in grads[n]]


class _EncoderFn(torch.autograd.Function):
    """Encoder forward / backward on the CUDA kernels for up to 64 utterances: ft_encoder_fwd / ft_encoder_bwd on x [B, 512, L],
    or, given tokens [B, L] and the embedding weight instead of x, ft_encoder_fwd_tokens / ft_encoder_bwd_tokens, which fuse the
    row gather into the first kernel and scatter the embedding gradient from the last one."""

    @staticmethod
    def forward(ctx, enc, x, tokens, emb_weight, in_lens, masked, dropout_p, *flat_params):
        params = _unflatten_params(_lib.ENC_PARAM_FIELDS, flat_params)
        if x is None:
            B, L = tokens.shape
            tokens, emb_weight, dev = tokens.contiguous(), emb_weight.detach().contiguous(), tokens.device
        else:
            B, _, L = x.shape
            x, dev = x.detach().contiguous().float(), x.device
        desc = _lib.encoder_desc(B, L, masked, dropout_p, enc.convolutions[0][1].eps)
        lens32 = in_lens.to(torch.int32) if masked else None
        out = torch.empty(B, L, 512, dtype=torch.float32, device=dev)
        rng = enc._rng_state(dev) if dropout_p > 0 else None
        saved = _lib.encoder_fwd(desc, params, x, lens32, rng, out, out.stride(0), out.stride(1), tokens=tokens, emb_weight=emb_weight)
        ctx.desc, ctx.params, ctx.saved, ctx.tokens, ctx.emb_weight = desc, params, saved, tokens, emb_weight
        return out

    @staticmethod
    def backward(ctx, d_out):
        if ctx.saved is None:
            raise RuntimeError("Encoder backward called twice (the saved activations were released)")
        d_in, grads = _lib.encoder_bwd(ctx.desc, ctx.params, d_out.contiguous().float(), ctx.saved, need_dx=ctx.needs_input_grad[1],
                                       tokens=ctx.tokens, emb_weight=ctx.emb_weight)
        ctx.saved = None
        d_x, d_emb = (d_in, None) if ctx.tokens is None else (None, d_in)
        return (None, d_x, None, d_emb, None, None, None, *_flatten_grads(_lib.ENC_PARAM_FIELDS, grads))


_ENC_MAX_BATCH = 64                  # utterances per encoder-kernel call (the kernels reject more)


class Encoder(nn.Module):
    """flowtron.py:467-525 (3 x conv+masked instance norm+relu+dropout, packed BiLSTM) on the encoder kernels
    (csrc/encoder.cu), which are built for 512 channels, 3 convolutions of width 5 and MaskedInstanceNorm1d."""

    def __init__(self, encoder_n_convolutions=3, encoder_embedding_dim=512, encoder_kernel_size=5, norm_fn=nn.BatchNorm1d):
        super().__init__()
        if (encoder_n_convolutions != 3 or encoder_kernel_size != 5 or encoder_embedding_dim != 512
                or norm_fn is not MaskedInstanceNorm1d):
            raise NotImplementedError("the sm_90a encoder kernels are built for encoder_n_convolutions=3, encoder_kernel_size=5, "
                                      "encoder_embedding_dim=512 and norm_fn=MaskedInstanceNorm1d (Flowtron with n_text_dim=512)")
        convolutions = []
        for _ in range(encoder_n_convolutions):
            convolutions.append(nn.Sequential(
                ConvNorm(encoder_embedding_dim, encoder_embedding_dim, kernel_size=encoder_kernel_size, stride=1,
                         padding=int((encoder_kernel_size - 1) / 2), dilation=1, w_init_gain='relu'),
                norm_fn(encoder_embedding_dim, affine=True)))
        self.convolutions = nn.ModuleList(convolutions)
        self.lstm = nn.LSTM(encoder_embedding_dim, int(encoder_embedding_dim / 2), 1, batch_first=True, bidirectional=True)
        self.p_dropout = 0.5        # flowtron.py:502 hard-codes 0.5; exposed so tests can run deterministic train-mode steps
        self._rng = None

    def _rng_state(self, device):
        """device uint64[2] = {seed, call counter} of the dropout masks (advanced on the device by every training forward)."""
        if self._rng is None or self._rng.device != device:
            self._rng = torch.tensor([torch.initial_seed() & 0x7FFFFFFFFFFFFFFF, 0], dtype=torch.int64, device=device)
        return self._rng

    def _run(self, x, tokens, emb_weight, in_lens, masked, dropout=True):
        """x [B, 512, L], or tokens [B, L] with the embedding weight -> [B, L, 512].  A batch above 64 utterances runs as
        consecutive calls of at most 64 (utterances are independent); `masked` is decided from the whole batch, so a 1-row
        tail call is masked like the rest."""
        src = x if tokens is None else tokens
        if not src.is_cuda:
            raise FlowtronB200Error("Encoder needs CUDA tensors: the sm_90a kernels are the only implementation")
        C = (x if tokens is None else emb_weight).size(1)
        if C != 512:
            raise ValueError(f"the encoder kernels take 512 channels, got {C}")
        dropout_p = self.p_dropout if dropout and self.training else 0.0
        params = _kernel_params(self)
        rows = lambda t, b0: None if t is None else t[b0:b0 + _ENC_MAX_BATCH]
        outs = [_EncoderFn.apply(self, rows(x, b0), rows(tokens, b0), emb_weight, rows(in_lens, b0), masked, dropout_p, *params)
                for b0 in range(0, src.size(0), _ENC_MAX_BATCH)]
        return outs[0] if len(outs) == 1 else torch.cat(outs, 0)

    def forward(self, x, in_lens):
        """x [B, 512, L] padded to max(in_lens) (DataCollate guarantees it, data.py:200-208) -> [B, L, 512], zero at
        l >= in_lens[b]: the reference's packed BiLSTM without packing and without a host sync on in_lens."""
        return self._run(x, None, None, in_lens, x.size(0) > 1)

    def infer(self, x):
        return self._run(x, None, None, None, False)

    def forward_tokens(self, tokens, embedding, in_lens):
        """Encoder.forward(embedding(tokens).transpose(1, 2), in_lens) with the lookup fused into the encoder kernels."""
        return self._run(None, tokens, embedding.weight, in_lens, tokens.size(0) > 1)

    def infer_tokens(self, tokens, embedding):
        """Encoder.infer(embedding(tokens).transpose(1, 2)) likewise."""
        return self._run(None, tokens, embedding.weight, None, False)

    def infer_ragged_tokens(self, tokens, embedding, in_lens):
        """Encoder.forward(embedding(tokens).transpose(1, 2), in_lens) without dropout for a padded batch in any length
        order, masked at every batch size: row b equals Encoder.infer on its own first in_lens[b] tokens."""
        return self._run(None, tokens, embedding.weight, in_lens, True, dropout=False)


class _MelEncoderFn(torch.autograd.Function):
    """MelEncoder forward / backward on the CUDA kernels for up to 64 utterances (ft_mel_encoder_fwd / ft_mel_encoder_bwd).
    all_lens: the whole batch's lengths, whose maximum divides the time sum."""

    @staticmethod
    def forward(ctx, enc, mel, out_lens, all_lens, dropout_p, *flat_params):
        params = _unflatten_params(_lib.MEL_ENC_PARAM_FIELDS, flat_params)
        mel = mel.detach().contiguous().float()
        emb = torch.empty(mel.size(0), 512, dtype=torch.float32, device=mel.device)
        rng = enc._rng_state(mel.device) if dropout_p > 0 else None
        ctx.desc, ctx.saved = _lib.mel_encoder_fwd(params, mel, out_lens, all_lens, rng, dropout_p, enc.convolutions[0][1].eps, emb)
        ctx.params = params
        return emb

    @staticmethod
    def backward(ctx, d_emb):
        if ctx.saved is None:
            raise RuntimeError("MelEncoder backward called twice (the saved activations were released)")
        grads = _lib.mel_encoder_bwd(ctx.desc, ctx.params, d_emb.contiguous().float(), ctx.saved)
        ctx.saved = None
        return (None, None, None, None, None, *_flatten_grads(_lib.MEL_ENC_PARAM_FIELDS, grads))


class MelEncoder(nn.Module):
    """flowtron.py:416-439, the mel encoder of the Gaussian-mixture prior (2 x conv k=3 + masked instance norm + relu + dropout,
    packed BiLSTM, mean over time) on its CUDA kernels (csrc/mel_encoder.cu), built for 512 channels, 2 convolutions of width 3
    and MaskedInstanceNorm1d.

    Every batch size runs masked; the reference leaves a single utterance unmasked, which is the same computation when its
    length is T (the collate contract T == max(out_lens)).  The time mean divides by max(out_lens), as the reference does, so a
    row's embedding depends on the longest row of its batch.  The caller's mel is only read; frames past a row's length are
    never read."""

    def __init__(self, encoder_embedding_dim=512, encoder_kernel_size=3, encoder_n_convolutions=2, norm_fn=MaskedInstanceNorm1d):
        super().__init__()
        if (encoder_n_convolutions != 2 or encoder_kernel_size != 3 or encoder_embedding_dim != 512
                or norm_fn is not MaskedInstanceNorm1d):
            raise NotImplementedError("the sm_90a mel-encoder kernels are built for encoder_n_convolutions=2, encoder_kernel_size=3, "
                                      "encoder_embedding_dim=512 and norm_fn=MaskedInstanceNorm1d (mel_encoder_n_hidden=512)")
        convolutions = []
        for i in range(encoder_n_convolutions):
            convolutions.append(nn.Sequential(
                ConvNorm(80 if i == 0 else encoder_embedding_dim, encoder_embedding_dim, kernel_size=encoder_kernel_size, stride=1,
                         padding=int((encoder_kernel_size - 1) / 2), dilation=1, w_init_gain='relu'),
                norm_fn(encoder_embedding_dim, affine=True)))
        self.convolutions = nn.ModuleList(convolutions)
        self.lstm = nn.LSTM(encoder_embedding_dim, int(encoder_embedding_dim / 2), 1, bidirectional=True)
        self.p_dropout = 0.5        # flowtron.py:431 hard-codes 0.5; exposed so tests can run deterministic train-mode steps
        self._rng = None

    def _rng_state(self, device):
        """device uint64[2] = {seed, call counter} of the dropout masks; the seed differs from the text encoder's so the two
        encoders draw independent masks."""
        if self._rng is None or self._rng.device != device:
            seed = (torch.initial_seed() ^ 0x5DEECE66D) & 0x7FFFFFFFFFFFFFFF
            self._rng = torch.tensor([seed, 0], dtype=torch.int64, device=device)
        return self._rng

    def forward(self, x, lens):
        """x [B, 80, T] with T == max(lens), lens [B] -> [B, 512].  Batches above 64 utterances run as consecutive calls of at
        most 64, each divided by the whole batch's longest length."""
        if not x.is_cuda:
            raise FlowtronB200Error("MelEncoder needs CUDA tensors: the sm_90a kernels are the only implementation")
        if x.dim() != 3 or x.size(1) != 80:
            raise ValueError(f"MelEncoder takes mel [B, 80, T], got {tuple(x.shape)}")
        if lens is None or lens.numel() != x.size(0):
            raise ValueError("MelEncoder needs one length per utterance")
        lens32 = lens.to(device=x.device, dtype=torch.int32).contiguous()
        dropout_p = self.p_dropout if self.training else 0.0
        params = _kernel_params(self)
        mb = _lib.MEL_ENC_MAX_BATCH
        outs = [_MelEncoderFn.apply(self, x[b0:b0 + mb], lens32[b0:b0 + mb], lens32, dropout_p, *params)
                for b0 in range(0, x.size(0), mb)]
        return outs[0] if len(outs) == 1 else torch.cat(outs, 0)

    def infer(self, x):
        raise NotImplementedError("MelEncoder.infer (flowtron.py:441-450) is never called by the reference; use forward")


class GaussianMixture(nn.Module):
    """flowtron.py:313-363: mixture weights, means and log-variances of the prior from the mel embedding (three linear layers
    and a softmax, in PyTorch like the speaker embedding), or fixed mean / log_var buffers [1, n_mel, K]."""

    def __init__(self, n_hidden, n_components, n_mel_channels, fixed_gaussian, mean_scale):
        super().__init__()
        self.n_mel_channels = n_mel_channels
        self.n_components = n_components
        self.fixed_gaussian = fixed_gaussian
        self.mean_scale = mean_scale
        self.prob_layer = LinearNorm(n_hidden, n_components)
        if not fixed_gaussian:
            self.mean_layer = LinearNorm(n_hidden, n_mel_channels * n_components)
            self.log_var_layer = LinearNorm(n_hidden, n_mel_channels * n_components)
        else:
            self.register_buffer('mean', self.generate_mean(n_mel_channels, n_components, mean_scale).float())
            self.register_buffer('log_var', self.generate_log_var(n_mel_channels, n_components).float())

    def generate_mean(self, n_dimensions, n_components, scale=3):
        ids = np.random.choice(range(n_dimensions), n_components, replace=False)
        return (torch.eye(n_dimensions).float()[ids] * scale).transpose(0, 1)[None]

    def generate_log_var(self, n_dimensions, n_components):
        return torch.zeros(1, n_dimensions, n_components).float()

    def generate_prob(self):
        return torch.ones(1, 1).float()

    def forward(self, outputs, bs):
        prob = torch.softmax(self.prob_layer(outputs), dim=1)
        if not self.fixed_gaussian:
            mean = self.mean_layer(outputs).view(bs, self.n_mel_channels, self.n_components)
            log_var = self.log_var_layer(outputs).view(bs, self.n_mel_channels, self.n_components)
        else:
            mean, log_var = self.mean, self.log_var
        return mean, log_var, prob


# --------------------------------------------------------------------------------------------- attention
def _attention_run(desc, in_lens, prior, attn_given, queries, keys, values, weights):
    """One ft_attention_fwd call -> (output [B, A, T], attn, attn_logprob or None, saved work area, fp32 operands)."""
    f32 = lambda t: None if t is None else t.detach().float().contiguous()
    queries, keys, values, prior = map(f32, (queries, keys, values, prior))
    weights = [f32(w) for w in weights]
    dev = values.device
    saved_bytes, scratch_bytes = _lib.attention_sizes(desc)
    saved = torch.empty(saved_bytes, dtype=torch.uint8, device=dev)
    scratch = torch.empty(scratch_bytes, dtype=torch.uint8, device=dev)
    output = torch.empty(desc.B, desc.A, desc.T, device=dev)
    if attn_given is None:
        attn = torch.empty(desc.B, desc.T, desc.L, device=dev)
        logprob = torch.empty_like(attn)
    else:
        attn, logprob = f32(attn_given), None
    _lib.attention_fwd(desc, _lib.attention_weights(*weights), queries, keys, values, in_lens, prior, output, attn, logprob,
                       saved, scratch)
    return output, attn, logprob, saved, (queries, keys, values, *weights)


class _AttentionFn(torch.autograd.Function):
    """Attention.forward on ft_attention_fwd / ft_attention_bwd.  Returns (output, attn, attn_logprob), or (output,) when the
    weights are given: the module hands the given tensor back itself, so its own gradient path is autograd's identity."""

    @staticmethod
    def forward(ctx, desc, in_lens, prior, attn_given, queries, keys, values, w_query, w_key, w_value, w_v):
        output, attn, logprob, saved, ops = _attention_run(desc, in_lens, prior, attn_given, queries, keys, values,
                                                           (w_query, w_key, w_value, w_v))
        ctx.set_materialize_grads(False)
        ctx.desc, ctx.saved, ctx.given = desc, saved, attn_given is not None
        ctx.save_for_backward(in_lens, attn, *ops)
        if ctx.given:
            return output
        return output, attn, logprob

    @staticmethod
    def backward(ctx, d_output, d_attn=None, d_logprob=None):
        in_lens, attn, queries, keys, values, w_query, w_key, w_value, w_v = ctx.saved_tensors
        c = lambda g: None if g is None else g.float().contiguous()
        d_output, d_attn, d_logprob = map(c, (d_output, d_attn, d_logprob))
        need = ctx.needs_input_grad       # (desc, in_lens, prior, attn_given, queries, keys, values, w_query, w_key, w_value, w_v)
        new = lambda i, like: torch.empty_like(like) if need[i] else None
        d_attn_given = new(3, attn)
        d_queries, d_keys, d_values = new(4, queries), new(5, keys), new(6, values)
        g_query, g_key, g_value, g_v = new(7, w_query), new(8, w_key), new(9, w_value), new(10, w_v)
        scratch = torch.empty(_lib.attention_sizes(ctx.desc)[1], dtype=torch.uint8, device=attn.device)
        _lib.attention_bwd(ctx.desc, _lib.attention_weights(w_query, w_key, w_value, w_v), queries, keys, values, in_lens, attn,
                           d_output, d_attn, d_logprob, d_queries, d_keys, d_values, d_attn_given,
                           _lib.attention_weights(g_query, g_key, g_value, g_v), ctx.saved, scratch)
        return None, None, None, d_attn_given, d_queries, d_keys, d_values, g_query, g_key, g_value, g_v


def _attention_lengths(mask: Tensor, B: int, L: int) -> Tensor:
    """Valid keys per row of a length mask [B, L, 1] (True at padded keys); ValueError for any other mask.  One host sync."""
    if tuple(mask.shape) != (B, L, 1):
        raise ValueError(f"Attention: mask must be [B, L, 1] = {[B, L, 1]}, got {list(mask.shape)}")
    valid = ~mask[..., 0].bool()
    lens = valid.sum(1)
    if not bool((valid == (torch.arange(L, device=mask.device)[None, :] < lens[:, None])).all()):
        raise ValueError("Attention: mask must be a length mask (valid keys a prefix of each row, as get_mask_from_lengths builds)")
    if int(lens.min()) == 0:
        raise ValueError("Attention: a mask row has no valid key (the softmax of that row is undefined)")
    return lens.to(torch.int32)


class Attention(nn.Module):
    """Parameter container + mutable ``temperature`` of flowtron.py:528-592.  AR_Step reads these parameters and runs the
    math inside its fused flow-step kernels; called on its own, the module runs the same attention kernels with its own
    Q / K / V projections (ft_attention_fwd / ft_attention_bwd), differentiable in every input and parameter."""

    def __init__(self, n_mel_channels=80, n_speaker_dim=128, n_text_channels=512, n_att_channels=128, temperature=1.0):
        super().__init__()
        self.temperature = temperature
        self.query = LinearNorm(n_mel_channels, n_att_channels, bias=False, w_init_gain='tanh')
        self.key = LinearNorm(n_text_channels + n_speaker_dim, n_att_channels, bias=False, w_init_gain='tanh')
        self.value = LinearNorm(n_text_channels + n_speaker_dim, n_att_channels, bias=False, w_init_gain='tanh')
        self.v = LinearNorm(n_att_channels, 1, bias=False, w_init_gain='tanh')
        self.score_mask_value = -float("inf")

    def forward(self, queries, keys, values, mask=None, attn=None, attn_prior=None, *, in_lens=None):
        """queries [T, B, Dq], keys / values [L, B, E], mask [B, L, 1] (True at padded keys) or None, attn [B, T, L] forced
        weights or None, attn_prior [B, T, L] or None -> (output [B, A, T], attn [B, T, L], attn_logprob [B, T, L] or None), as
        flowtron.py:559-592.  in_lens: int CUDA [B] valid keys per row, the sync-free alternative to ``mask`` (trusted: each
        row needs at least one valid key).  With ``attn`` given, mask / in_lens / attn_prior are ignored and attn is returned
        as given."""
        Wq, Wk, Wv, wv = (self.query.linear_layer.weight, self.key.linear_layer.weight, self.value.linear_layer.weight,
                          self.v.linear_layer.weight)
        A, Dq, E = Wq.size(0), Wq.size(1), Wk.size(1)
        if queries.dim() != 3 or keys.dim() != 3 or tuple(values.shape) != tuple(keys.shape):
            raise ValueError(f"Attention: queries [T, B, Dq] and keys / values [L, B, E] expected, got {list(queries.shape)}, "
                             f"{list(keys.shape)}, {list(values.shape)}")
        T, B, L = queries.size(0), queries.size(1), keys.size(0)
        if queries.size(2) != Dq or keys.size(1) != B or keys.size(2) != E:
            raise ValueError(f"Attention: queries must be [T, B, {Dq}] and keys / values [L, B, {E}]")
        _lib.check_text_len(L, "Attention")
        given = attn is not None
        if given:
            if tuple(attn.shape) != (B, T, L):
                raise ValueError(f"Attention: attn must be [B, T, L] = {[B, T, L]}, got {list(attn.shape)}")
            mask = in_lens = attn_prior = None                  # ignored, as in the reference (flowtron.py:585-588)
        else:
            if mask is not None and in_lens is not None:
                raise ValueError("Attention: pass either mask or in_lens, not both")
            if attn_prior is not None:
                if attn_prior.requires_grad:
                    raise NotImplementedError("Attention: attn_prior is data; a gradient w.r.t. it is not implemented")
                if tuple(attn_prior.shape) != (B, T, L):
                    raise ValueError(f"Attention: attn_prior must be [B, T, L] = {[B, T, L]}, got {list(attn_prior.shape)}")
            if in_lens is not None and in_lens.numel() != B:
                raise ValueError("Attention: in_lens needs one length per utterance")
        if A % 8 or Dq % 8 or E % 8:
            raise NotImplementedError(f"Attention: the sm_90a projections need n_mel_channels, n_text_channels + n_speaker_dim "
                                      f"and n_att_channels to be multiples of 8 (got {Dq}, {E}, {A})")
        if mask is not None:
            in_lens = _attention_lengths(mask, B, L)
        tensors = (queries, keys, values, attn, attn_prior, in_lens, Wq)
        if not all(t.is_cuda for t in tensors if t is not None):
            raise FlowtronB200Error("Attention needs CUDA tensors: the sm_90a kernels are the only implementation")
        if in_lens is not None:
            in_lens = in_lens.to(device=queries.device, dtype=torch.int32).contiguous()
        desc = _lib.FtAttentionDesc(T, B, L, Dq, E, A, int(attn_prior is not None), int(given), float(self.temperature))
        args = (None if given else queries, None if given else keys, values,
                None if given else Wq, None if given else Wk, Wv, None if given else wv)
        if torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in (attn, *args)):
            out = _AttentionFn.apply(desc, in_lens, attn_prior, attn, *args)
            if given:
                return out, attn, None
            return out
        output, a, logprob, _, _ = _attention_run(desc, in_lens, attn_prior, attn, args[0], args[1], args[2], args[3:])
        return output, (attn if given else a), logprob


# --------------------------------------------------------------------------------------------- AR step
def _lens_i32(lens: Optional[Tensor], device) -> Optional[Tensor]:
    if lens is None:
        return None
    return lens.to(device=device, dtype=torch.int32).contiguous()


# Parameters whose gradients are produced by the attention-LSTM half of the backward (ft_ar_step_bwd_attn_lstm: the
# attention LSTM itself, plus lstm layer 0 and the attention query/key/value projections, whose weight-gradient GEMMs are
# deferred so they run underneath that BPTT kernel); indices into AR_Step._param_list() / _lib.AR_WEIGHT_FIELDS.
_ATTN_HALF = (0, 1, 2, 3, 4, 5, 6, 7, 12, 13, 14)
_MAIN_HALF = tuple(i for i in range(24) if i not in _ATTN_HALF)


class _FlowState:
    """What the two autograd nodes of one flow step share between forward and the two backward calls.  want / want_mel /
    want_text: which of the 24 parameter gradients, d_mel and d_text the backward computes (the rest are None and their
    work is skipped, ft_ar_step_bwd_plan); node_a: node A exists, i.e. mel or an _ATTN_HALF parameter requires grad."""
    __slots__ = ("desc", "saved", "plist", "mel_c", "in_lens", "out_lens", "attn", "carry", "grads", "text_shape", "has_gate",
                 "want", "want_mel", "want_text", "node_a")

    def clear(self):
        for k in self.__slots__:
            setattr(self, k, None)


class _ArStepAttnLstmFn(torch.autograd.Function):
    """Autograd node A of a flow step: owns `mel` and the _ATTN_HALF parameters.  Its forward does nothing (the whole
    forward pass is ONE C call, issued by node B); it returns a token that node B consumes, so that A.backward runs after
    B.backward.  Splitting the backward in two nodes lets the autograd engine run everything that depends only on d_text
    (the text encoder's backward, on its own stream) concurrently with the attention LSTM's BPTT of the first flow."""

    @staticmethod
    def forward(ctx, state, mel, *params_a):
        ctx.state = state
        return mel.new_zeros(1)

    @staticmethod
    def backward(ctx, g_token):
        st = ctx.state
        if st is None or st.saved is None or st.carry is None:
            raise FlowtronB200Error("AR_Step backward ran twice: the flow's saved activations are released after the first "
                                    "backward (retain_graph is not supported on the CUDA path)")
        dev = st.mel_c.device
        d_mel = torch.empty_like(st.mel_c) if st.want_mel else None
        _, scratch_bytes = _lib.ar_step_sizes(st.desc)
        scratch = _lib.scratch_buffer(scratch_bytes, dev)
        _lib.ar_step_bwd_attn_lstm(st.desc, _lib.make_weights(st.plist), st.out_lens, d_mel, _lib.make_weights(st.grads),
                                   st.saved, scratch, st.carry)
        grads_a = [st.grads[i] for i in _ATTN_HALF]
        st.clear()                                   # saved activations, carry, the output `attn` -> ctx reference cycle
        ctx.state = None
        return (None, d_mel, *grads_a)


class _ArStepFn(torch.autograd.Function):
    """Autograd node B: ft_ar_step_fwd (the whole forward) / ft_ar_step_bwd_main."""

    @staticmethod
    def forward(ctx, state, step, reversed_flag, token, mel, text, in_lens, out_lens, attn_prior, text_ready, *params_b):
        if not mel.is_cuda:
            raise FlowtronB200Error("AR_Step needs CUDA tensors: the sm_90a kernels are the only implementation")
        T, B, M = mel.shape
        L, _, E = text.shape
        dev = mel.device
        has_gate = hasattr(step, 'gate_layer')
        # What the backward has to produce (only used when grad mode made these nodes): the inputs' requires_grad.  The token
        # requires grad exactly when node A exists, and then node A's parameters need the gradients their requires_grad asks
        # for.
        need = ctx.needs_input_grad
        state.node_a, state.want_mel, state.want_text = need[3], need[4], need[5]
        params = step._param_list()
        want = [False] * 24
        for k, i in enumerate(_MAIN_HALF):
            want[i] = need[10 + k]
        for i in _ATTN_HALF:
            want[i] = state.node_a and params[i].requires_grad
        state.want = want
        desc = _lib.FtArStepDesc(T, B, L, M, step.lstm.hidden_size, step.attention_layer.query.linear_layer.out_features,
                                 E, int(reversed_flag), int(has_gate), int(attn_prior is not None),
                                 float(step.attention_layer.temperature), int(not state.want_mel))
        mel_c = mel.detach().float().contiguous()
        text_c = text.detach().float().contiguous()
        prior_c = None if attn_prior is None else attn_prior.detach().float().contiguous()
        plist = [p.detach() if p is not None else None for p in params]
        plist = [p if (p is None or p.is_contiguous()) else p.contiguous() for p in plist]
        weights = _lib.make_weights(plist)
        saved_bytes, scratch_bytes = _lib.ar_step_sizes(desc)
        saved = torch.empty(saved_bytes, dtype=torch.uint8, device=dev)
        scratch = _lib.scratch_buffer(scratch_bytes, dev)
        mel_out = torch.empty(T, B, M, device=dev)
        log_s = torch.empty(T, B, M, device=dev)
        gates = torch.empty(T, B, 1, device=dev) if has_gate else None
        attn = torch.empty(B, T, L, device=dev)
        logprob = torch.empty(B, T, L, device=dev)
        # text_ready: `text` was produced on another stream; the flow waits for it inside the C call, not here
        _lib.ar_step_fwd(desc, weights, mel_c, text_c, in_lens, out_lens, prior_c, mel_out, log_s, gates, attn, logprob,
                         saved, scratch, text_ready)
        state.desc, state.saved, state.plist = desc, saved, plist
        state.mel_c, state.in_lens, state.out_lens, state.attn = mel_c, in_lens, out_lens, attn
        state.text_shape, state.has_gate = text.shape, has_gate
        ctx.state = state
        ctx.has_gate = has_gate
        if has_gate:
            return mel_out, log_s, gates, attn, logprob
        return mel_out, log_s, attn, logprob

    @staticmethod
    def backward(ctx, *grads):
        if ctx.has_gate:
            d_mel_out, d_log_s, d_gates, d_attn, d_lp = grads
        else:
            d_mel_out, d_log_s, d_attn, d_lp = grads
            d_gates = None
        c = lambda g: None if g is None else g.float().contiguous()
        d_mel_out, d_log_s, d_gates, d_attn, d_lp = map(c, (d_mel_out, d_log_s, d_gates, d_attn, d_lp))
        st = ctx.state
        if st is None or st.saved is None:
            raise FlowtronB200Error("AR_Step backward ran twice: the flow's saved activations are released after the first "
                                    "backward (retain_graph is not supported on the CUDA path)")
        desc = st.desc
        dev = st.mel_c.device
        d_text = torch.empty(st.text_shape, device=dev, dtype=torch.float32) if st.want_text else None
        st.grads = [torch.empty_like(p) if w else None for p, w in zip(st.plist, st.want)]
        _, scratch_bytes = _lib.ar_step_sizes(desc)
        scratch = _lib.scratch_buffer(scratch_bytes, dev)
        st.carry = torch.empty(_lib.ar_step_bwd_carry_bytes(desc), dtype=torch.uint8, device=dev)
        _lib.ar_step_bwd_main(desc, _lib.make_weights(st.plist), st.mel_c, st.in_lens, st.out_lens, st.attn, d_mel_out, d_log_s,
                              d_gates, d_attn, d_lp, d_text, _lib.make_weights(st.grads), st.saved, scratch, st.carry)
        grads_b = [st.grads[i] for i in _MAIN_HALF]
        node_a = st.node_a
        if not node_a:
            st.clear()                               # no node A to release the flow's saved activations and carry
        ctx.state = None
        # (state, step, reversed, token, mel, text, in_lens, out_lens, prior, text_ready, *params_b): mel's gradient comes
        # out of node A
        return (None, None, None, torch.zeros(1, device=dev) if node_a else None, None, d_text, None, None, None, None, *grads_b)


class AR_Step(nn.Module):
    """flowtron.py:645-828.  Same parameters / state_dict keys; forward/infer run on the sm_90a kernels."""

    def __init__(self, n_mel_channels, n_speaker_dim, n_text_channels, n_in_channels, n_hidden, n_attn_channels,
                 n_lstm_layers, add_gate, use_cumm_attention):
        super().__init__()
        if use_cumm_attention:
            raise NotImplementedError("use_cumm_attention is outside the hot-path scope (off in every shipped config)")
        if n_lstm_layers != 2 or n_hidden != 1024:
            raise NotImplementedError("the sm_90a kernels are built for n_lstm_layers=2, n_hidden=1024 (config.json:56-57)")
        self.use_cumm_attention = use_cumm_attention
        self.conv = nn.Conv1d(n_hidden, 2 * n_mel_channels, 1)
        self.conv.weight.data = 0.0 * self.conv.weight.data
        self.conv.bias.data = 0.0 * self.conv.bias.data
        self.lstm = nn.LSTM(n_hidden + n_attn_channels, n_hidden, n_lstm_layers)
        self.attention_lstm = nn.LSTM(n_mel_channels, n_hidden)
        self.attention_layer = Attention(n_hidden, n_speaker_dim, n_text_channels, n_attn_channels)
        self.dense_layer = DenseLayer(in_dim=n_hidden, sizes=[n_hidden, n_hidden])
        if add_gate:
            self.gate_threshold = 0.5
            self.gate_layer = LinearNorm(n_hidden + n_attn_channels, 1, bias=True, w_init_gain='sigmoid')

    def _param_list(self):
        """Order of _lib.AR_WEIGHT_FIELDS."""
        al, ls, at, dl = self.attention_lstm, self.lstm, self.attention_layer, self.dense_layer
        gate = getattr(self, 'gate_layer', None)
        return [al.weight_ih_l0, al.weight_hh_l0, al.bias_ih_l0, al.bias_hh_l0,
                ls.weight_ih_l0, ls.weight_hh_l0, ls.bias_ih_l0, ls.bias_hh_l0,
                ls.weight_ih_l1, ls.weight_hh_l1, ls.bias_ih_l1, ls.bias_hh_l1,
                at.query.linear_layer.weight, at.key.linear_layer.weight, at.value.linear_layer.weight,
                at.v.linear_layer.weight,
                dl.layers[0].linear_layer.weight, dl.layers[0].linear_layer.bias,
                dl.layers[1].linear_layer.weight, dl.layers[1].linear_layer.bias,
                self.conv.weight, self.conv.bias,
                None if gate is None else gate.linear_layer.weight, None if gate is None else gate.linear_layer.bias]

    def _run(self, mel, text, mask, out_lens, attn_prior, reversed_flag, text_ready):
        _lib.check_text_len(text.size(0), "AR_Step")
        dev = mel.device
        in_lens = None
        if mask is not None:
            in_lens = (~mask[..., 0]).sum(1).to(torch.int32).contiguous()
        plist = self._param_list()
        state = _FlowState()
        state.clear()
        token = _ArStepAttnLstmFn.apply(state, mel, *[plist[i] for i in _ATTN_HALF])
        out = _ArStepFn.apply(state, self, reversed_flag, token, mel, text, in_lens, _lens_i32(out_lens, dev), attn_prior,
                              text_ready, *[plist[i] for i in _MAIN_HALF])
        if hasattr(self, 'gate_layer'):
            mel_out, log_s, gates, attn, lp = out
        else:
            (mel_out, log_s, attn, lp), gates = out, None
        return mel_out, log_s, gates, attn, lp

    def forward(self, mel, text, mask, out_lens, attn_prior=None, *, text_ready=None):
        """text_ready: a recorded torch.cuda.Event for `text` when another stream produces it (None: already there)."""
        return self._run(mel, text, mask, out_lens, attn_prior, False, text_ready)

    def infer(self, residual, text, attns, attn_prior=None):
        return ar_step_infer_trimmed(self, residual, text, attns, attn_prior, reversed_flag=False)

    def infer_ragged(self, residual, text, in_lens, frame_lens, attns=None, attn_prior=None):
        """Ragged batch: residual [T,B,M], text [L,B,E], in_lens / frame_lens int32 CUDA [B] or None, forced alignments
        attns [B, Ta, L] as this flow's ``forward`` returns its attention -> (out, attention [T,B,L], n_frames); see
        inference.ar_step_infer."""
        return ar_step_infer(self, residual, text, False, in_lens, frame_lens, attns, attn_prior)


class AR_Back_Step(nn.Module):
    """flowtron.py:595-642.  The flip/roll of the reference is an index map inside the kernels (no copies, no host syncs)."""

    def __init__(self, n_mel_channels, n_speaker_dim, n_text_dim, n_in_channels, n_hidden, n_attn_channels, n_lstm_layers,
                 add_gate, use_cumm_attention):
        super().__init__()
        self.ar_step = AR_Step(n_mel_channels, n_speaker_dim, n_text_dim, n_mel_channels + n_speaker_dim, n_hidden,
                               n_attn_channels, n_lstm_layers, add_gate, use_cumm_attention)

    def forward(self, mel, text, mask, out_lens, attn_prior=None, *, text_ready=None):
        if out_lens is None:
            out_lens = torch.full((mel.size(1),), mel.size(0), dtype=torch.long, device=mel.device)
        return self.ar_step._run(mel, text, mask, out_lens, attn_prior, True, text_ready)

    def infer(self, residual, text, attns, attn_prior=None):
        return ar_step_infer_trimmed(self.ar_step, residual, text, attns, attn_prior, reversed_flag=True)

    def infer_ragged(self, residual, text, in_lens, frame_lens, attns=None, attn_prior=None):
        """As AR_Step.infer_ragged; row b runs back to front over its own first frame_lens[b] frames, and row (b, i) of
        attns is generation step i, i.e. natural frame frame_lens[b] - 1 - i: the flipped order this flow's ``forward``
        returns."""
        return ar_step_infer(self.ar_step, residual, text, True, in_lens, frame_lens, attns, attn_prior)


# --------------------------------------------------------------------------------------------- model
# Padded frame count from which ft_ar_step_fwd runs the attention LSTM's input projection as a separate GEMM rather than
# folded into the recurrence (kAttnChunk + 64 in csrc/ar_step.cu); the two paths round differently.
_ATTN_OVERLAP_MIN_T = 320


def _key_padding_mask(in_lens: Tensor, L: int) -> Tensor:
    """[B, L, 1], True at the padded tokens l >= in_lens[b]; built on in_lens's device, with no host read."""
    return ~(torch.arange(L, device=in_lens.device)[None, :] < in_lens[:, None])[..., None]


# Outputs of Flowtron._encode_rows by name -> the dimension their batch runs along ([T, B, ...]: 1, [B, T, L]: 0); the
# other of dimensions 0 and 1 is time.  "log_s", "attns" and "attn_logprob" are per-flow lists.
_ENCODE_BATCH_DIM = {"z": 1, "log_s": 1, "gate": 1, "attns": 0, "attn_logprob": 0}


class Flowtron(nn.Module):
    """flowtron.py:831-961 without cumulative attention; n_components > 1 adds the Gaussian-mixture prior (MelEncoder +
    GaussianMixture), whose mean, log_var and prob `forward` returns for FlowtronLoss(gm_loss=True)."""

    def __init__(self, n_speakers, n_speaker_dim, n_text, n_text_dim, n_flows, n_mel_channels, n_hidden,
                 n_attn_channels, n_lstm_layers, use_gate_layer, mel_encoder_n_hidden, n_components, fixed_gaussian,
                 mean_scale, dummy_speaker_embedding, use_cumm_attention):
        super().__init__()
        norm_fn = MaskedInstanceNorm1d
        self.speaker_embedding = nn.Embedding(n_speakers, n_speaker_dim)
        self.embedding = nn.Embedding(n_text, n_text_dim)
        self.flows = nn.ModuleList()
        self.encoder = Encoder(norm_fn=norm_fn, encoder_embedding_dim=n_text_dim)
        self.dummy_speaker_embedding = dummy_speaker_embedding
        if n_components > 1:
            self.mel_encoder = MelEncoder(mel_encoder_n_hidden, norm_fn=norm_fn)
            self.gaussian_mixture = GaussianMixture(mel_encoder_n_hidden, n_components, n_mel_channels, fixed_gaussian, mean_scale)
        for i in range(n_flows):
            add_gate = True if (i == (n_flows - 1) and use_gate_layer) else False
            cls = AR_Step if i % 2 == 0 else AR_Back_Step
            self.flows.append(cls(n_mel_channels, n_speaker_dim, n_text_dim, n_mel_channels + n_speaker_dim, n_hidden,
                                  n_attn_channels, n_lstm_layers, add_gate, use_cumm_attention))

    # Optional: run two half batches as independent pipelines on two CUDA streams.  This does NOT shorten the recurrence
    # chain (a half batch takes as many dependent steps as the full batch); it only lets one half's GEMMs / attention /
    # launch gaps overlap the other half's recurrences.  Off by default.
    n_streams = 1
    # run the Encoder underneath the first flow's attention LSTM
    overlap_encoder = True
    min_split_batch = 8

    # Utterances per flow-kernel launch: the flow kernels take at most 32, so a larger batch (configs[2]: B = 64) runs as
    # consecutive launches of up to 32 utterances each.
    max_kernel_batch = 32

    def _run_flows(self, mel, encoder_outputs, mask, out_lens, attn_prior, text_ready=None, text_slices=None):
        """Every flow over the batch, in launches of at most max_kernel_batch utterances; the first flow of each launch
        waits for `text_ready`.  text_slices: the launches' text, made contiguous on the stream that produced it."""
        B = mel.size(1)
        mkb = self.max_kernel_batch
        if B > mkb:                            # larger batches run as consecutive chunks (utterances are independent)
            return self._run_slices([(b0, min(b0 + mkb, B)) for b0 in range(0, B, mkb)], mel, encoder_outputs, mask,
                                    out_lens, attn_prior, text_ready, text_slices)
        log_s_list, attns_list, attns_logprob_list, gate = [], [], [], None
        for i, flow in enumerate(self.flows):
            mel, log_s, gate, attn_out, attn_logprob_out = flow(mel, encoder_outputs, mask, out_lens, attn_prior,
                                                                text_ready=text_ready if i == 0 else None)
            log_s_list.append(log_s)
            attns_list.append(attn_out)
            attns_logprob_list.append(attn_logprob_out)
        return mel, log_s_list, gate, attns_list, attns_logprob_list

    def _run_slices(self, bounds, mel, encoder_outputs, mask, out_lens, attn_prior, text_ready=None, text_slices=None,
                    streams=None):
        """_run_flows on each batch slice [b0, b1) of `bounds`, outputs concatenated along the batch.  text_slices[k]
        replaces slice k of `encoder_outputs` when given.  With `streams`, slice k runs on streams[k] and the outputs are
        joined back onto the caller's stream."""
        cur = torch.cuda.current_stream() if streams else None
        parts = []
        for k, (b0, b1) in enumerate(bounds):
            if streams:
                streams[k].wait_stream(cur)
            with torch.cuda.stream(streams[k] if streams else None):     # None: stay on the current stream
                parts.append(self._run_flows(mel[:, b0:b1], encoder_outputs[:, b0:b1] if text_slices is None else text_slices[k],
                                             mask[b0:b1], None if out_lens is None else out_lens[b0:b1],
                                             None if attn_prior is None else attn_prior[b0:b1], text_ready))
        for s in streams or ():
            cur.wait_stream(s)

        def cat(ts, dim):
            if streams:
                for t in ts:
                    t.record_stream(cur)
            return torch.cat(ts, dim)
        n_flows = len(self.flows)
        return (cat([p[0] for p in parts], 1), [cat([p[1][i] for p in parts], 1) for i in range(n_flows)],
                None if parts[0][2] is None else cat([p[2] for p in parts], 1),
                [cat([p[3][i] for p in parts], 0) for i in range(n_flows)],
                [cat([p[4][i] for p in parts], 0) for i in range(n_flows)])

    def _with_speaker(self, speaker_ids, text):
        """flowtron.py:871-880: the Encoder's [B, L, n_text] output + the speaker vector -> [L, B, n_text + n_speaker]."""
        speaker_ids = speaker_ids * 0 if self.dummy_speaker_embedding else speaker_ids
        speaker_vecs = self.speaker_embedding(speaker_ids)
        text = text.transpose(0, 1)
        return torch.cat([text, speaker_vecs.expand(text.size(0), -1, -1)], 2)

    def _encode(self, speaker_ids, text, in_lens):
        return self._with_speaker(speaker_ids, self.encoder.forward_tokens(text, self.embedding, in_lens))

    def _encode_ragged(self, speaker_ids, text, in_lens):
        """_encode on the Encoder's masked kernels without dropout (in_lens int32 on the device), as the padded-batch
        entry points run it."""
        return self._with_speaker(speaker_ids, self.encoder.infer_ragged_tokens(text, self.embedding, in_lens))

    def forward(self, mel, speaker_ids, text, in_lens, out_lens, attn_prior=None):
        """Texts of up to _lib.MAX_TEXT_LEN (1024) tokens; longer ones raise ValueError before any work."""
        mean, log_var, prob = None, None, None
        n_text = text.size(1)
        _lib.check_text_len(n_text, "Flowtron.forward")
        B = mel.size(0)
        # The first flow needs the text encoding only after its attention LSTM (T dependent steps that read mel alone), so
        # the encoder's ~700 small latency-bound kernels can run on a second stream underneath it; the flow's C entry
        # point waits for `text_ready` right before it first reads the encoding.
        overlap = self.overlap_encoder and mel.is_cuda and self.n_streams <= 1 and B <= 64
        text_ready, text_slices = None, None
        if overlap:
            cur = torch.cuda.current_stream(mel.device)
            es = _encoder_overlap_stream(mel.device)
            es.wait_stream(cur)
            with torch.cuda.stream(es):
                encoder_outputs = self._encode(speaker_ids, text, in_lens)
                if B > self.max_kernel_batch:
                    # the flows will run on slices of the batch: make them contiguous HERE, on the encoder's stream, in front of
                    # the event (a .contiguous() issued later on the caller's stream would read the encoding before it exists)
                    mkb = self.max_kernel_batch
                    text_slices = [encoder_outputs[:, b0:b0 + mkb].contiguous() for b0 in range(0, B, mkb)]
                    for t in text_slices:
                        t.record_stream(cur)
                text_ready = torch.cuda.Event()
                text_ready.record(es)
            encoder_outputs.record_stream(cur)
        else:
            encoder_outputs = self._encode(speaker_ids, text, in_lens)
        # The mixture prior needs only mel: its encoder runs on a third stream beside the flows and joins the caller's stream
        # after them, so the loss (the first reader of mean / log_var / prob) waits for it on the device.
        gm_stream = None
        if hasattr(self, 'gaussian_mixture'):
            if mel.is_cuda:
                cur = torch.cuda.current_stream(mel.device)
                gm_stream = _mel_encoder_stream(mel.device)
                gm_stream.wait_stream(cur)
            with torch.cuda.stream(gm_stream):
                mel_embedding = self.mel_encoder(mel, out_lens)
                mean, log_var, prob = self.gaussian_mixture(mel_embedding, mel_embedding.size(0))
        mel = mel.permute(2, 0, 1)
        # key-padding mask from the padded text length (== max(in_lens) by the collate contract): no .item() host sync
        mask = _key_padding_mask(in_lens, n_text)
        split = self.n_streams > 1 and mel.is_cuda and B >= self.min_split_batch and out_lens is not None
        if not split:
            out = self._run_flows(mel, encoder_outputs, mask, out_lens, attn_prior, text_ready, text_slices)
        else:
            if not hasattr(self, "_side_streams") or self._side_streams[0].device != mel.device:
                self._side_streams = [torch.cuda.Stream(device=mel.device) for _ in range(2)]
            out = self._run_slices([(0, B // 2), (B // 2, B)], mel, encoder_outputs, mask, out_lens, attn_prior,
                                   streams=self._side_streams)
        if gm_stream is not None:
            cur.wait_stream(gm_stream)
            for t in (mean, log_var, prob):
                t.record_stream(cur)
        return (*out, mean, log_var, prob)

    def encode(self, mel, speaker_ids, text, in_lens, out_lens, attn_prior=None, return_attns=False):
        """The mel -> z direction for a padded batch of reference utterances, as style transfer uses it.

        mel [B, 80, T] f32, speaker_ids [B], text [B, L] int64 (row b valid in [0, in_lens[b])), in_lens [B], out_lens [B],
        attn_prior [B, T, L] or None -> z [B, 80, T], zero at t >= out_lens[b].

        Row b of ``z[:, :, :out_lens[b]]`` equals ``forward(mel[b:b+1, :, :out_lens[b]], speaker_ids[b:b+1],
        text[b:b+1, :in_lens[b]], ...)[0].permute(1, 2, 0)``: the reference notebook's one-utterance-at-a-time call.  The
        flows run as in ``forward`` (launches of at most 32 utterances) and the text encoder on its masked kernels without
        dropout, under ``torch.no_grad()`` whatever ``self.training`` is; no autograd state is kept.  ``z`` is a view of the
        flows' ``[T, B, 80]`` output, so ``style.posterior_mean`` reads it without a copy.

        Lengths given as host sequences or CPU tensors are checked (ValueError unless 1 <= in_lens[b] <= L and
        1 <= out_lens[b] <= T); CUDA length tensors are trusted, as ``forward`` trusts them, and the call makes no host
        synchronisation, so it can be captured in a CUDA graph.  Texts over _lib.MAX_TEXT_LEN tokens raise ValueError.

        The flow step computes the attention LSTM's input projection one of two ways, chosen from the padded frame count
        (folded into the recurrence below _ATTN_OVERLAP_MIN_T frames, a separate GEMM from there on), and the two round
        differently.  With host out_lens, a batch padded to at least that many frames runs its shorter rows as a separate
        launch padded to their own longest, so every row takes the path its B = 1 run takes and equals it bit for bit.
        CUDA out_lens cannot be split without a host synchronisation: such rows then differ from their B = 1 run by
        rounding (about 6e-5 of max |z| on the H100).

        ``return_attns=True`` returns ``(z, attns)``: ``attns[f]`` [B, T, L] is flow f's attention as ``forward`` returns it in
        ``attns_list`` (row b left-aligned in that flow's own time order: an AR_Back_Step's rows run back to front over
        their out_lens[b] frames), zero at t >= out_lens[b] and l >= in_lens[b] -- what ``infer_aligned`` takes."""
        checked = self._encode_args(mel, speaker_ids, text, in_lens, out_lens, attn_prior, "Flowtron.encode")
        out = self._encode_batch(mel, speaker_ids, text, attn_prior, *checked, ("z", "attns") if return_attns else ("z",))
        z = out["z"].permute(1, 2, 0)
        return (z, out["attns"]) if return_attns else z

    def _batch_args(self, where, x, x_name, speaker_ids, text, in_lens, lens, lens_name, lens_hi=None, check=None,
                    cuda=()):
        """The argument checks every padded-batch entry point makes -> (B, T, L, in_lens, lens), the lengths int32 on x's
        device (``lens`` None for an entry point without per-row frame lengths).

        x [B, n_mel, T] (``x_name`` in the messages), speaker_ids [B], text [B, L] with L <= _lib.MAX_TEXT_LEN.  Host
        in_lens must lie in [1, L] and host ``lens`` in [1, min(T, lens_hi)]; CUDA lengths are trusted and not read, so
        the call makes no host synchronisation.  ``check(B, T, L)`` makes the entry point's own ValueError checks.  Every
        ValueError comes before the CUDA check of x, text, speaker_ids and ``cuda``, and all of it before any allocation or
        launch.  An entry point that takes no text passes speaker_ids, text and in_lens as None and gets L and in_lens
        back as None."""
        has_text = text is not None
        if x.dim() != 3 or (has_text and (text.dim() != 2 or speaker_ids.dim() != 1)):
            raise ValueError(f"{where} expects {x_name} [B, n_mel, T]" + (", speaker_ids [B] and text [B, L]" if has_text else ""))
        B, _, T = x.shape
        L = text.size(1) if has_text else None
        if has_text:
            _lib.check_text_len(L, where)
        if B < 1 or T < 1 or (has_text and (text.size(0) != B or speaker_ids.size(0) != B or L < 1)):
            raise ValueError(f"{where}: batch sizes disagree or are empty: {x_name} {tuple(x.shape)}" +
                             (f", speaker_ids {tuple(speaker_ids.shape)}, text {tuple(text.shape)}" if has_text else ""))
        if check is not None:
            check(B, T, L)
        if has_text:
            in_lens = _lib.ragged_lengths(in_lens, B, L, "in_lens")
        if lens is not None:
            lens = _lib.ragged_lengths(lens, B, T if lens_hi is None else min(T, lens_hi), lens_name)
        if not all(t.is_cuda for t in (x, *((text, speaker_ids) if has_text else ()), *cuda)):
            raise FlowtronB200Error(f"{where} needs CUDA tensors: the sm_90a kernels are the only implementation")
        dev = x.device
        return (B, T, L, in_lens.to(device=dev, dtype=torch.int32) if has_text else None,
                None if lens is None else lens.to(device=dev, dtype=torch.int32))

    def mixture(self, mel, out_lens):
        """Per-utterance Gaussian-mixture parameters of a padded batch of reference mels, for ``style.sample_mixture``.

        mel [B, 80, T] f32, out_lens [B] -> (mean, log_var, prob) as ``GaussianMixture.forward`` returns them: mean /
        log_var [B, 80, K] with learned Gaussians, the fixed [1, 80, K] buffers otherwise, prob [B, K].  Row b is the
        MelEncoder + GaussianMixture of ``mel[b:b+1, :, :out_lens[b]]`` alone, in eval semantics (no dropout) whatever
        ``self.training`` is, and without autograd state.  ``forward`` instead divides every row's time sum by the batch's
        longest length (the reference's mean over the padded output); here the MelEncoder kernels run once on the batch
        and each row's embedding is rescaled by max(out_lens) / out_lens[b], so it is its own time mean.  That rescaling
        rounds twice more than the B = 1 call's single division: a row's embedding lies within 4 ulps of its B = 1 call's,
        and its mixture parameters agree with that call to 1e-5 of their largest magnitude.

        Arguments are checked as the other padded-batch entry points check them (ValueError for shapes and host lengths
        outside [1, T], FlowtronB200Error for CPU tensors); CUDA out_lens are trusted, and the call then makes no host
        synchronisation, so it can be captured in a CUDA graph.  A model without the mixture prior raises ValueError."""
        where = "Flowtron.mixture"
        if not hasattr(self, 'gaussian_mixture'):
            raise ValueError(f"{where}: the model has no Gaussian-mixture prior (n_components <= 1)")

        def check(B, T, L):
            if mel.size(1) != 80:
                raise ValueError(f"{where}: mel must be [B, 80, T], got {tuple(mel.shape)}")
        B, _, _, _, lens = self._batch_args(where, mel, "mel", None, None, None, out_lens, "out_lens", check=check)
        with torch.no_grad():
            was = self.mel_encoder.training
            self.mel_encoder.train(False)
            try:
                emb = self.mel_encoder(mel, lens)
            finally:
                self.mel_encoder.train(was)
            n = lens.float()
            emb = emb * (n.max() / n)[:, None]
            return self.gaussian_mixture(emb, B)

    def _encode_args(self, mel, speaker_ids, text, in_lens, out_lens, attn_prior, where, cuda=()):
        """encode's argument checks (``cuda``: more tensors that must be on the device) -> (in_lens, out_lens int32 on the
        device, groups: None, or for host lengths the (rows, their longest) on each side of _ATTN_OVERLAP_MIN_T)."""
        def check(B, T, L):
            if attn_prior is not None and tuple(attn_prior.shape) != (B, T, L):
                raise ValueError(f"{where}: attn_prior must be [B, T, L] = {(B, T, L)}, got {tuple(attn_prior.shape)}")
        host = not (torch.is_tensor(out_lens) and out_lens.is_cuda)
        if attn_prior is not None:
            cuda = (*cuda, attn_prior)
        B, _, _, in_lens, out_l = self._batch_args(where, mel, "mel", speaker_ids, text, in_lens, out_lens, "out_lens",
                                                   check=check, cuda=cuda)
        groups = None                       # host lengths: (rows, their longest) on each side of _ATTN_OVERLAP_MIN_T
        if host:
            lens = torch.as_tensor(out_lens).tolist()
            short = [b for b in range(B) if lens[b] < _ATTN_OVERLAP_MIN_T]
            long_rows = [b for b in range(B) if lens[b] >= _ATTN_OVERLAP_MIN_T]
            groups = [(rows, max(lens[b] for b in rows)) for rows in (short, long_rows) if rows]
        return in_lens, out_l, groups

    def _encode_batch(self, mel, speaker_ids, text, attn_prior, in_lens, out_lens, groups, outputs):
        """encode's work on checked inputs, one _encode_rows call per row group -> _encode_rows's ``outputs`` for the
        whole batch: each group's rows scattered into zeros of the batch's B and T."""
        B, T = mel.size(0), mel.size(2)
        with torch.no_grad():
            if groups is None or groups == [(list(range(B)), T)]:
                return self._encode_rows(mel, speaker_ids, text, in_lens, out_lens, attn_prior, outputs)
            full = {}
            for rows, t in groups:
                idx = torch.tensor(rows, device=mel.device)
                prior = None if attn_prior is None else attn_prior[idx, :t]
                part = self._encode_rows(mel[idx, :, :t], speaker_ids[idx], text[idx], in_lens[idx], out_lens[idx], prior,
                                         outputs)
                for key, v in part.items():
                    bd = _ENCODE_BATCH_DIM[key if isinstance(key, str) else key[0]]       # time is dimension 1 - bd
                    vs = v if isinstance(v, list) else [v]
                    if key not in full:
                        full[key] = [None if g is None else g.new_zeros(((T, B) if bd else (B, T)) + g.shape[2:])
                                     for g in vs]
                    for dst, g in zip(full[key], vs):
                        if g is not None:
                            dst.narrow(1 - bd, 0, t).index_copy_(bd, idx, g)
        return {k: v if isinstance(part[k], list) else v[0] for k, v in full.items()}

    def _encode_rows(self, mel, speaker_ids, text, in_lens, out_lens, attn_prior, outputs):
        """Flowtron.encode's work on checked inputs (lengths int32 on the device) -> {name: output} for each name in
        ``outputs``: "z" [T, B, 80], zero past out_lens; "attns", the flows' attention [B, T, L] zeroed outside each row's
        lengths; and as ``forward`` returns them, defined inside each row's lengths, "log_s" (every flow's [T, B, 80]),
        "gate" (logits [T, B, 1], or None without a gate layer) and "attn_logprob" (every flow's [B, T, L]).  A name may
        also be (name, f): flow f's tensor of a per-flow output.  Only what ``outputs`` names is masked."""
        T, dev = mel.size(2), mel.device
        encoder_outputs = self._encode_ragged(speaker_ids, text, in_lens)
        mask = _key_padding_mask(in_lens, encoder_outputs.size(0))
        z, log_s, gate, attns, logprobs = self._run_flows(mel.permute(2, 0, 1), encoder_outputs, mask, out_lens, attn_prior)
        out = {"log_s": log_s, "gate": gate, "attn_logprob": logprobs}
        if "z" in outputs or "attns" in outputs:
            # forward leaves frames at or past out_lens[b] undefined
            past = torch.arange(T, device=dev)[:, None] >= out_lens[None, :]
            out["z"] = z.masked_fill_(past[:, :, None], 0.0)
            if "attns" in outputs:
                outside = past.t()[:, :, None] | mask.transpose(1, 2)                 # [B, T, 1] | [B, 1, L]
                out["attns"] = [a.masked_fill(outside, 0.0) for a in attns]
        return {k: out[k] if isinstance(k, str) else out[k[0]][k[1]] for k in outputs}

    def infer(self, residual, speaker_ids, text, temperature=1.0, gate_threshold=0.5, attns=None, attn_prior=None):
        """residual [B, 80, T] -> (mel [B, 80, T'], attention_weights: per flow in application order, T' rows [B, 1, L]).

        T' is the longest row: with B == 1 it is where the gate fired (the reference's ``break``); with B > 1 every row
        equals its own B == 1 run and emits zeros after its own gate fired (the reference raises there, SURVEY.md 3.2).
        ``attns``: one forced alignment per flow, in flow-index order, each covering the T frames (see
        ``inference.batch_major`` for the accepted forms); ``attn_prior`` [B, >= T, L].  One host synchronisation, at the
        end.  Texts of up to _lib.MAX_TEXT_LEN (1024) tokens; longer ones raise ValueError before any work."""
        _lib.check_text_len(text.size(-1), "Flowtron.infer")
        B, _, T = residual.shape
        L = text.size(-1)
        if attns is not None:
            attns = [batch_major(a, B, L).to(residual.device) for a in attns]
            if any(a.size(1) < T for a in attns):
                raise ValueError(f"attns cover {[a.size(1) for a in attns]} frames, residual has {T}")
        encoder_outputs = self._with_speaker(speaker_ids, self.encoder.infer_tokens(text, self.embedding))
        self._set_gate(gate_threshold, temperature)
        out, attention, n_frames = self._infer_flows(residual, encoder_outputs, None, None, attns, attn_prior)
        n = int(n_frames.max().item())
        if n < T:                               # only a gate stops a row before T here
            print("Hitting gate limit")
        return out[:n].permute(1, 2, 0), [[a.unsqueeze(1) for a in attn[:n]] for attn in attention]

    def _infer_flows(self, residual, encoder_outputs, in_lens, n_frames, attns=None, attn_prior=None):
        """The per-row inverse of every flow, last flow first: residual [B, 80, T] -> (out [T, B, 80] zero past each row's
        n_frames, the flows' attention [T, B, L] in application order, n_frames int32 [B]).  The first flow applied gets
        the budgets ``n_frames`` (None: T), every later flow the previous flow's frame counts, on the device."""
        residual = residual.permute(2, 0, 1)
        attention = []
        for f in reversed(range(len(self.flows))):
            residual, attn, n_frames = self.flows[f].infer_ragged(residual, encoder_outputs, in_lens, n_frames,
                                                                  None if attns is None else attns[f], attn_prior)
            attention.append(attn)
        return residual, attention, n_frames

    def infer_batch(self, residual, speaker_ids, text, in_lens, temperature=1.0, gate_threshold=0.5, *, max_frames=None,
                    attns=None, attn_prior=None):
        """Inference over a padded batch of texts of different lengths, each with its own frame budget.

        residual [B, 80, T] f32, speaker_ids [B] int64, text [B, L] int64 (row b valid in [0, in_lens[b])), in_lens [B],
        max_frames [B] (default: T for every row) -> (mel [B, 80, T], mel_lens int64 [B], attention_weights).

        Row b of ``mel[:, :, :mel_lens[b]]`` equals ``infer(residual[b:b+1, :, :max_frames[b]], speaker_ids[b:b+1],
        text[b:b+1, :in_lens[b]])[0]`` and ``mel_lens[b]`` its length; ``mel`` is zero past ``mel_lens[b]``.  Text tokens at or
        past in_lens[b] and residual frames at or past max_frames[b] are never used.  ``attention_weights``: one [B, T, L]
        tensor per flow in the order ``infer`` returns them, in that flow's generation order, zero past the flow's output
        length and at tokens >= in_lens[b].

        The rows may come in any length order.  The first flow applied gets the budgets ``max_frames``, every later flow the
        previous flow's frame counts, on the device: there is no host synchronisation (and no "Hitting gate limit" print),
        so with lengths given as CUDA tensors the whole call can be captured in a CUDA graph.  Lengths given as host
        sequences or CPU tensors are checked first (ValueError unless 1 <= in_lens[b] <= L <= 256 and
        1 <= max_frames[b] <= T); CUDA length tensors are trusted, as ``forward`` trusts ``in_lens``.  Any B works; the flows
        run in slices of at most 16 utterances per kernel launch.  Forced alignments (``attns``) and ``attn_prior`` are
        not supported here."""
        if attns is not None or attn_prior is not None:
            raise ValueError("Flowtron.infer_batch does not take attns or attn_prior (use infer)")

        def check(B, T, L):
            if L > 256:         # the ragged entry point is validated up to 256 tokens; infer takes up to MAX_TEXT_LEN
                raise ValueError(f"Flowtron.infer_batch: text length {L} > 256 is not supported by the inference kernel")
        if max_frames is None and residual.dim() == 3:
            max_frames = [residual.size(2)] * residual.size(0)
        _, _, _, in_lens, lens = self._batch_args("Flowtron.infer_batch", residual, "residual", speaker_ids, text, in_lens,
                                                  max_frames, "max_frames", check=check)
        encoder_outputs = self._encode_ragged(speaker_ids, text, in_lens)
        self._set_gate(gate_threshold, temperature)
        out, attention, lens = self._infer_flows(residual, encoder_outputs, in_lens, lens)
        return out.permute(1, 2, 0), lens.long(), [a.transpose(0, 1) for a in attention]

    def infer_aligned(self, residual, speaker_ids, text, in_lens, attns, n_frames, gate_threshold=1.0):
        """Inference over a padded batch with forced alignments: every flow uses the given attention weights instead of
        computing its own, so each row keeps the text-to-frame timing of ``attns`` (voice conversion with the z of a recorded
        utterance, rhythm transfer with a sampled z).

        residual [B, 80, T] f32, speaker_ids [B], text [B, L] int64 (row b valid in [0, in_lens[b])), in_lens [B],
        attns: one [B, Ta, L] f32 tensor per flow in flow-index order, Ta >= max n_frames -- what
        ``encode(return_attns=True)`` returns -- n_frames [B]: frames of row b -> (mel [B, 80, T], mel_lens int64 [B]).

        Row b of ``mel[:, :, :mel_lens[b]]`` equals ``infer(residual[b:b+1, :, :n_frames[b]], speaker_ids[b:b+1],
        text[b:b+1, :in_lens[b]], gate_threshold=gate_threshold, attns=[a[b, :n_frames[b], :in_lens[b]] for a in attns])[0]``;
        ``mel`` is zero past ``mel_lens[b]``.  Weights at tokens >= in_lens[b] and frames >= n_frames[b], padded text and
        residual frames past n_frames[b] are never used.  The default gate_threshold of 1 disables the gate, so
        ``mel_lens == n_frames``; below 1 a row stops where its gate fires.  The first flow applied gets the budgets
        ``n_frames``, every later flow the previous flow's frame counts, on the device.

        Texts of up to _lib.MAX_TEXT_LEN tokens, any B (slices of 16 utterances per kernel launch), rows in any length
        order.  Host lengths are checked (ValueError unless 1 <= in_lens[b] <= L and 1 <= n_frames[b] <= min(T, Ta)); CUDA
        length tensors are trusted and the call then makes no host synchronisation, so it can be captured in a CUDA graph."""
        where = "Flowtron.infer_aligned"
        if not isinstance(attns, (list, tuple)) or len(attns) != len(self.flows):
            raise ValueError(f"{where}: attns must be a list of {len(self.flows)} tensors, one per flow")
        Ta = attns[0].size(1) if torch.is_tensor(attns[0]) and attns[0].dim() == 3 else 0

        def check(B, T, L):
            for a in attns:
                if not torch.is_tensor(a) or tuple(a.shape) != (B, Ta, L) or Ta < 1 or not a.is_floating_point():
                    raise ValueError(f"{where}: every attns[f] must be a float tensor [B, Ta, L] = ({B}, Ta, {L}), got "
                                     f"{tuple(a.shape) if torch.is_tensor(a) else type(a).__name__}")
        _, _, _, in_lens, lens = self._batch_args(where, residual, "residual", speaker_ids, text, in_lens, n_frames,
                                                  "n_frames", Ta, check, attns)
        with torch.no_grad():
            encoder_outputs = self._encode_ragged(speaker_ids, text, in_lens)
            self._set_gate(gate_threshold)                  # the temperature stays as it is
            out, _, lens = self._infer_flows(residual, encoder_outputs, in_lens, lens, attns)
        return out.permute(1, 2, 0), lens.long()

    def convert(self, mel, speaker_ids, target_speaker_ids, text, in_lens, out_lens, attn_prior=None):
        """Voice conversion of a padded batch of recorded utterances: each is mapped to z with its own speaker
        (``encode``), then z is inverted with ``target_speaker_ids`` under the alignments the first direction found
        (``infer_aligned``), so the converted utterance keeps the recording's timing.

        mel [B, 80, T] f32, speaker_ids / target_speaker_ids [B], text [B, L] int64, in_lens [B], out_lens [B], attn_prior
        [B, T, L] or None (used by the mel -> z direction only) -> mel_converted [B, 80, T], out_lens[b] frames per row, zero
        past them.  With target_speaker_ids == speaker_ids the result is ``mel`` again up to rounding.

        Arguments are checked as ``encode`` checks them; the gate is off.  With CUDA length tensors the whole call makes no
        host synchronisation and can be captured in a CUDA graph."""
        if target_speaker_ids.dim() != 1 or target_speaker_ids.size(0) != mel.size(0):
            raise ValueError(f"target_speaker_ids must hold {mel.size(0)} values, got shape {tuple(target_speaker_ids.shape)}")
        z, attns = self.encode(mel, speaker_ids, text, in_lens, out_lens, attn_prior, return_attns=True)
        return self.infer_aligned(z, target_speaker_ids, text, in_lens, attns, out_lens)[0]

    def align(self, mel, speaker_ids, text, in_lens, out_lens, attn_prior=None, flow=0):
        """Hard alignments of a padded batch of recorded utterances: which token each frame belongs to and how many frames
        each token lasts, by monotonic alignment search (``align.mas``) over flow ``flow``'s attention log-probabilities.

        mel [B, 80, T] f32, speaker_ids [B], text [B, L] int64, in_lens [B], out_lens [B], attn_prior [B, T, L] or None ->
        (durations int64 [B, L], token_of_frame int64 [B, T]): each of row b's in_lens[b] tokens lasts at least one frame,
        the durations sum to out_lens[b] and are 0 from in_lens[b] on; token_of_frame[b, t] is in natural time and -1 from
        out_lens[b] on.

        The mel -> z direction runs exactly as in ``encode``: the same argument checks, no autograd state, the text encoder
        without dropout and, with host lengths, the same short / long row split, so row b equals its own B = 1 call bit for
        bit.  The search reads the flow's ``attn_logprob`` as ``forward`` returns it (an AR_Back_Step's in flipped time,
        mapped back inside the kernel), so the path is the one under the prior's posterior when ``attn_prior`` is given and
        under log(attention + 1e-8) otherwise.  Host lengths must also give every row at least as many frames as tokens
        (ValueError); with CUDA length tensors such a row gets zero durations and -1 everywhere, and the call makes no host
        synchronisation, so it can be captured in a CUDA graph."""
        if isinstance(flow, bool) or not isinstance(flow, (int, np.integer)) or not 0 <= flow < len(self.flows):
            raise ValueError(f"Flowtron.align: flow must be a flow index in [0, {len(self.flows)}), got {flow!r}")
        _lib.check_frames_cover_tokens(in_lens, out_lens)
        checked = self._encode_args(mel, speaker_ids, text, in_lens, out_lens, attn_prior, "Flowtron.align")
        key = ("attn_logprob", int(flow))
        logp = self._encode_batch(mel, speaker_ids, text, attn_prior, *checked, (key,))[key]
        return mas(logp, checked[0], checked[1], time_reversed=isinstance(self.flows[flow], AR_Back_Step))

    def infer_durations(self, residual, speaker_ids, text, in_lens, durations, gate_threshold=1.0):
        """Inference with the timing given as per-token durations: every flow is forced onto the hard alignment in which
        token l of row b lasts durations[b, l] frames (duration editing, speaking-rate control).

        residual [B, 80, T] f32, speaker_ids [B], text [B, L] int64, in_lens [B], durations [B, L] integers (what ``align``
        returns, edited or not) -> (mel [B, 80, T], mel_lens int64 [B]).  Row b lasts n_b = durations[b, :in_lens[b]].sum()
        frames; durations past in_lens[b] are ignored.  One-hot maps (``align.hard_attention``, back to front for an
        AR_Back_Step) spanning the T frames go to ``infer_aligned`` with n_frames = n_b, computed on the device; with the
        default gate_threshold of 1 the gate is off and ``mel_lens`` is n_b.

        Host durations are checked (ValueError unless they are non-negative and every row sums to between 1 and T), as are
        host in_lens (1 <= in_lens[b] <= L); CUDA tensors are trusted, and then the call makes no host synchronisation and
        can be captured in a CUDA graph."""
        where = "Flowtron.infer_durations"

        def check(B, T, L):
            if (not torch.is_tensor(durations) or tuple(durations.shape) != (B, L) or durations.is_floating_point()
                    or durations.dtype == torch.bool):
                raise ValueError(f"{where}: durations must be an integer tensor [B, L] = ({B}, {L}), got "
                                 f"{tuple(durations.shape) if torch.is_tensor(durations) else type(durations).__name__}")
            if not durations.is_cuda:
                sums = durations.sum(1)
                if bool((durations < 0).any()) or bool((sums < 1).any()) or bool((sums > T).any()):
                    raise ValueError(f"{where}: durations must be non-negative with row sums in [1, {T}], got row sums "
                                     f"{sums.tolist()}")
        _, T, L, in_lens, _ = self._batch_args(where, residual, "residual", speaker_ids, text, in_lens, None, None,
                                               check=check)
        dev = residual.device
        durations = durations.to(device=dev)
        kept = torch.arange(L, device=dev)[None, :] < in_lens[:, None]
        n_frames = torch.where(kept, durations.clamp(min=0), 0).sum(1).to(torch.int32)
        attns = [hard_attention(durations, in_lens, T, time_reversed=isinstance(f, AR_Back_Step)) for f in self.flows]
        return self.infer_aligned(residual, speaker_ids, text, in_lens, attns, n_frames, gate_threshold)

    def score(self, mel, speaker_ids, text, in_lens, out_lens, attn_prior=None, gate_target=None, *, sigma=1.0,
              blank_logprob=-1):
        """Per-utterance losses of a padded batch of recorded utterances under this model: which rows it handles badly.

        mel [B, 80, T] f32, speaker_ids [B], text [B, L] int64, in_lens [B], out_lens [B], attn_prior [B, T, L] or None,
        gate_target [B, T] or None (None: the collate's target, 1 from frame out_lens[b] - 1 on) -> dict of CUDA f32
        tensors, FlowtronLoss's terms for each row on its own, without the batch mean:

        * ``nll`` [B]: ``(sum_{t < out_lens[b], m} z^2 / (2 sigma^2) - sum_flows sum log_s) / (out_lens[b] * 80)``.  With
          n_components > 1 the Gaussian term is the mixture NLL of FlowtronLoss(gm_loss=True), with the mixture parameters
          from the MelEncoder run once on this padded batch, as ``forward`` runs it.  That encoder averages over the padded
          length (the reference's mean over time), so mixture rows depend on the batch they come in.
        * ``gate`` [B]: the mean gate BCE over the row's frames, or None when the model has no gate layer.
        * ``ctc`` [n_flows, B]: flow f's attention-CTC cost of row b (AttentionCTCLoss's per-utterance term; a back step's
          log-probabilities are read in its flipped time by the kernel's index map).

        The batch losses follow from the rows: FlowtronLoss's ``loss`` = sum_b out_lens[b] nll[b] / sum_b out_lens[b], its
        ``gate_loss`` likewise from ``gate``, and its ``loss_ctc`` = ``ctc.mean()``.

        The mel -> z direction runs exactly as in ``encode``: eval semantics and no autograd state whatever
        ``self.training`` is, the text encoder on its masked kernels, flows in launches of at most 32 utterances, and with
        host lengths the same short / long row split, so every row of a model without the mixture equals its own B = 1
        call bit for bit.  The per-row sums (``ft_nll_rows``, ``ft_gmm_nll_rows``) have a fixed order and no atomics.  Host
        lengths are checked (ValueError); CUDA length tensors are trusted, and the call then makes no host
        synchronisation, so it can be captured in a CUDA graph.  Texts of up to _lib.MAX_TEXT_LEN tokens."""
        where = "Flowtron.score"
        if gate_target is not None and mel.dim() == 3 and tuple(gate_target.shape) != (mel.size(0), mel.size(2)):
            raise ValueError(f"{where}: gate_target must be [B, T] = {(mel.size(0), mel.size(2))}, got {tuple(gate_target.shape)}")
        mixture = hasattr(self, 'gaussian_mixture')
        if mixture and self.gaussian_mixture.n_components > _lib.GMM_MAX_COMPONENTS:
            raise ValueError(f"{where}: the mixture-NLL kernels take at most {_lib.GMM_MAX_COMPONENTS} components")
        in_l, out_l, groups = self._encode_args(mel, speaker_ids, text, in_lens, out_lens, attn_prior, where,
                                                () if gate_target is None else (gate_target,))
        B, M, T = mel.shape
        dev = mel.device
        with torch.no_grad():
            out = self._encode_batch(mel, speaker_ids, text, attn_prior, in_l, out_l, groups,
                                     ("z", "log_s", "gate", "attn_logprob"))
            z, log_s_list, gate, logprobs = out["z"], out["log_s"], out["gate"], out["attn_logprob"]
            gt = None
            if gate is not None:
                gt = (gate_target.float().contiguous() if gate_target is not None else
                      (torch.arange(T, device=dev)[None, :] >= (out_l - 1)[:, None]).float())
            rows = torch.empty(B, 4, device=dev)
            _lib.nll_rows(z.contiguous(), [ls.float().contiguous() for ls in log_s_list],
                          None if gate is None else gate.float().contiguous(), gt, out_l, rows)
            n_el = rows[:, 3] * M
            if mixture:
                was = self.mel_encoder.training
                self.mel_encoder.train(False)
                try:
                    emb = self.mel_encoder(mel, out_l)
                finally:
                    self.mel_encoder.train(was)
                mean, log_var, prob = self.gaussian_mixture(emb, B)
                gmm = torch.empty(B, device=dev)
                _lib.gmm_nll_rows(z.contiguous(), out_l, mean.float().contiguous(), log_var.float().contiguous(),
                                  prob.float().contiguous(), mean.size(0) == B, gmm)
                nll = (gmm - rows[:, 1]) / n_el
            else:
                nll = (rows[:, 0] / (2 * sigma * sigma) - rows[:, 1]) / n_el
            ctc = torch.empty(len(self.flows), B, device=dev)
            dlp = torch.empty(B, T, text.size(1), device=dev)         # the kernel's gradient output, unused here
            for f, lp in enumerate(logprobs):
                _lib.attn_ctc_loss(lp.float().contiguous(), in_l, out_l, isinstance(self.flows[f], AR_Back_Step),
                                   float(blank_logprob), ctc[f], dlp)
        return {"nll": nll, "gate": None if gate is None else rows[:, 2] / rows[:, 3], "ctc": ctc}

    def test_invertibility(self, residual, speaker_ids, text, temperature=1.0, gate_threshold=0.5, attns=None):
        """flowtron.py:932-954: mean |forward(infer(residual)) - residual| over the frames ``infer`` produced (compared
        back to front for an even number of flows, as the reference does).  Call it as ``infer``; temperature,
        gate_threshold and attns go to ``infer``, and ``forward`` then runs with the attention temperature ``infer`` set.
        Every row is taken as L tokens and the generated frame count long.  The reference expects 1e-5 or less in fp32;
        both directions here use fp16 tensor-core operands, so the value can be larger."""
        with torch.no_grad():
            mel, _ = self.infer(residual, speaker_ids, text, temperature, gate_threshold, attns)
            B, L, n = mel.size(0), text.size(-1), mel.size(2)
            in_lens = torch.full((B,), L, dtype=torch.long, device=mel.device)
            out_lens = torch.full((B,), n, dtype=torch.long, device=mel.device)
            residual_recon = self.forward(mel, speaker_ids, text, in_lens, out_lens)[0]
            residual_permuted = residual.permute(2, 0, 1)
            if len(self.flows) % 2 == 0:
                residual_permuted = torch.flip(residual_permuted, (0,))
                residual_recon = torch.flip(residual_recon, (0,))
            return (residual_recon - residual_permuted[0:residual_recon.shape[0]]).abs().mean()

    @staticmethod
    def set_temperature_and_gate(flow, temperature, gate_threshold):
        """One flow's attention temperature (None: left as it is) and, if it has a gate, its gate threshold."""
        flow = flow.ar_step if hasattr(flow, "ar_step") else flow
        if temperature is not None:
            flow.attention_layer.temperature = temperature
        if hasattr(flow, 'gate_layer'):
            flow.gate_threshold = gate_threshold

    def _set_gate(self, gate_threshold, temperature=None):
        """Every flow's gate threshold and, unless None, attention temperature, for the inverse direction."""
        for flow in self.flows:
            self.set_temperature_and_gate(flow, temperature, gate_threshold)


# --------------------------------------------------------------------------------------------- loss
class _NllGateFn(torch.autograd.Function):
    """Masked Gaussian NLL + log-det + gate BCE (flowtron.py:205-243) as two CUDA reductions."""

    @staticmethod
    def forward(ctx, sigma, z, gate_pred, gate_target, out_lens, *log_s_list):
        if not z.is_cuda:
            raise FlowtronB200Error("FlowtronLoss needs CUDA tensors")
        T, B, M = z.shape
        dev = z.device
        zc = z.detach().float().contiguous()
        lsl = [ls.detach().float().contiguous() for ls in log_s_list]
        gp = None if gate_pred is None else gate_pred.detach().float().contiguous()
        gt = None if gate_pred is None else gate_target.detach().float().contiguous()
        lens = out_lens.to(device=dev, dtype=torch.int32).contiguous()
        sums = torch.empty(4, device=dev)
        _lib.nll_reduce(zc, lsl, gp, gt, lens, sums)
        n = sums[3]
        nll = (sums[0] / (2 * sigma * sigma) - sums[1]) / (n * M)
        gate_loss = (sums[2] / n).reshape(1)
        ctx.sigma, ctx.n_flows = sigma, len(lsl)
        ctx.save = (zc, gp, gt, lens, sums, lsl)
        return nll, gate_loss

    @staticmethod
    def backward(ctx, g_nll, g_gate):
        zc, gp, gt, lens, sums, lsl = ctx.save
        dz = torch.empty_like(zc)
        dls = torch.empty_like(zc)
        dgate = None if gp is None else torch.empty_like(gp)
        gn = g_nll.reshape(1).float().contiguous()
        gg = None if g_gate is None else g_gate.reshape(1).float().contiguous()
        _lib.nll_grad(zc, gp, gt, lens, ctx.sigma, sums, gn, gg, dz, dls, dgate)
        return (None, dz, dgate, None, None, *([dls] * ctx.n_flows))


class _GmmNllFn(torch.autograd.Function):
    """Mixture NLL of the Gaussian-mixture prior over n * n_mel valid elements (flowtron.py:217-235 without the log-det term) on
    ft_gmm_nll_reduce / ft_gmm_nll_grad.  mean / log_var: [B, M, K] learned or [1, M, K] buffers (no gradient)."""

    @staticmethod
    def forward(ctx, z, out_lens, mean, log_var, prob):
        T, B, M = z.shape
        K = prob.size(1)
        if K > _lib.GMM_MAX_COMPONENTS:
            raise ValueError(f"the mixture-NLL kernels take at most {_lib.GMM_MAX_COMPONENTS} components, got {K}")
        if not z.is_cuda:
            raise FlowtronB200Error("FlowtronLoss needs CUDA tensors")
        learned = ctx.needs_input_grad[2] or ctx.needs_input_grad[3]
        if mean.size(0) not in (1, B) or (learned and mean.size(0) != B):
            raise ValueError(f"mean / log_var must be [B, M, K], or [1, M, K] buffers without a gradient; got {tuple(mean.shape)}")
        per_row = mean.size(0) == B
        zc = z.detach().float().contiguous()
        mc, lc, pc = (t.detach().float().contiguous() for t in (mean, log_var, prob))
        lens = _lens_i32(out_lens, z.device)
        sums = torch.empty(2, device=z.device)
        _lib.gmm_nll_reduce(zc, lens, mc, lc, pc, per_row, sums)
        ctx.save = (zc, lens, mc, lc, pc, per_row, sums)
        ctx.learned = learned
        return sums[0] / (sums[1] * M)

    @staticmethod
    def backward(ctx, g):
        zc, lens, mc, lc, pc, per_row, sums = ctx.save
        gn = (g.reshape(1).float() / (sums[1] * zc.size(2))).contiguous()
        learned = ctx.learned
        dz, dprob = torch.empty_like(zc), torch.empty_like(pc)
        dmean = torch.empty_like(mc) if learned else None
        dlog_var = torch.empty_like(lc) if learned else None
        _lib.gmm_nll_grad(zc, lens, mc, lc, pc, per_row, gn, dz, dmean, dlog_var, dprob)
        return dz, None, dmean, dlog_var, dprob


class _AttnCtcFn(torch.autograd.Function):
    """Batched attention-CTC cost per utterance and its gradient in one launch (ft_attn_ctc_loss, csrc/ctc.cu)."""

    @staticmethod
    def forward(ctx, attn_logprob, in_lens, out_lens, time_reversed, blank_logprob):
        if not attn_logprob.is_cuda:
            raise FlowtronB200Error("AttentionCTCLoss needs CUDA tensors: the sm_90a kernel is the only implementation")
        lp = attn_logprob.detach().float().contiguous()
        dev = lp.device
        cost = torch.empty(lp.size(0), device=dev)
        dlp = torch.empty_like(lp)
        _lib.attn_ctc_loss(lp, _lens_i32(in_lens, dev), _lens_i32(out_lens, dev), time_reversed, blank_logprob, cost, dlp)
        ctx.save_for_backward(dlp)
        return cost

    @staticmethod
    def backward(ctx, g_cost):
        (dlp,) = ctx.saved_tensors
        return dlp * g_cost.reshape(-1, 1, 1), None, None, None, None


class AttentionCTCLoss(nn.Module):
    """flowtron.py:155-182.  Same constructor and call signature; the per-utterance Python loop (blank padding, slicing,
    log_softmax, nn.CTCLoss, `.item()` host syncs) is ONE kernel launch for the whole batch (SURVEY §8f row 4).
    ``time_reversed=True`` consumes an AR_Back_Step's attn_logprob in its flipped time directly, replacing the
    reference's in-place roll + flip (flowtron.py:250-256, 266-270)."""

    def __init__(self, blank_logprob=-1):
        super().__init__()
        self.log_softmax = nn.LogSoftmax(dim=3)
        self.blank_logprob = blank_logprob
        self.CTCLoss = nn.CTCLoss(zero_infinity=True)

    def forward(self, attn, in_lens, out_lens, attn_logprob, time_reversed=False):
        assert attn_logprob is not None
        lp = attn_logprob[:, 0] if attn_logprob.dim() == 4 else attn_logprob          # [B, 1, T, L] like the reference
        cost = _AttnCtcFn.apply(lp, in_lens, out_lens, bool(time_reversed), float(self.blank_logprob))
        return cost.sum() / lp.shape[0]


class FlowtronLoss(nn.Module):
    def __init__(self, sigma=1.0, gm_loss=False, gate_loss=True, use_ctc_loss=False, ctc_loss_weight=0.0, blank_logprob=-1):
        super().__init__()
        self.sigma = sigma
        self.gm_loss = gm_loss
        self.gate_loss = gate_loss
        self.use_ctc_loss = use_ctc_loss
        self.ctc_loss_weight = ctc_loss_weight
        self.blank_logprob = blank_logprob
        self.attention_loss = AttentionCTCLoss(blank_logprob=self.blank_logprob)

    def forward(self, model_output, gate_target, in_lengths, out_lengths, is_validation=False):
        z, log_s_list, gate_pred, attn_list, attn_logprob_list, mean, log_var, prob = model_output
        use_gate = self.gate_loss > 0 and gate_pred is not None
        if self.gm_loss:
            # sigma = inf turns the Gaussian term of ft_nll_reduce off: it then gives -sum log_s / (n M) and the gate loss
            # (z is passed detached, so its zero gradient is dropped); the mixture NLL replaces the Gaussian term
            loss, gate_loss = _NllGateFn.apply(math.inf, z.detach(), gate_pred if use_gate else None, gate_target, out_lengths,
                                               *log_s_list)
            loss = loss + _GmmNllFn.apply(z, out_lengths, mean, log_var, prob)
        else:
            loss, gate_loss = _NllGateFn.apply(self.sigma, z, gate_pred if use_gate else None, gate_target, out_lengths,
                                               *log_s_list)
        if not use_gate:
            gate_loss = torch.zeros(1, device=z.device)
        loss_ctc = torch.zeros_like(gate_loss)
        if self.use_ctc_loss:
            for cur_flow_idx, flow_attn in enumerate(attn_list):
                cur = attn_logprob_list[cur_flow_idx]
                # back steps return flipped time; the reference un-rolls / un-flips in place (flowtron.py:250-256) and
                # restores afterwards (:266-270) -- here the kernel indexes the flipped tensor directly
                loss_ctc = loss_ctc + self.attention_loss(flow_attn.unsqueeze(1), in_lengths, out_lengths,
                                                          attn_logprob=cur.unsqueeze(1),
                                                          time_reversed=(cur_flow_idx % 2 != 0))
            loss_ctc = loss_ctc / float(len(attn_list))
        return loss, gate_loss, loss_ctc
