"""WaveGlow vocoder, inference direction (tacotron2/waveglow/glow.py of the reference), on the sm_90a kernels of
csrc/waveglow.cu: log-mel [B, 80, F] -> audio [B, 256 F].

The module has the reference's attribute names and state_dict keys (weight-norm form by default, plain weights after
WaveGlow.remove_weightnorm), so `WaveGlow(**config["waveglow_config"]).load_state_dict(checkpoint_state_dict)` works with
either form.  For infer, its parameters are packed once per weight version into the kernels' layouts (weight norm folded, fp16 GEMM
operands, tap-split and gate-interleaved in_layer / cond_layer rows, the upsample as a GEMM, fp32 inverses of convinv).
forward (training, the z direction) packs the same layouts with differentiable device ops on every call, so the kernels'
gradients of the packed weights reach upsample, WN and convinv parameters (weight_g / weight_v in weight-norm form) through
torch autograd; see DESIGN.md §4.21.
"""
from __future__ import annotations

from ctypes import c_int

import torch
import torch.nn.functional as F

from . import _lib
from ._lib import FlowtronB200Error
from .synth import waveglow_channels


class Invertible1x1Conv(torch.nn.Module):
    def __init__(self, c):
        super().__init__()
        self.conv = torch.nn.Conv1d(c, c, kernel_size=1, stride=1, padding=0, bias=False)
        W = torch.linalg.qr(torch.randn(c, c))[0]             # random orthonormal, det +1 (glow.py:64-73)
        if torch.det(W) < 0:
            W[:, 0] = -W[:, 0]
        self.conv.weight.data = W.view(c, c, 1)


def _wn(conv):
    return torch.nn.utils.weight_norm(conv, name="weight")


class WN(torch.nn.Module):
    def __init__(self, n_in_channels, n_mel_channels, n_layers, n_channels, kernel_size):
        super().__init__()
        self.n_layers = n_layers
        self.n_channels = n_channels
        self.in_layers = torch.nn.ModuleList()
        self.res_skip_layers = torch.nn.ModuleList()
        self.start = _wn(torch.nn.Conv1d(n_in_channels, n_channels, 1))
        self.end = torch.nn.Conv1d(n_channels, 2 * n_in_channels, 1)
        self.end.weight.data.zero_()
        self.end.bias.data.zero_()
        self.cond_layer = _wn(torch.nn.Conv1d(n_mel_channels, 2 * n_channels * n_layers, 1))
        for i in range(n_layers):
            d = 2 ** i
            self.in_layers.append(_wn(torch.nn.Conv1d(n_channels, 2 * n_channels, kernel_size, dilation=d, padding=d)))
            rs = 2 * n_channels if i < n_layers - 1 else n_channels
            self.res_skip_layers.append(_wn(torch.nn.Conv1d(n_channels, rs, 1)))


def _weight(conv) -> torch.Tensor:
    """Effective weight: g * v / |v| (norm over all dims but 0) for a weight-normed conv, else its weight.  The fold runs
    on the host with the op torch.nn.utils.remove_weight_norm uses, so both forms of one checkpoint pack bit-identically."""
    if hasattr(conv, "weight_g"):
        return torch._weight_norm(conv.weight_v.detach().float().cpu(), conv.weight_g.detach().float().cpu(), 0)
    return conv.weight.detach().float()


def _effective_weight(conv) -> torch.Tensor:
    """_weight's fold as a differentiable device op (gradients reach weight_g and weight_v)."""
    if hasattr(conv, "weight_g"):
        return torch._weight_norm(conv.weight_v, conv.weight_g, 0)
    return conv.weight


_WG_MAX_BATCH = 128              # WG_MAX_B of csrc/waveglow.cu


class WaveGlowNoCpuPath(FlowtronB200Error, NotImplementedError):
    """WaveGlow.forward on CPU tensors or a CPU module: the sm_90a kernels are the only implementation, so training on the
    CPU is not implemented.  A FlowtronB200Error like every device-placement error of the library, and a
    NotImplementedError, as forward has raised on the CPU since before training was built."""


class WaveGlowLoss(torch.nn.Module):
    """glow.py:43-58: sum(z^2) / (2 sigma^2) - sum(log_s) - sum(log_det_W), over the number of elements of z."""

    def __init__(self, sigma=1.0):
        super().__init__()
        self.sigma = sigma

    def forward(self, model_output):
        z, log_s_list, log_det_W_list = model_output
        log_s_total = sum(torch.sum(log_s) for log_s in log_s_list)
        log_det_W_total = sum(log_det_W_list)
        loss = torch.sum(z * z) / (2 * self.sigma * self.sigma) - log_s_total - log_det_W_total
        return loss / (z.size(0) * z.size(1) * z.size(2))


_FP16_FIELDS = ("up_w", "in_w", "rs_w")     # the GEMM operands; every other packed field is fp32


def _set_field(struct, key, value):
    """struct.name[k][i]... = value for key (name, k, i, ...)."""
    name, *idx = key
    if not idx:
        setattr(struct, name, value)
        return
    arr = getattr(struct, name)
    for j in idx[:-1]:
        arr = arr[j]
    arr[idx[-1]] = value


def _train_kernel_weights(packed):
    """The tensors ft_waveglow_train_fwd / _bwd read, by FtWaveGlowTrainWeights field: the packed weights in fp16 (GEMM
    operands) or fp32, plus the backward's transposed fp16 copies in_wT (the three dilated taps of in_w) and rs_wT."""
    out = {}
    for key, t in packed.items():
        t = t.detach()
        out[key] = t.to(torch.float16 if key[0] in _FP16_FIELDS else torch.float32).contiguous()
        if key[0] == "in_w":
            taps = t[:, :768].reshape(512, 3, 256).permute(2, 1, 0).reshape(256, 1536)
            out[("in_wT",) + key[1:]] = taps.to(torch.float16).contiguous()
        elif key[0] == "rs_w":
            out[("rs_wT",) + key[1:]] = t.t().to(torch.float16).contiguous()
    return out


class _WaveGlowTrainFn(torch.autograd.Function):
    """ft_waveglow_train_fwd / ft_waveglow_train_bwd on the fp32 packed weights (keys: their FtWaveGlowTrainWeights
    fields, as WaveGlow._layout names them): the kernels read fp16 copies (and the backward's transposed ones), made here
    on the device; the gradients come back for the fp32 packed tensors."""

    @staticmethod
    def forward(ctx, cfg, keys, spect, audio, *packed):
        n_flows, n_early_every, n_early_size, L, B, Fr, N = cfg
        Tn = N // 8
        desc = _lib.FtWaveGlowTrainDesc(n_mel=80, n_flows=n_flows, n_group=8, n_early_every=n_early_every,
                                        n_early_size=n_early_size, n_layers=L, n_channels=256, kernel_size=3, B=B, F=Fr, N=N)
        kernel = _train_kernel_weights(dict(zip(keys, packed)))
        w = _lib.FtWaveGlowTrainWeights()
        for key, t in kernel.items():
            _set_field(w, key, t.data_ptr())
        dev = spect.device
        z = torch.empty(B, 8, Tn, device=dev)
        log_s = [torch.empty(B, t.shape[0] // 2, Tn, device=dev) for key, t in zip(keys, packed) if key[0] == "conv_w"]
        saved = torch.empty(_lib.waveglow_train_saved_bytes(desc), dtype=torch.uint8, device=dev)
        _lib.waveglow_train_fwd(desc, w, spect, audio, z, log_s, saved)
        ctx.state = (desc, w, kernel, saved, keys, [t.shape for t in packed])
        ctx.set_materialize_grads(False)
        return (z, *log_s)

    @staticmethod
    def backward(ctx, d_z, *d_log_s):
        desc, w, _kernel, saved, keys, shapes = ctx.state
        dev = saved.device
        g = _lib.FtWaveGlowTrainGrads()
        grads = []
        for key, shape in zip(keys, shapes):
            if key[0] == "in_w":        # per tap (split-K needs each output contiguous), concatenated afterwards
                parts = [torch.empty(512, 256, device=dev) for _ in range(3)] + [torch.empty(512, 640, device=dev)]
                for t, part in enumerate(parts):
                    _set_field(g, key + (t,), part.data_ptr())
                grads.append(parts)
            else:
                grads.append(torch.empty(shape, dtype=torch.float32, device=dev))
                _set_field(g, key, grads[-1].data_ptr())
        dz = None if d_z is None else d_z.float().contiguous()
        dls = [None if t is None else t.float().contiguous() for t in d_log_s]
        _lib.waveglow_train_bwd(desc, w, dz, dls, saved, g)
        ctx.state = None
        return (None, None, None, None, *[torch.cat(t, 1) if isinstance(t, list) else t for t in grads])


class WaveGlow(torch.nn.Module):
    def __init__(self, n_mel_channels, n_flows, n_group, n_early_every, n_early_size, WN_config):
        super().__init__()
        C, K, L = WN_config["n_channels"], WN_config["kernel_size"], WN_config["n_layers"]
        if n_group != 8 or K != 3 or C != 256 or n_mel_channels != 80:
            raise NotImplementedError("the sm_90a WaveGlow kernels are built for n_mel_channels 80, n_group 8, n_channels 256, "
                                      "kernel_size 3 (the shipped waveglow config)")
        if not (1 <= n_flows <= _lib.WG_MAX_FLOWS and 1 <= L <= _lib.WG_MAX_LAYERS) or n_early_size % 2 or n_early_every < 1:
            raise NotImplementedError("n_flows <= 16, n_layers <= 8 (dilation <= 128) and an even n_early_size are built")
        self.upsample = torch.nn.ConvTranspose1d(n_mel_channels, n_mel_channels, 1024, stride=256)
        self.n_flows = n_flows
        self.n_group = n_group
        self.n_early_every = n_early_every
        self.n_early_size = n_early_size
        self.n_mel_channels = n_mel_channels
        self.WN_config = dict(WN_config)
        self.WN = torch.nn.ModuleList()
        self.convinv = torch.nn.ModuleList()
        self.channels = waveglow_channels(dict(n_group=n_group, n_flows=n_flows, n_early_every=n_early_every,
                                               n_early_size=n_early_size))      # (n_remaining_channels, n_half) per flow
        if self.channels[-1][0] < 2:
            raise NotImplementedError("early outputs leave fewer than 2 channels")
        for c, n_half in self.channels:
            self.convinv.append(Invertible1x1Conv(c))
            self.WN.append(WN(n_half, n_mel_channels * n_group, **WN_config))
        self.n_remaining_channels = self.channels[-1][0]
        self._packed = None
        self._packed_key = None

    def forward(self, forward_input):
        """(spect [B, 80, F], audio [B, N]) -> (z [B, 8, N/8], log_s_list, log_det_W_list), as glow.py:196-245: z in the
        reference's channel order (early outputs first), log_s_list[k] [B, n_half_k, N/8], log_det_W_list[k] the scalar
        B (N/8) logdet(W_k).  N is a multiple of 8 and at most 256 F (every Mel2Samp segment).  Differentiable in every
        parameter; spect and audio are data and take no gradient."""
        spect, audio = forward_input
        if spect.dim() != 3 or spect.shape[1] != self.n_mel_channels:
            raise ValueError(f"spect must be [B, {self.n_mel_channels}, F], got {tuple(spect.shape)}")
        if audio.dim() != 2 or audio.shape[0] != spect.shape[0]:
            raise ValueError(f"audio must be [B, N] with the B of spect ({spect.shape[0]}), got {tuple(audio.shape)}")
        B, _, Fr = spect.shape
        N = audio.shape[1]
        if not 1 <= B <= _WG_MAX_BATCH:
            raise ValueError(f"batch must be 1..{_WG_MAX_BATCH}, got {B}")
        if N < self.n_group or N % self.n_group:
            raise ValueError(f"audio length N = {N} must be a positive multiple of n_group = {self.n_group}")
        if N > 256 * Fr:
            raise ValueError(f"audio length N = {N} exceeds the 256 F = {256 * Fr} samples the spectrogram covers")
        if spect.requires_grad or audio.requires_grad:
            raise ValueError("WaveGlow.forward computes no gradient for spect or audio: pass them without requires_grad")
        if not spect.is_cuda or not audio.is_cuda or not self.upsample.weight.is_cuda:
            raise WaveGlowNoCpuPath("WaveGlow.forward needs the module, spect and audio on CUDA: the sm_90a kernels are the "
                                    "only implementation")
        cfg = (self.n_flows, self.n_early_every, self.n_early_size, self.WN_config["n_layers"], B, Fr, N)
        packed = self._train_params()
        outs = _WaveGlowTrainFn.apply(cfg, tuple(packed), spect.float().contiguous(), audio.float().contiguous(),
                                      *packed.values())
        Tn = N // self.n_group
        log_det_W_list = [B * Tn * torch.logdet(inv.conv.weight.squeeze(-1)) for inv in self.convinv]
        return outs[0], list(outs[1:]), log_det_W_list

    def _layout(self, fold):
        """The kernels' packed weights in fp32, keyed by FtWaveGlowTrainWeights field: (name,), (name, flow) or (name, flow,
        layer), in the order up_w, up_b, then per flow conv_w, start_w, start_b, end_w, end_b and per layer in_w, in_b,
        rs_w, rs_b.  fold(conv) is a conv's effective weight (its weight-norm fold).  up_w is the ConvTranspose1d as one GEMM
        over frames f-3..f; in_w = [tap0 | tap1 | tap2 | cond_layer slice] and in_b = in_layer + cond bias have their rows
        interleaved (2c: tanh input of channel c, 2c+1: its sigmoid input)."""
        M, L, C = self.n_mel_channels, self.WN_config["n_layers"], self.WN_config["n_channels"]

        def gate_rows(x):
            return x.reshape(2, C, -1).transpose(0, 1).reshape(x.shape)

        # upsample: W[ci, c, t + 256 j] -> up_w[g*640 + c*8 + jj, j*96 + ci], t = 8 g + jj
        up = self.upsample.weight.float().view(M, M, 4, 32, 8).permute(3, 1, 4, 2, 0)      # [g, c, jj, j, ci]
        out = {("up_w",): F.pad(up, (0, 96 - M)).reshape(32 * M * 8, 4 * 96),
               ("up_b",): self.upsample.bias.float().view(1, M, 1).expand(32, M, 8).reshape(-1)}
        for k, wn in enumerate(self.WN):
            cond_w, cond_b = fold(wn.cond_layer)[:, :, 0], wn.cond_layer.bias.float()
            out[("conv_w", k)] = self.convinv[k].conv.weight.float()[:, :, 0]
            out[("start_w", k)] = fold(wn.start)[:, :, 0]
            out[("start_b", k)] = wn.start.bias.float()
            out[("end_w", k)] = wn.end.weight.float()[:, :, 0]
            out[("end_b", k)] = wn.end.bias.float()
            for i in range(L):
                wi, sl = fold(wn.in_layers[i]), slice(2 * C * i, 2 * C * (i + 1))
                out[("in_w", k, i)] = gate_rows(torch.cat([wi[:, :, 0], wi[:, :, 1], wi[:, :, 2], cond_w[sl]], 1))
                out[("in_b", k, i)] = gate_rows(wn.in_layers[i].bias.float() + cond_b[sl])
                out[("rs_w", k, i)] = fold(wn.res_skip_layers[i])[:, :, 0]
                out[("rs_b", k, i)] = wn.res_skip_layers[i].bias.float()
        return out

    def _train_params(self):
        """_layout with the differentiable device fold: the packed weights _WaveGlowTrainFn takes, through which torch
        autograd reaches the parameters."""
        return self._layout(_effective_weight)

    @staticmethod
    def remove_weightnorm(model):
        for wn in model.WN:
            wn.start = torch.nn.utils.remove_weight_norm(wn.start)
            wn.in_layers = torch.nn.ModuleList(torch.nn.utils.remove_weight_norm(c) for c in wn.in_layers)
            wn.cond_layer = torch.nn.utils.remove_weight_norm(wn.cond_layer)
            wn.res_skip_layers = torch.nn.ModuleList(torch.nn.utils.remove_weight_norm(c) for c in wn.res_skip_layers)
        model._packed = None
        return model

    # -------------------------------------------------------------------------------------------- packing
    def _weights_key(self):
        return tuple((t.data_ptr(), t._version, t.device) for t in self.state_dict(keep_vars=True).values())

    @torch.no_grad()
    def _pack(self):
        key = self._weights_key()
        if self._packed is not None and self._packed_key == key:
            return self._packed
        dev = self.upsample.weight.device
        w = _lib.FtWaveGlowWeights()
        keep = []

        def put(field, t, dtype):
            keep.append(t.to(device=dev, dtype=dtype).contiguous())
            _set_field(w, field, keep[-1].data_ptr())

        for field, t in self._layout(_weight).items():
            if field[0] != "conv_w":
                put(field, t, torch.float16 if field[0] in _FP16_FIELDS else torch.float32)
        for k, inv in enumerate(self.convinv):
            put(("inv_w", k), torch.linalg.inv(inv.conv.weight.detach().double().squeeze(-1).cpu()).float(), torch.float32)
        self._packed = (w, keep)
        self._packed_key = key
        return self._packed

    def draw_noise(self, B, Tg, device):
        """The noise infer() draws when none is given, in the reference's order and shapes (the first flow's channels, then
        each early injection), on the current CUDA generator, arranged in the `noise` layout [B, 8, Tg]."""
        noise = torch.zeros(B, self.n_group, Tg, device=device)
        c = self.channels[-1][0]
        noise[:, self.n_group - c:] = torch.randn(B, c, Tg, device=device)
        for k in reversed(range(self.n_flows)):
            if k % self.n_early_every == 0 and k > 0:
                ck, e = self.channels[k][0], self.n_early_size
                noise[:, self.n_group - ck - e: self.n_group - ck] = torch.randn(B, e, Tg, device=device)
        return noise

    @torch.no_grad()
    def infer(self, spect, sigma=1.0, *, noise=None, lengths=None):
        """spect [B, 80, F] log-mel -> audio [B, 256 F] (WaveGlow.infer, glow.py:251-293).
        noise: optional [B, 8, 32 F] in the channel order of WaveGlow.forward's z (for the shipped config: 0:2 injected
        after flow 4, 2:4 after flow 8, 4:8 the initial draw), multiplied by sigma; None draws it on the current CUDA
        generator in the reference's order.  lengths: optional per-row frame counts; row b is then the B=1 result on
        spect[b, :, :lengths[b]] and zero after 256 lengths[b] samples.  A host sequence or CPU tensor is range-checked
        (ValueError unless every count is in 1..F).  A CUDA tensor (int32 or int64, shape [B], e.g. infer_batch's
        mel_lens) is used in place with no host synchronisation, so the call can be captured in a CUDA graph and replayed
        with new lengths; only its shape and dtype are checked, and a count outside 1..F gives an unspecified row (it is
        clamped, never read past the inputs)."""
        if spect.dim() != 3 or spect.shape[1] != self.n_mel_channels:
            raise ValueError(f"spect must be [B, {self.n_mel_channels}, F], got {tuple(spect.shape)}")
        B, _, Fr = spect.shape
        Tg = 32 * Fr
        frames_dev = None
        if lengths is None:
            frames = [Fr] * B
        elif torch.is_tensor(lengths) and lengths.is_cuda:
            if tuple(lengths.shape) != (B,) or lengths.dtype not in (torch.int32, torch.int64):
                raise ValueError(f"CUDA lengths must be int32 or int64 of shape ({B},), got {lengths.dtype} "
                                 f"{tuple(lengths.shape)}")
            if lengths.device != spect.device:
                raise ValueError(f"lengths are on {lengths.device}, spect on {spect.device}")
            frames, frames_dev = None, lengths.to(torch.int32).contiguous()
        else:
            frames = [int(n) for n in (lengths.tolist() if torch.is_tensor(lengths) else lengths)]
            if len(frames) != B or any(n < 1 or n > Fr for n in frames):
                raise ValueError(f"lengths must hold {B} frame counts in 1..{Fr}, got {frames}")
        if noise is not None and tuple(noise.shape) != (B, self.n_group, Tg):
            raise ValueError(f"noise must be [B, {self.n_group}, 32 F] = {(B, self.n_group, Tg)}, got {tuple(noise.shape)}")
        if not spect.is_cuda or not self.upsample.weight.is_cuda or (noise is not None and not noise.is_cuda):
            raise FlowtronB200Error("WaveGlow.infer needs the module, spect and noise on CUDA: the sm_90a kernels are the only "
                                    "implementation")
        if noise is None:
            noise = self.draw_noise(B, Tg, spect.device)
        w, _keep = self._pack()
        mel = spect.detach().float().contiguous()
        noise = noise.detach().float().contiguous()
        audio = torch.empty(B, 256 * Fr, device=spect.device, dtype=torch.float32)
        fr = None if frames is None else (c_int * B)(*frames)
        desc = _lib.FtWaveGlowDesc(n_mel=self.n_mel_channels, n_flows=self.n_flows, n_group=self.n_group,
                                   n_early_every=self.n_early_every, n_early_size=self.n_early_size,
                                   n_layers=self.WN_config["n_layers"], n_channels=self.WN_config["n_channels"],
                                   kernel_size=self.WN_config["kernel_size"], B=B, F_max=Fr, frames=fr)
        _lib.waveglow_infer(desc, w, mel, noise, float(sigma), audio, frames_dev)
        return audio


def waveglow_flops(frames: int, cfg) -> float:
    """Model FLOPs of one infer over `frames` mel frames: per group row per flow 2(3C+640)2C L + 2 C 2C (L-1) + 2 C C
    (last res_skip) + 2 n_half C (start) + 2 C 2 n_half (end), 32 group rows per frame, plus the upsample 2 * 320 * 20480
    per frame."""
    C, L = cfg["WN_config"]["n_channels"], cfg["WN_config"]["n_layers"]
    per_group = 0.0
    for c, nh in waveglow_channels(cfg):
        per_group += 2 * (3 * C + 640) * 2 * C * L + 2 * C * 2 * C * (L - 1) + 2 * C * C + 2 * nh * C + 2 * C * 2 * nh
    return frames * (32 * per_group + 2 * 320 * 20480)
