"""WaveGlow vocoder, inference direction (tacotron2/waveglow/glow.py of the reference), on the sm_90a kernels of
csrc/waveglow.cu: log-mel [B, 80, F] -> audio [B, 256 F].

The module has the reference's attribute names and state_dict keys (weight-norm form by default, plain weights after
WaveGlow.remove_weightnorm), so `WaveGlow(**config["waveglow_config"]).load_state_dict(checkpoint_state_dict)` works with
either form.  Its parameters are packed once per weight version into the kernels' layouts (weight norm folded, fp16 GEMM
operands, tap-split and gate-interleaved in_layer / cond_layer rows, the upsample as a GEMM, fp32 inverses of convinv).
Only inference is built: forward (training) raises.
"""
from __future__ import annotations

from ctypes import c_int

import torch
import torch.nn.functional as F

from . import _lib
from ._lib import FlowtronB200Error


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
        n_half = n_group // 2
        c = n_group
        self.channels = []                                      # (n_remaining_channels, n_half) per flow
        for k in range(n_flows):
            if k % n_early_every == 0 and k > 0:
                n_half -= n_early_size // 2
                c -= n_early_size
            if c < 2:
                raise NotImplementedError("early outputs leave fewer than 2 channels")
            self.convinv.append(Invertible1x1Conv(c))
            self.WN.append(WN(n_half, n_mel_channels * n_group, **WN_config))
            self.channels.append((c, n_half))
        self.n_remaining_channels = c
        self._packed = None
        self._packed_key = None

    def forward(self, forward_input):
        raise NotImplementedError("WaveGlow training (forward / WaveGlowLoss) is not built; use infer()")

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
        M, L, C = self.n_mel_channels, self.WN_config["n_layers"], self.WN_config["n_channels"]
        keep = []

        def dev_t(t, dtype):
            t = t.to(device=dev, dtype=dtype).contiguous()
            keep.append(t)
            return t.data_ptr()

        w = _lib.FtWaveGlowWeights()
        # upsample: W[ci, c, t + 256 j] -> up_w[g*640 + c*8 + jj, j*96 + ci], t = 8 g + jj
        W = self.upsample.weight.detach().float().view(M, M, 4, 32, 8)            # [ci, c, j, g, jj]
        up = W.permute(3, 1, 4, 2, 0)                                                # [g, c, jj, j, ci]
        up = F.pad(up, (0, 96 - M)).reshape(32 * M * 8, 4 * 96)
        w.up_w = dev_t(up, torch.float16)
        w.up_b = dev_t(self.upsample.bias.detach().float().view(1, M, 1).expand(32, M, 8).reshape(-1), torch.float32)
        inter = torch.stack([torch.arange(C), torch.arange(C) + C], 1).reshape(-1)   # row 2c: tanh c, 2c+1: sigmoid c
        for k, wn in enumerate(self.WN):
            cond_w = _weight(wn.cond_layer)[:, :, 0]
            cond_b = wn.cond_layer.bias.detach().float()
            for i in range(L):
                wi = _weight(wn.in_layers[i])                                         # [2C, C, 3]
                sl = slice(2 * C * i, 2 * C * (i + 1))
                full = torch.cat([wi[:, :, 0], wi[:, :, 1], wi[:, :, 2], cond_w[sl]], 1)
                w.in_w[k][i] = dev_t(full[inter], torch.float16)
                w.in_b[k][i] = dev_t((wn.in_layers[i].bias.detach().float() + cond_b[sl])[inter], torch.float32)
                w.rs_w[k][i] = dev_t(_weight(wn.res_skip_layers[i])[:, :, 0], torch.float16)
                w.rs_b[k][i] = dev_t(wn.res_skip_layers[i].bias.detach().float(), torch.float32)
            w.start_w[k] = dev_t(_weight(wn.start)[:, :, 0], torch.float32)
            w.start_b[k] = dev_t(wn.start.bias.detach().float(), torch.float32)
            w.end_w[k] = dev_t(wn.end.weight.detach().float()[:, :, 0], torch.float32)
            w.end_b[k] = dev_t(wn.end.bias.detach().float(), torch.float32)
            inv = torch.linalg.inv(self.convinv[k].conv.weight.detach().double().squeeze(-1).cpu())
            w.inv_w[k] = dev_t(inv.float(), torch.float32)
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
        generator in the reference's order.  lengths: optional host sequence of per-row frame counts; row b is then the
        B=1 result on spect[b, :, :lengths[b]] and zero after 256 lengths[b] samples."""
        if spect.dim() != 3 or spect.shape[1] != self.n_mel_channels:
            raise ValueError(f"spect must be [B, {self.n_mel_channels}, F], got {tuple(spect.shape)}")
        B, _, Fr = spect.shape
        Tg = 32 * Fr
        if lengths is None:
            frames = [Fr] * B
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
        fr = (c_int * B)(*frames)
        desc = _lib.FtWaveGlowDesc(n_mel=self.n_mel_channels, n_flows=self.n_flows, n_group=self.n_group,
                                   n_early_every=self.n_early_every, n_early_size=self.n_early_size,
                                   n_layers=self.WN_config["n_layers"], n_channels=self.WN_config["n_channels"],
                                   kernel_size=self.WN_config["kernel_size"], B=B, F_max=Fr, frames=fr)
        _lib.waveglow_infer(desc, w, mel, noise, float(sigma), audio)
        return audio


def waveglow_flops(frames: int, cfg) -> float:
    """Model FLOPs of one infer over `frames` mel frames: per group row per flow 2(3C+640)2C L + 2 C 2C (L-1) + 2 C C
    (last res_skip) + 2 n_half C (start) + 2 C 2 n_half (end), 32 group rows per frame, plus the upsample 2 * 320 * 20480
    per frame."""
    C, L = cfg["WN_config"]["n_channels"], cfg["WN_config"]["n_layers"]
    from .synth import waveglow_channels
    per_group = 0.0
    for c, nh in waveglow_channels(cfg):
        per_group += 2 * (3 * C + 640) * 2 * C * L + 2 * C * 2 * C * (L - 1) + 2 * C * C + 2 * nh * C + 2 * C * 2 * nh
    return frames * (32 * per_group + 2 * 320 * 20480)
