"""WaveGlow Denoiser (tacotron2/waveglow/denoiser.py of the reference): removes the constant hiss a WaveGlow model adds by
subtracting the magnitude spectrum of its output on a silent mel ("bias") from every frame of the audio's spectrum.

The state_dict is the reference's (``bias_spec`` [1, 513, 1], ``stft.forward_basis`` / ``stft.inverse_basis``), so a
reference Denoiser's state loads strictly.  ``forward`` is two kernels: ft_stft_transform, then ft_stft_inverse with the
bias subtraction and the clamp folded into its spectrum load (csrc/istft.cu).
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib
from ._lib import FlowtronB200Error
from .audio_processing import STFT, aligned_waveform


class Denoiser(torch.nn.Module):
    """Removes model bias from audio produced with WaveGlow."""

    def __init__(self, waveglow, filter_length=1024, n_overlap=4, win_length=1024, mode='zeros'):
        super().__init__()
        dev, dtype = waveglow.upsample.weight.device, waveglow.upsample.weight.dtype
        self.stft = STFT(filter_length=filter_length, hop_length=int(filter_length / n_overlap),
                         win_length=win_length).to(dev)
        if mode == 'zeros':
            mel_input = torch.zeros((1, 80, 88), dtype=dtype, device=dev)
        elif mode == 'normal':
            mel_input = torch.randn((1, 80, 88), dtype=dtype, device=dev)
        else:
            raise ValueError("Mode {} if not supported".format(mode))
        with torch.no_grad():
            bias_audio = waveglow.infer(mel_input, sigma=0.0).float()
            bias_spec, _ = self.stft.transform(bias_audio)
        self.register_buffer('bias_spec', bias_spec[:, :, :1].contiguous())

    def forward(self, audio, strength=0.1, *, lengths=None):
        """audio [B, N] -> [B, 1, (N // hop) * hop], denoised as the reference does: magnitude max(m - strength * bias, 0),
        phase kept.  lengths: optional per-row sample counts (e.g. 256 * frames from WaveGlow.infer(lengths=)); row b is
        then the B = 1 result on audio[b, :lengths[b]] and zero after (lengths[b] // hop) * hop samples.

        Short rows: the reflect padding needs more than n_fft / 2 samples, so a B = 1 call on at most n_fft / 2 samples
        raises ValueError, and so do host lengths (a sequence or CPU tensor) with such a row or a count above N.  A CUDA
        tensor of lengths (int32 or int64, shape [B]) is planned on the device with no host synchronisation, so the call
        can be captured in a CUDA graph and replayed with new lengths; only its shape and dtype are checked, a row of at
        most n_fft / 2 samples (fewer than 3 WaveGlow frames) comes out all zero, and counts above N are taken as N."""
        stft = self.stft
        n_fft, hop = stft.filter_length, stft.hop_length
        if n_fft != 1024 or hop not in _lib.STFT_INVERSE_HOPS:
            raise NotImplementedError("the Denoiser is built for filter_length 1024 and n_overlap 2, 4 or 8")
        if audio.dim() != 2:
            raise ValueError(f"audio must be [B, N], got {tuple(audio.shape)}")
        audio = audio.to(self.bias_spec.device).detach().float()     # the reference's audio.cuda().float()
        if not audio.is_cuda:
            raise FlowtronB200Error("Denoiser needs CUDA tensors: the sm_90a kernels are the only implementation")
        B, N = audio.shape
        dev = audio.device
        n_out = (N // hop) * hop
        if lengths is None:
            if N <= n_fft // 2:
                raise ValueError("audio shorter than the reflect padding")
            flat = audio.contiguous()
            F = 1 + N // hop
            so = torch.arange(B + 1, device=dev, dtype=torch.int64) * N
            fo = torch.arange(B + 1, device=dev, dtype=torch.int64) * F
            total = B * F
            out = torch.empty(B, 1, n_out, device=dev)
        else:
            if torch.is_tensor(lengths) and lengths.is_cuda:
                if tuple(lengths.shape) != (B,) or lengths.dtype not in (torch.int32, torch.int64):
                    raise ValueError(f"CUDA lengths must be int32 or int64 of shape ({B},), got {lengths.dtype} "
                                     f"{tuple(lengths.shape)}")
                if lengths.device != dev:
                    raise ValueError(f"lengths are on {lengths.device}, audio on {dev}")
                lens_d = lengths.to(torch.int64).contiguous()
                n_samples, total = B * N, B * (1 + N // hop)         # bounds: the true totals are planned on the device
            else:
                lens = np.asarray([int(n) for n in (lengths.tolist() if torch.is_tensor(lengths) else lengths)], dtype=np.int64)
                if len(lens) != B or lens.min() <= n_fft // 2 or lens.max() > N:
                    raise ValueError(f"lengths must hold {B} sample counts in {n_fft // 2 + 1}..{N}, got {lens.tolist()}")
                lens_d = torch.from_numpy(lens).to(dev, non_blocking=True)
                n_samples, total = int(lens.sum()), int((1 + lens // hop).sum())
            flat = torch.empty(n_samples, device=dev)
            so = torch.empty(B + 1, device=dev, dtype=torch.int64)
            fo = torch.empty_like(so)
            _lib.stft_pack_rows(audio.contiguous(), lens_d, n_fft, hop, flat, so, fo)
            out = torch.zeros(B, 1, n_out, device=dev)
        flat = aligned_waveform(flat)
        oo = torch.arange(B, device=dev, dtype=torch.int64) * n_out
        mag = torch.empty(total * (n_fft // 2 + 1), device=dev)
        phase = torch.empty_like(mag)
        _lib.stft_transform(flat, so, fo, B, total, stft._window, n_fft, hop, mag, phase)
        _lib.stft_inverse(mag, phase, fo, oo, B, total, stft._window, n_fft, hop, out,
                          bias=self.bias_spec.detach().float().reshape(-1).contiguous(), strength=float(strength))
        return out
