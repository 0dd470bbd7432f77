"""CPU restatement of STFT.inverse and the WaveGlow Denoiser (TEST INFRASTRUCTURE), built on the fp32 transform
restatement of oracle/stft_oracle.py.

STFT.inverse (audio_processing.py:237-265) convolves with the inverse basis pinv(scale * fourier_basis) * window, which is
irfft(.) * window / scale, and its final ``* filter_length / hop`` cancels that scale; irfft ignores the imaginary parts
of the DC and Nyquist bins, as the pinv basis does.  So the inverse restated here in fp64 is irfft, window, overlap-add,
division by window_sumsquare (:7-56) where it exceeds float32's tiny, and 512 samples trimmed at each end.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle.stft_oracle import hann_periodic, pad_center, stft_transform


def stft_inverse(magnitude, phase, filter_length=1024, hop_length=256, win_length=1024) -> torch.Tensor:
    """[B, N/2+1, F] magnitude and phase -> fp64 [B, 1, (F-1)*hop]."""
    m = np.asarray(magnitude, dtype=np.float64)
    p = np.asarray(phase, dtype=np.float64)
    B, _, n_frames = m.shape
    frames = np.fft.irfft(m * np.exp(1j * p), n=filter_length, axis=1)               # [B, N, F]
    w = torch.from_numpy(pad_center(hann_periodic(win_length), filter_length)).float().double().numpy()
    frames = frames * w[None, :, None]
    n = filter_length + hop_length * (n_frames - 1)
    out = np.zeros((B, n))
    env = np.zeros(n)
    for i in range(n_frames):
        out[:, i * hop_length: i * hop_length + filter_length] += frames[:, :, i]
        env[i * hop_length: i * hop_length + filter_length] += w * w
    nz = env > np.finfo(np.float32).tiny
    out[:, nz] /= env[nz]
    half = filter_length // 2
    return torch.from_numpy(out[:, None, half: n - half])


def denoise(audio: torch.Tensor, bias_spec, strength: float, filter_length=1024, hop_length=256, win_length=1024):
    """Denoiser.forward (tacotron2/waveglow/denoiser.py): the fp32 transform restatement, magnitude
    max(m - bias_spec * strength, 0), then the fp64 inverse.  audio [B, N] -> [B, 1, (N // hop) * hop]."""
    mag, phase = stft_transform(audio.float(), filter_length, hop_length, win_length)
    bias = torch.as_tensor(np.asarray(bias_spec, dtype=np.float32)).reshape(1, -1, 1)
    mag = torch.clamp(mag - bias * strength, 0.0)
    return stft_inverse(mag, phase, filter_length, hop_length, win_length)
