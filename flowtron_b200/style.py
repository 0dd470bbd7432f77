"""Style transfer by posterior sampling (the reference's inference_style_transfer.ipynb) on the sm_90a kernels.

The whole chain, for K reference utterances of the style to transfer::

    mels = stft.mel_spectrogram_ragged(wavs)                  # TacotronSTFT: one [80, F_k] log-mel per reference recording
    # pad the mels into mel [K, 80, T] and the texts into text [K, L]; out_lens / in_lens hold the true lengths
    z = model.encode(mel, speaker_ids, text, in_lens, out_lens)          # [K, 80, T], zero past out_lens
    mu = posterior_mean(z, out_lens, n_frames, lambd=1e-4, aggregation='batch')   # [1, 80, n_frames]
    residual = mu + sigma * torch.randn(1, 80, n_frames, device=mu.device)        # sampling stays with the caller
    mel_out, _ = model.infer(residual, speaker_id, new_text)   # or infer_batch with mu broadcast over the rows
    audio = waveglow.infer(mel_out, sigma=0.75)
    audio = denoiser(audio, 0.01)

With ``aggregation='time_and_batch'`` the mean is ``[1, 80, 1]`` and broadcasts over the residual's frames
(``mu + sigma * torch.randn(1, 80, n_frames)``).
"""
from __future__ import annotations

import math

import torch
from torch import Tensor

from . import _lib
from ._lib import FlowtronB200Error

_MODES = {"batch": _lib.POSTERIOR_BATCH, "time_and_batch": _lib.POSTERIOR_TIME_AND_BATCH}


def posterior_mean(z: Tensor, out_lens, n_frames: int, lambd: float = 1e-4, aggregation: str = "batch") -> Tensor:
    """Posterior mean of the reference z values, shrunk towards the prior's zero mean.

    z [K, 80, T] f32 CUDA (``Flowtron.encode``'s output; any [K, M, T] tensor with M <= 128), out_lens [K]: the valid frames
    of each row.  With ratio = K / lambd and scale = ratio / (ratio + 1):

    * ``'batch'``: each row's first out_lens[k] frames are repeated in time until they cover n_frames and cut there, the K
      rows are averaged frame by frame, and the mean is multiplied by scale -> [1, 80, n_frames];
    * ``'time_and_batch'``: each row is averaged over its own frames, then over the K, times scale -> [1, 80, 1].

    One kernel launch (``ft_posterior_mean``), no host synchronisation when out_lens is a CUDA tensor (trusted, as
    ``Flowtron.encode`` trusts it); lengths given on the host must lie in [1, T].  A non-positive lambd, an unknown
    aggregation and n_frames < 1 raise ValueError, CPU tensors FlowtronB200Error."""
    if aggregation not in _MODES:
        raise ValueError(f"aggregation must be one of {sorted(_MODES)}, got {aggregation!r}")
    lambd = float(lambd)
    if not (lambd > 0.0 and math.isfinite(lambd)):
        raise ValueError(f"lambd must be a positive number, got {lambd}")
    if isinstance(n_frames, bool) or int(n_frames) != n_frames or n_frames < 1:
        raise ValueError(f"n_frames must be a positive integer, got {n_frames}")
    n_frames = int(n_frames)
    if z.dim() != 3:
        raise ValueError(f"z must be [K, n_mel, T], got shape {tuple(z.shape)}")
    K, M, T = z.shape
    if K < 1 or T < 1:
        raise ValueError(f"z is empty: {tuple(z.shape)}")
    if M > 128:
        raise ValueError(f"the posterior-mean kernel takes at most 128 mel channels, got {M}")
    out_lens = _lib.ragged_lengths(out_lens, K, T, "out_lens")
    if not z.is_cuda:
        raise FlowtronB200Error("posterior_mean needs CUDA tensors: the sm_90a kernel is the only implementation")
    dev = z.device
    ratio = K / lambd
    scale = ratio / (ratio + 1.0)
    zt = z.permute(2, 0, 1)                 # [T, K, M]: Flowtron.encode's storage order, so no copy for its output
    zt = zt.float().contiguous()
    lens = out_lens.to(device=dev, dtype=torch.int32).contiguous()
    mode = _MODES[aggregation]
    if mode == _lib.POSTERIOR_BATCH:
        out = torch.empty(1, M, n_frames, dtype=torch.float32, device=dev)
    else:
        out = torch.empty(1, M, 1, dtype=torch.float32, device=dev)
    _lib.posterior_mean(zt, lens, n_frames, mode, scale, out)
    return out
