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

A model trained with the Gaussian-mixture prior (n_components > 1, FlowtronLoss(gm_loss=True)) maps mels to its mixture,
not to N(0, I), so its residual is drawn from that mixture::

    mean, log_var, prob = model.mixture(ref_mel, ref_lens)            # per-utterance mixtures of reference mels
    z = sample_mixture(mean, log_var, prob, n_frames, T, sigma=0.8)  # [B, 80, T], zero past n_frames
    mel_out, mel_lens, _ = model.infer_batch(z, speaker_ids, text, in_lens, max_frames=n_frames)

``prob`` may also be written by hand (one-hot rows pick a component, uniform rows the whole mixture), and
``gmm_responsibilities(model.encode(...), out_lens, mean, log_var, prob)`` shows which components recorded utterances use.
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


_rng_states = {}


def _default_rng_state(device) -> Tensor:
    """The sampler's device {seed, counter} word for ``device`` when the caller passes none."""
    key = (device.type, device.index)
    if key not in _rng_states:
        seed = (torch.initial_seed() ^ 0x2545F4914F6CDD1D) & 0x7FFFFFFFFFFFFFFF
        _rng_states[key] = torch.tensor([seed, 0], dtype=torch.int64, device=device)
    return _rng_states[key]


def _mixture_args(where, mean, log_var, prob, B):
    """Shape checks of (mean, log_var, prob) against B rows -> (K, per_row).  ValueError on any mismatch."""
    if not all(torch.is_tensor(t) for t in (mean, log_var, prob)):
        raise ValueError(f"{where}: mean, log_var and prob must be tensors")
    if prob.dim() != 2 or prob.size(0) != B:
        raise ValueError(f"{where}: prob must be [B, K] with B = {B}, got {tuple(prob.shape)}")
    K = prob.size(1)
    if not 1 <= K <= _lib.GMM_MAX_COMPONENTS:
        raise ValueError(f"{where}: the mixture kernels take 1 to {_lib.GMM_MAX_COMPONENTS} components, got {K}")
    if mean.dim() != 3 or tuple(mean.shape) != tuple(log_var.shape) or mean.size(0) not in (1, B) or mean.size(2) != K \
            or not 1 <= mean.size(1) <= 80:
        raise ValueError(f"{where}: mean and log_var must both be [B or 1, n_mel <= 80, K] with B = {B}, K = {K}, got "
                         f"{tuple(mean.shape)} and {tuple(log_var.shape)}")
    return K, mean.size(0) == B


def sample_mixture(mean: Tensor, log_var: Tensor, prob: Tensor, n_frames, T: int, sigma: float = 1.0, component=None,
                   *, rng_state: Tensor = None) -> Tensor:
    """Draw z from the Gaussian-mixture prior, element by element as FlowtronLoss(gm_loss=True) models it.

    mean / log_var [B, 80, K] (learned Gaussians) or [1, 80, K] (fixed ones, shared by every row), prob [B, K] -- what
    ``Flowtron.mixture`` returns, or weights the caller wrote (non-negative, positive sum, not necessarily normalised) --
    n_frames [B] in [1, T] -> z [B, 80, T] f32.  For t < n_frames[b], element (c, t) of row b takes component k drawn
    from prob[b] (or k = component[b] when ``component``, ints [B] in [-1, K), gives one; -1 draws) and is
    ``mean[b|0, c, k] + sigma * exp(log_var[b|0, c, k] / 2) * eps`` with eps ~ N(0, 1); z is zero from n_frames[b] on.  It
    feeds ``infer_batch(residual=z, max_frames=n_frames)`` and the other synthesis entry points as it is.

    Randomness is counter based: ``rng_state`` is an int64 CUDA tensor [seed, counter] (default: one per device, seeded
    from ``torch.initial_seed()``); the draws of element (b, c, t) depend only on (seed, counter, b, c, t), so row b
    equals its B = 1 call and a larger T changes no valid element.  Each call adds 1 to the counter on the device, so
    replays of a captured CUDA graph draw new values, in the order eager calls would.  One sampling launch plus the counter
    update, no allocation besides z, no host synchronisation.  Host n_frames and component are checked (ValueError); CUDA
    ones are trusted (a component value outside [0, K) then draws).  Shape errors and K > 32 raise ValueError, CPU
    tensors FlowtronB200Error, all before any device work."""
    where = "sample_mixture"
    if isinstance(T, bool) or int(T) != T or T < 1:
        raise ValueError(f"{where}: T must be a positive integer, got {T}")
    T = int(T)
    sigma = float(sigma)
    if not (sigma >= 0.0 and math.isfinite(sigma)):
        raise ValueError(f"{where}: sigma must be a finite non-negative number, got {sigma}")
    B = prob.size(0) if torch.is_tensor(prob) and prob.dim() == 2 else -1
    K, per_row = _mixture_args(where, mean, log_var, prob, B)
    n_frames = _lib.ragged_lengths(n_frames, B, T, "n_frames")
    if component is not None:
        if torch.is_tensor(component) and component.is_cuda:
            if component.dim() != 1 or component.numel() != B or component.is_floating_point():
                raise ValueError(f"{where}: component must hold {B} integers, got {tuple(component.shape)}")
        else:
            c = torch.as_tensor(component)
            if c.dim() != 1 or c.numel() != B or c.is_floating_point() or c.dtype == torch.bool:
                raise ValueError(f"{where}: component must hold {B} integers, got shape {tuple(c.shape)}")
            if bool((c < -1).any()) or bool((c >= K).any()):
                raise ValueError(f"{where}: component values must lie in [-1, {K}), got {c.tolist()}")
            component = c
    if rng_state is not None and (not torch.is_tensor(rng_state) or rng_state.dtype != torch.int64
                                  or tuple(rng_state.shape) != (2,)):
        raise ValueError(f"{where}: rng_state must be an int64 tensor [2] = (seed, counter)")
    if not all(t.is_cuda for t in (mean, log_var, prob)) or (rng_state is not None and not rng_state.is_cuda):
        raise FlowtronB200Error(f"{where} needs CUDA tensors: the sm_90a kernel is the only implementation")
    dev = prob.device
    rng = _default_rng_state(dev) if rng_state is None else rng_state
    lens = n_frames.to(device=dev, dtype=torch.int32)
    comp = None if component is None else component.to(device=dev, dtype=torch.int32)
    z = torch.empty(B, mean.size(1), T, dtype=torch.float32, device=dev)
    _lib.gmm_sample(mean.float().contiguous(), log_var.float().contiguous(), prob.float().contiguous(), per_row, lens,
                    comp, sigma, rng, z)
    return z


def gmm_responsibilities(z: Tensor, out_lens, mean: Tensor, log_var: Tensor, prob: Tensor) -> Tensor:
    """Which mixture components each utterance's z lands in.

    z [B, 80, T] f32 (``Flowtron.encode``'s output), out_lens [B], mean / log_var [B or 1, 80, K], prob [B, K] (what
    ``Flowtron.mixture`` returns) -> r [B, K]: r[b, k] is the mean over row b's valid elements (t < out_lens[b], every
    channel) of the posterior prob_k N_k(z) / sum_j prob_j N_j(z), formed in log space with the mixture NLL's max shift;
    each row sums to 1 up to rounding.

    One kernel pass and a per-row reduction in a fixed order with no atomics (``ft_gmm_responsibilities``): row b equals
    its B = 1 call bit for bit.  Host out_lens must lie in [1, T] (ValueError); CUDA ones are trusted and the call makes no
    host synchronisation.  Shape errors and K > 32 raise ValueError, CPU tensors FlowtronB200Error."""
    where = "gmm_responsibilities"
    if not torch.is_tensor(z) or z.dim() != 3:
        raise ValueError(f"{where}: z must be [B, n_mel, T], got {tuple(z.shape) if torch.is_tensor(z) else type(z).__name__}")
    B, M, T = z.shape
    if B < 1 or T < 1:
        raise ValueError(f"{where}: z is empty: {tuple(z.shape)}")
    K, per_row = _mixture_args(where, mean, log_var, prob, B)
    if mean.size(1) != M:
        raise ValueError(f"{where}: z has {M} channels, mean {mean.size(1)}")
    out_lens = _lib.ragged_lengths(out_lens, B, T, "out_lens")
    if not all(t.is_cuda for t in (z, mean, log_var, prob)):
        raise FlowtronB200Error(f"{where} needs CUDA tensors: the sm_90a kernel is the only implementation")
    dev = z.device
    zt = z.permute(2, 0, 1).float().contiguous()      # [T, B, M]: Flowtron.encode's storage order, so no copy for its output
    resp = torch.empty(B, K, dtype=torch.float32, device=dev)
    _lib.gmm_responsibilities(zt, out_lens.to(device=dev, dtype=torch.int32), mean.float().contiguous(),
                              log_var.float().contiguous(), prob.float().contiguous(), per_row, resp)
    return resp
