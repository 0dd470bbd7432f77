"""Mel front-end with the reference's API (audio_processing.py: TacotronSTFT :96-134, STFT :172-270).

``TacotronSTFT.mel_spectrogram(y[B,N]) -> [B,80,F]`` runs on the GPU: for the shipped filter_length 1024 as ONE fused
kernel (csrc/mel_fused.cu: reflect pad + window on the load, per-warp 1024-point FFT in shared memory, |X|, sparse
filterbank, log; waveform read once, mel written once), for other sizes as framing kernel + batched cuFFT + fused
magnitude / filterbank / log (csrc/mel.cu).  ``mel_spectrogram_packed`` / ``mel_spectrogram_ragged`` are the batched
forms for a whole dataset shard (what data.py:149-155 does one utterance at a time on a CPU worker); int16 PCM input is
scaled by 1/32768 on load (data.py:150).  ``STFT.transform`` returns (magnitude, phase) like the reference.
``STFT.inverse`` (:237-265) is one kernel for filter_length 1024 and hop 128 / 256 / 512 (csrc/istft.cu: per-warp inverse
FFT, window, overlap-add and the window sum-square normalisation), ``STFT.forward`` is transform + inverse, and
``griffin_lim`` (:59-75) alternates the two; the WaveGlow Denoiser built on them is flowtron_b200.denoiser.
Buffers ``mel_basis``, ``stft_fn.forward_basis``, ``stft_fn.inverse_basis`` keep the reference's state_dict layout.
"""
from __future__ import annotations

import numpy as np
import torch

from . import _lib
from ._lib import FlowtronB200Error


def _hz_to_mel(f):
    f = np.asarray(f, dtype=np.float64)
    lin = f * 3.0 / 200.0
    return np.where(f >= 1000.0, 15.0 + np.log(np.maximum(f, 1e-10) / 1000.0) * (27.0 / np.log(6.4)), lin)


def _mel_to_hz(m):
    m = np.asarray(m, dtype=np.float64)
    return np.where(m >= 15.0, 1000.0 * np.exp((m - 15.0) * (np.log(6.4) / 27.0)), m * 200.0 / 3.0)


def mel_filterbank(sr, n_fft, n_mels=80, fmin=0.0, fmax=None):
    """Slaney-scale, area-normalised triangular filterbank == librosa.filters.mel(sr, n_fft, n_mels, fmin, fmax)
    with librosa<=0.8 defaults (htk=False, norm=1), the call at audio_processing.py:104-105."""
    fmax = sr / 2.0 if fmax is None else fmax
    bins = np.linspace(0.0, sr / 2.0, 1 + n_fft // 2)
    edges = _mel_to_hz(np.linspace(_hz_to_mel(fmin), _hz_to_mel(fmax), n_mels + 2))
    lower = (bins[None, :] - edges[:-2, None]) / (edges[1:-1] - edges[:-2])[:, None]
    upper = (edges[2:, None] - bins[None, :]) / (edges[2:] - edges[1:-1])[:, None]
    fb = np.maximum(0.0, np.minimum(lower, upper)) * (2.0 / (edges[2:] - edges[:-2]))[:, None]
    return fb.astype(np.float32)


def _padded_window(win_length, filter_length):
    w = 0.5 - 0.5 * np.cos(2.0 * np.pi * np.arange(win_length) / win_length)      # get_window('hann', fftbins=True)
    lp = (filter_length - win_length) // 2
    return np.pad(w, (lp, filter_length - win_length - lp))


def aligned_waveform(x):
    """x as a contiguous float32 tensor whose storage starts on an 8-byte boundary: the transform kernel reads sample pairs
    as float2, so a view that starts at an odd float offset (e.g. one row of an odd-length batch) is copied first."""
    x = x.detach().float().contiguous()
    return x if x.data_ptr() % 8 == 0 else x.clone()


class STFT(torch.nn.Module):
    def __init__(self, filter_length=800, hop_length=200, win_length=800, window='hann'):
        super().__init__()
        assert window == 'hann' and filter_length >= win_length
        self.filter_length, self.hop_length, self.win_length, self.window = filter_length, hop_length, win_length, window
        fb = np.fft.fft(np.eye(filter_length))
        cutoff = filter_length // 2 + 1
        fb = np.vstack([np.real(fb[:cutoff]), np.imag(fb[:cutoff])])
        scale = filter_length / hop_length
        w = torch.from_numpy(_padded_window(win_length, filter_length)).float()
        self.register_buffer('forward_basis', (torch.FloatTensor(fb[:, None, :]) * w).float())
        self.register_buffer('inverse_basis', (torch.FloatTensor(np.linalg.pinv(scale * fb).T[:, None, :]) * w).float())
        self.register_buffer('_window', w, persistent=False)

    def transform(self, input_data):
        """audio_processing.py:207-235: input [B, N] -> (magnitude [B, n_fft/2+1, F], phase [B, n_fft/2+1, F]),
        F = 1 + N // hop, phase = atan2(imag, real).  CUDA only (fused FFT kernel, filter_length 1024)."""
        if not input_data.is_cuda:
            raise FlowtronB200Error("STFT.transform needs CUDA tensors: the sm_90a path is the only implementation")
        if self.filter_length != 1024:
            raise NotImplementedError("STFT.transform is built for filter_length 1024 (config.json:31)")
        B, N = input_data.shape
        if N <= self.filter_length // 2:
            raise ValueError("input shorter than the reflect padding")
        self.num_samples = N
        F = 1 + N // self.hop_length
        dev = input_data.device
        so = torch.arange(B + 1, device=dev, dtype=torch.int64) * N
        fo = torch.arange(B + 1, device=dev, dtype=torch.int64) * F
        cutoff = self.filter_length // 2 + 1
        magnitude = torch.empty(B, cutoff, F, device=dev)
        phase = torch.empty(B, cutoff, F, device=dev)
        _lib.stft_transform(input_data.detach().float().contiguous(), so, fo, B, B * F, self._window, self.filter_length,
                            self.hop_length, magnitude, phase)
        return magnitude, phase

    def inverse(self, magnitude, phase):
        """audio_processing.py:237-265: (magnitude, phase) [B, n_fft/2+1, F] -> [B, 1, (F-1) * hop].  CUDA only (one
        kernel, filter_length 1024, hop 128 / 256 / 512); F == 1 gives an empty signal."""
        if self.filter_length != 1024 or self.hop_length not in _lib.STFT_INVERSE_HOPS:
            raise NotImplementedError("STFT.inverse is built for filter_length 1024 and hop_length 128, 256 or 512")
        cutoff = self.filter_length // 2 + 1
        if magnitude.dim() != 3 or magnitude.shape[1] != cutoff or magnitude.shape != phase.shape:
            raise ValueError(f"magnitude and phase must both be [B, {cutoff}, F], got {tuple(magnitude.shape)} and "
                             f"{tuple(phase.shape)}")
        if not magnitude.is_cuda or not phase.is_cuda:
            raise FlowtronB200Error("STFT.inverse needs CUDA tensors: the sm_90a path is the only implementation")
        B, _, F = magnitude.shape
        hop, dev = self.hop_length, magnitude.device
        out = torch.empty(B, 1, (F - 1) * hop, device=dev)
        if F == 1 or B == 0:
            return out
        fo = torch.arange(B + 1, device=dev, dtype=torch.int64) * F
        oo = torch.arange(B, device=dev, dtype=torch.int64) * ((F - 1) * hop)
        _lib.stft_inverse(magnitude.detach().float().contiguous(), phase.detach().float().contiguous(), fo, oo, B, B * F,
                          self._window, self.filter_length, hop, out)
        return out

    def forward(self, input_data):
        """audio_processing.py:267-270: transform, keep (magnitude, phase), return their inverse."""
        self.magnitude, self.phase = self.transform(aligned_waveform(input_data))
        return self.inverse(self.magnitude, self.phase)


def griffin_lim(magnitudes, stft_fn, n_iters=30, *, angles=None):
    """audio_processing.py:59-75: phase reconstruction from magnitudes [B, n_fft/2+1, F] (CUDA) -> signal [B, (F-1) * hop].
    angles=None draws the initial phase as the reference does (numpy's global generator, so a numpy seed reproduces the
    reference's draw) and copies it to the device once; explicit ``angles`` (CUDA, like magnitudes) make the call
    1 + 2 n_iters kernel launches with no host work in between, so it can be captured in a CUDA graph."""
    if angles is None:
        a = np.angle(np.exp(2j * np.pi * np.random.rand(*magnitudes.size()))).astype(np.float32)
        angles = torch.from_numpy(a).to(magnitudes.device)
    signal = stft_fn.inverse(magnitudes, angles).squeeze(1)
    for _ in range(n_iters):
        _, angles = stft_fn.transform(signal)
        signal = stft_fn.inverse(magnitudes, angles).squeeze(1)
    return signal


class TacotronSTFT(torch.nn.Module):
    def __init__(self, filter_length=1024, hop_length=256, win_length=1024, n_mel_channels=80, sampling_rate=22050,
                 mel_fmin=0.0, mel_fmax=None):
        super().__init__()
        self.n_mel_channels, self.sampling_rate = n_mel_channels, sampling_rate
        self.stft_fn = STFT(filter_length, hop_length, win_length)
        basis = mel_filterbank(sampling_rate, filter_length, n_mel_channels, mel_fmin, mel_fmax)
        self.register_buffer('mel_basis', torch.from_numpy(basis).float())
        nz = basis > 0
        lo = np.where(nz.any(1), nz.argmax(1), 0).astype(np.int32)
        hi = np.where(nz.any(1), basis.shape[1] - nz[:, ::-1].argmax(1), 0).astype(np.int32)
        self.register_buffer('_band_lo', torch.from_numpy(lo), persistent=False)
        self.register_buffer('_band_hi', torch.from_numpy(hi), persistent=False)

    def spectral_normalize(self, magnitudes):
        return torch.log(torch.clamp(magnitudes, min=1e-5))

    def spectral_de_normalize(self, magnitudes):
        return torch.exp(magnitudes)

    def _run(self, flat, so, fo, n_utt, total, out):
        hop, n_fft = self.stft_fn.hop_length, self.stft_fn.filter_length
        if n_fft == 1024:
            _lib.mel_spectrogram_fused(flat, so, fo, n_utt, total, self.stft_fn._window, self.mel_basis, self._band_lo,
                                       self._band_hi, n_fft, hop, 1e-5, out)
        else:
            if flat.dtype != torch.float32:
                flat = flat.float() / 32768.0
            _lib.mel_spectrogram(flat, so, fo, n_utt, total, self.stft_fn._window, self.mel_basis, self._band_lo,
                                 self._band_hi, n_fft, hop, 1e-5, out)

    def mel_spectrogram_packed(self, flat, lengths, out=None):
        """Whole-shard form: ``flat`` = the utterances concatenated (f32 in [-1, 1] or int16 PCM, CUDA), ``lengths`` = their
        sample counts (host sequence; each > filter_length/2).  Returns (mel_packed, frame_offsets): per-utterance
        [n_mel, 1 + N_u // hop] blocks concatenated (utterance u = mel_packed[fo[u]*n_mel : fo[u+1]*n_mel].view(n_mel, -1))
        and the host int64 prefix sums fo.  One kernel launch for the whole shard; no host sync."""
        if not flat.is_cuda:
            raise FlowtronB200Error("TacotronSTFT needs CUDA tensors: the sm_90a path is the only implementation")
        if flat.dtype not in (torch.float32, torch.int16):
            raise TypeError("waveform must be float32 in [-1, 1] or int16 PCM")
        hop, n_fft = self.stft_fn.hop_length, self.stft_fn.filter_length
        lens = np.asarray(lengths, dtype=np.int64)
        if lens.min() <= n_fft // 2:
            raise ValueError("utterance shorter than the reflect padding (torch's reflect pad raises too)")
        so = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
        fo = np.concatenate([[0], np.cumsum(1 + lens // hop)]).astype(np.int64)
        assert int(so[-1]) == flat.numel(), "lengths do not add up to the packed waveform"
        dev = flat.device
        total = int(fo[-1])
        if out is None:
            out = torch.empty(total * self.n_mel_channels, device=dev)
        self._run(flat.contiguous(), torch.from_numpy(so).to(dev, non_blocking=True), torch.from_numpy(fo).to(dev, non_blocking=True),
                  len(lens), total, out)
        return out, fo

    def mel_spectrogram_ragged(self, wavs):
        """wavs: list of 1-D float tensors in [-1, 1] (any lengths > filter_length/2) -> list of [n_mel, 1 + N//hop]."""
        if not wavs[0].is_cuda:
            raise FlowtronB200Error("TacotronSTFT needs CUDA tensors: the sm_90a path is the only implementation")
        flat = torch.cat([w.reshape(-1).float() for w in wavs]) if len(wavs) > 1 else wavs[0].reshape(-1).float().contiguous()
        out, fo = self.mel_spectrogram_packed(flat, [int(w.numel()) for w in wavs])
        return [out[fo[i] * self.n_mel_channels: fo[i + 1] * self.n_mel_channels].view(self.n_mel_channels, -1)
                for i in range(len(wavs))]

    def mel_spectrogram(self, y):
        """y: [B, N] in [-1, 1] -> [B, n_mel_channels, 1 + N // hop]  (audio_processing.py:117-134)."""
        assert torch.min(y.data) >= -1
        assert torch.max(y.data) <= 1
        if not y.is_cuda:
            raise FlowtronB200Error("TacotronSTFT needs CUDA tensors: the cuFFT/sm_90a path is the only implementation")
        B, N = y.shape
        hop, n_fft = self.stft_fn.hop_length, self.stft_fn.filter_length
        if N <= n_fft // 2:
            raise ValueError("input shorter than the reflect padding")
        F = 1 + N // hop
        dev = y.device
        so = torch.arange(B + 1, device=dev, dtype=torch.int64) * N
        fo = torch.arange(B + 1, device=dev, dtype=torch.int64) * F
        out = torch.empty(B, self.n_mel_channels, F, device=dev)
        self._run(y.detach().float().contiguous(), so, fo, B, B * F, out)
        return out
