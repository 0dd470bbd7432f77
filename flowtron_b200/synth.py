"""Deterministic synthetic weights and inputs (the reference ships no data: filelists point at
/path_to_ljs/..., SURVEY.md §2.1 row 16).  Shared by bench.py, __graft_entry__.smoke(), the golden
generator and the tests.

Weights are a pure function of (parameter name, shape, seed) — independent of module construction
order — so the reference model (in tests/make_golden.py), the oracle and the CUDA path all see
identical values without shipping a 240 MB checkpoint.  The key layout is the reference's
state_dict layout (SURVEY.md §8a row 15; train.py:131-139).
"""
from __future__ import annotations

import math
import zlib
from typing import Dict, Tuple

import numpy as np
import torch

DEFAULT_MODEL_CONFIG = dict(  # /root/reference/config.json:49-66
    n_speakers=1, n_speaker_dim=128, n_text=185, n_text_dim=512, n_flows=2, n_mel_channels=80,
    n_attn_channels=640, n_hidden=1024, n_lstm_layers=2, mel_encoder_n_hidden=512, n_components=0,
    mean_scale=0.0, fixed_gaussian=True, dummy_speaker_embedding=False, use_gate_layer=True,
    use_cumm_attention=False)


def param_shapes(cfg: dict) -> Dict[str, Tuple[int, ...]]:
    """state_dict key -> shape for Flowtron(**cfg) (n_components=0, no cumulative attention)."""
    H, A, M = cfg["n_hidden"], cfg["n_attn_channels"], cfg["n_mel_channels"]
    Dt, Ds = cfg["n_text_dim"], cfg["n_speaker_dim"]
    E = Dt + Ds
    s: Dict[str, Tuple[int, ...]] = {}
    s["speaker_embedding.weight"] = (cfg["n_speakers"], Ds)
    s["embedding.weight"] = (cfg["n_text"], Dt)
    for i in range(3):
        s[f"encoder.convolutions.{i}.0.conv.weight"] = (Dt, Dt, 5)
        s[f"encoder.convolutions.{i}.0.conv.bias"] = (Dt,)
        s[f"encoder.convolutions.{i}.1.weight"] = (Dt,)
        s[f"encoder.convolutions.{i}.1.bias"] = (Dt,)
    for sfx in ("", "_reverse"):
        s[f"encoder.lstm.weight_ih_l0{sfx}"] = (4 * (Dt // 2), Dt)
        s[f"encoder.lstm.weight_hh_l0{sfx}"] = (4 * (Dt // 2), Dt // 2)
        s[f"encoder.lstm.bias_ih_l0{sfx}"] = (4 * (Dt // 2),)
        s[f"encoder.lstm.bias_hh_l0{sfx}"] = (4 * (Dt // 2),)
    for i in range(cfg["n_flows"]):
        pre = f"flows.{i}" if i % 2 == 0 else f"flows.{i}.ar_step"
        s[f"{pre}.conv.weight"] = (2 * M, H, 1)
        s[f"{pre}.conv.bias"] = (2 * M,)
        for l in range(cfg["n_lstm_layers"]):
            s[f"{pre}.lstm.weight_ih_l{l}"] = (4 * H, (H + A) if l == 0 else H)
            s[f"{pre}.lstm.weight_hh_l{l}"] = (4 * H, H)
            s[f"{pre}.lstm.bias_ih_l{l}"] = (4 * H,)
            s[f"{pre}.lstm.bias_hh_l{l}"] = (4 * H,)
        s[f"{pre}.attention_lstm.weight_ih_l0"] = (4 * H, M)
        s[f"{pre}.attention_lstm.weight_hh_l0"] = (4 * H, H)
        s[f"{pre}.attention_lstm.bias_ih_l0"] = (4 * H,)
        s[f"{pre}.attention_lstm.bias_hh_l0"] = (4 * H,)
        s[f"{pre}.attention_layer.query.linear_layer.weight"] = (A, H)
        s[f"{pre}.attention_layer.key.linear_layer.weight"] = (A, E)
        s[f"{pre}.attention_layer.value.linear_layer.weight"] = (A, E)
        s[f"{pre}.attention_layer.v.linear_layer.weight"] = (1, A)
        for j in range(2):
            s[f"{pre}.dense_layer.layers.{j}.linear_layer.weight"] = (H, H)
            s[f"{pre}.dense_layer.layers.{j}.linear_layer.bias"] = (H,)
        if i == cfg["n_flows"] - 1 and cfg["use_gate_layer"]:
            s[f"{pre}.gate_layer.linear_layer.weight"] = (1, H + A)
            s[f"{pre}.gate_layer.linear_layer.bias"] = (1,)
    return s


def _std_for(name: str, shape) -> float:
    if name.endswith("embedding.weight"):
        return 1.0
    if ".conv.weight" in name and name.startswith("flows"):
        return 0.02                       # non-trivial affine coupling (reference zero-inits, flowtron.py:652)
    if ".conv.bias" in name and name.startswith("flows"):
        return 0.02
    if "lstm" in name:                    # torch LSTM default U(-k,k), k=1/sqrt(H): std = k/sqrt(3)
        H = shape[0] // 4
        return 1.0 / math.sqrt(3.0 * H)
    if name.endswith(".1.weight"):        # instance-norm affine weight (offset +1 applied below)
        return 0.1
    if name.endswith("bias"):
        return 0.05
    if len(shape) >= 2:                   # xavier-like
        fan_out, fan_in = shape[0], int(np.prod(shape[1:]))
        return math.sqrt(2.0 / (fan_in + fan_out))
    return 0.05


def synth_params(cfg: dict, seed: int = 1234, scale: float = 1.0, dtype=torch.float32) -> Dict[str, torch.Tensor]:
    """Deterministic N(0, std(name)) weights for every state_dict key."""
    out = {}
    for name, shape in param_shapes(cfg).items():
        g = torch.Generator(device="cpu")
        g.manual_seed((seed * 1000003 + zlib.crc32(name.encode())) % (2 ** 63 - 1))
        t = torch.randn(shape, generator=g, dtype=torch.float32) * (_std_for(name, shape) * scale)
        if name.endswith(".1.weight"):
            t = t + 1.0
        out[name] = t.to(dtype)
    return out


def gmm_param_shapes(cfg: dict) -> Dict[str, Tuple[int, ...]]:
    """state_dict key -> shape of the Gaussian-mixture prior's modules (mel_encoder, gaussian_mixture) for
    Flowtron(**cfg) with n_components > 1; learned Gaussians only (the fixed ones are buffers, see synth_gmm_params)."""
    Hm, K, M = cfg["mel_encoder_n_hidden"], cfg["n_components"], cfg["n_mel_channels"]
    s: Dict[str, Tuple[int, ...]] = {}
    for i in range(2):
        s[f"mel_encoder.convolutions.{i}.0.conv.weight"] = (Hm, M if i == 0 else Hm, 3)
        s[f"mel_encoder.convolutions.{i}.0.conv.bias"] = (Hm,)
        s[f"mel_encoder.convolutions.{i}.1.weight"] = (Hm,)
        s[f"mel_encoder.convolutions.{i}.1.bias"] = (Hm,)
    for sfx in ("", "_reverse"):
        s[f"mel_encoder.lstm.weight_ih_l0{sfx}"] = (4 * (Hm // 2), Hm)
        s[f"mel_encoder.lstm.weight_hh_l0{sfx}"] = (4 * (Hm // 2), Hm // 2)
        s[f"mel_encoder.lstm.bias_ih_l0{sfx}"] = (4 * (Hm // 2),)
        s[f"mel_encoder.lstm.bias_hh_l0{sfx}"] = (4 * (Hm // 2),)
    layers = ("prob",) if cfg["fixed_gaussian"] else ("prob", "mean", "log_var")
    for n in layers:
        out = K if n == "prob" else M * K
        s[f"gaussian_mixture.{n}_layer.linear_layer.weight"] = (out, Hm)
        s[f"gaussian_mixture.{n}_layer.linear_layer.bias"] = (out,)
    return s


def synth_gmm_params(cfg: dict, seed: int = 1234) -> Dict[str, torch.Tensor]:
    """Deterministic weights for every state_dict key of Flowtron(**cfg) with n_components > 1: synth_params for the rest of
    the model, the same per-name rule for the prior's parameters and, with fixed_gaussian, the reference's buffers
    (mean = mean_scale * n_components distinct unit vectors, log_var = 0) from a seeded choice of the unit vectors."""
    out = synth_params(dict(cfg, n_components=0), seed)
    for name, shape in gmm_param_shapes(cfg).items():
        g = torch.Generator(device="cpu")
        g.manual_seed((seed * 1000003 + zlib.crc32(name.encode())) % (2 ** 63 - 1))
        t = torch.randn(shape, generator=g, dtype=torch.float32) * _std_for(name, shape)
        out[name] = t + 1.0 if name.endswith(".1.weight") else t
    if cfg["fixed_gaussian"]:
        M, K = cfg["n_mel_channels"], cfg["n_components"]
        g = torch.Generator(device="cpu")
        g.manual_seed(seed)
        ids = torch.randperm(M, generator=g)[:K]
        out["gaussian_mixture.mean"] = (torch.eye(M)[ids] * float(cfg["mean_scale"])).transpose(0, 1)[None].contiguous()
        out["gaussian_mixture.log_var"] = torch.zeros(1, M, K)
    return out


def synth_batch(B: int, T: int, L: int, cfg: dict = DEFAULT_MODEL_CONFIG, seed: int = 1234,
                out_lens=None, in_lens=None, with_prior: bool = False, logmel_stats: bool = False):
    """Synthetic training batch in DataCollate layout (data.py:197-246):
    mel [B,80,T] f32, speaker_ids [B], text [B,L] i64, in_lens [B] (sorted desc), out_lens [B],
    gate_target [B,T], attn_prior [B,T,L] | None.  Pads are zero like the collate's."""
    g = torch.Generator(device="cpu")
    g.manual_seed(seed)
    if out_lens is None:
        lo = max(1, T // 2)
        out_lens = torch.randint(lo, T + 1, (B,), generator=g)
        out_lens[int(torch.randint(0, B, (1,), generator=g))] = T
    else:
        out_lens = torch.as_tensor(out_lens, dtype=torch.long)
    if in_lens is None:
        in_lens = torch.clamp((out_lens.float() / T * L).round().long(), min=max(1, L // 4), max=L)
        in_lens[out_lens.argmax()] = L
    else:
        in_lens = torch.as_tensor(in_lens, dtype=torch.long)
    order = torch.argsort(in_lens, descending=True, stable=True)      # collate sorts by text length
    in_lens, out_lens = in_lens[order].contiguous(), out_lens[order].contiguous()
    M = cfg["n_mel_channels"]
    mel = torch.randn(B, M, T, generator=g)
    if logmel_stats:
        mel = (mel * 2.0 - 5.5).clamp_(-11.5, 2.0)
    text = torch.randint(0, cfg["n_text"], (B, L), generator=g)
    spk = torch.randint(0, cfg["n_speakers"], (B,), generator=g)
    tmask = torch.arange(T)[None, :] < out_lens[:, None]
    lmask = torch.arange(L)[None, :] < in_lens[:, None]
    mel = mel * tmask[:, None, :]
    text = text * lmask
    gate = (torch.arange(T)[None, :] >= (out_lens[:, None] - 1)).float()
    prior = None
    if with_prior:
        prior = torch.zeros(B, T, L)
        for b in range(B):
            pb = beta_binomial_prior(int(in_lens[b]), int(out_lens[b]))
            prior[b, : int(out_lens[b]), : int(in_lens[b])] = torch.from_numpy(pb).float()
    return dict(mel=mel, speaker_ids=spk, text=text, in_lens=in_lens, out_lens=out_lens,
                gate_target=gate, attn_prior=prior)


def beta_binomial_prior(phoneme_count: int, mel_count: int, scaling: float = 1.0) -> np.ndarray:
    """Attention prior of data.py:31-41 (BetaBinomial(k; n=P-1, a=s*i, b=s*(M+1-i)), i=1..M) in closed form via
    log-gamma; float64 [mel_count, phoneme_count].  (The reference loops scipy.stats.betabinom per frame.)"""
    from scipy.special import gammaln
    P, Mx = phoneme_count, mel_count
    k = np.arange(P, dtype=np.float64)[None, :]
    i = np.arange(1, Mx + 1, dtype=np.float64)[:, None]
    a, b, n = scaling * i, scaling * (Mx + 1 - i), float(P - 1)
    logc = gammaln(n + 1) - gammaln(k + 1) - gammaln(n - k + 1)
    logb = (gammaln(k + a) + gammaln(n - k + b) - gammaln(n + a + b)
            - (gammaln(a) + gammaln(b) - gammaln(a + b)))
    return np.exp(logc + logb)


def ljs_like_lengths(B: int, T: int, seed: int, lo_frac: float = 0.5):
    """cfg-2 style lengths (SURVEY.md §8d): out_lens ~ U{lo..T} with the max forced to T,
    in_lens = round(out_lens / 6.5) clipped to [40, 160]."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    out_lens = torch.randint(int(T * lo_frac), T + 1, (B,), generator=g)
    out_lens[0] = T
    in_lens = torch.clamp((out_lens.float() / 6.5).round().long(), 40, 160)
    return out_lens, in_lens


# ------------------------------------------------------------------------------------------------ WaveGlow
DEFAULT_WAVEGLOW_CONFIG = dict(  # tacotron2/waveglow/config.json "waveglow_config" (waveglow_256channels_v4.pt)
    n_mel_channels=80, n_flows=12, n_group=8, n_early_every=4, n_early_size=2,
    WN_config=dict(n_layers=8, n_channels=256, kernel_size=3))


def waveglow_channels(cfg: dict):
    """[(n_remaining_channels, n_half)] per flow k, as WaveGlow.__init__ assigns them."""
    out, c = [], cfg["n_group"]
    for k in range(cfg["n_flows"]):
        if k % cfg["n_early_every"] == 0 and k > 0:
            c -= cfg["n_early_size"]
        out.append((c, c // 2))
    return out


def waveglow_param_shapes(cfg: dict, weight_norm: bool = True) -> Dict[str, Tuple[int, ...]]:
    """state_dict key -> shape of the reference WaveGlow(**cfg), in weight-norm form (weight_g / weight_v) or, with
    weight_norm=False, as after WaveGlow.remove_weightnorm (plain weight)."""
    M, G = cfg["n_mel_channels"], cfg["n_group"]
    wn = cfg["WN_config"]
    L, C, K = wn["n_layers"], wn["n_channels"], wn["kernel_size"]
    s: Dict[str, Tuple[int, ...]] = {"upsample.weight": (M, M, 1024), "upsample.bias": (M,)}

    def conv(pre, co, ci, k, normed=True):
        s[f"{pre}.bias"] = (co,)
        if normed and weight_norm:
            s[f"{pre}.weight_g"] = (co, 1, 1)
            s[f"{pre}.weight_v"] = (co, ci, k)
        else:
            s[f"{pre}.weight"] = (co, ci, k)

    for k, (c, nh) in enumerate(waveglow_channels(cfg)):
        pre = f"WN.{k}"
        for i in range(L):
            conv(f"{pre}.in_layers.{i}", 2 * C, C, K)
        for i in range(L):
            conv(f"{pre}.res_skip_layers.{i}", 2 * C if i < L - 1 else C, C, 1)
        conv(f"{pre}.start", C, nh, 1)
        conv(f"{pre}.end", 2 * nh, C, 1, normed=False)
        conv(f"{pre}.cond_layer", 2 * C * L, M * G, 1)
        s[f"convinv.{k}.conv.weight"] = (c, c, 1)
    return s


def synth_waveglow_params(cfg: dict = DEFAULT_WAVEGLOW_CONFIG, seed: int = 1234) -> Dict[str, torch.Tensor]:
    """Deterministic WaveGlow weights in weight-norm form (reference state_dict keys).  weight_g differs from |weight_v| so a
    weight-norm fold is exercised; `end` is non-zero (max |log_s| of about 0.1-0.5 on synth_waveglow_mel inputs) so every
    affine coupling acts; convinv is orthonormal with det > 0 like Invertible1x1Conv's initialisation."""
    g_ranges = {"start": (0.8, 1.2), "in_layers": (0.5, 1.0), "res_skip_layers": (0.3, 0.6), "cond_layer": (0.3, 0.6)}
    out = {}
    for name, shape in waveglow_param_shapes(cfg, weight_norm=True).items():
        g = torch.Generator(device="cpu")
        g.manual_seed((seed * 1000003 + zlib.crc32(name.encode())) % (2 ** 63 - 1))
        if name.startswith("convinv"):
            c = shape[0]
            q = torch.linalg.qr(torch.randn(c, c, generator=g, dtype=torch.float64))[0]
            if torch.det(q) < 0:
                q[:, 0] = -q[:, 0]
            t = q.float().view(c, c, 1)
        elif name.endswith("weight_g"):
            lo, hi = g_ranges[name.split(".")[2]]
            t = lo + (hi - lo) * torch.rand(shape, generator=g)
        elif name.endswith("weight_v"):
            t = torch.randn(shape, generator=g)
        elif name == "upsample.weight":
            t = torch.randn(shape, generator=g) * 0.01
        elif name.endswith("end.weight"):
            t = torch.randn(shape, generator=g) * 0.012
        elif name.endswith("end.bias"):
            t = torch.randn(shape, generator=g) * 0.01
        else:                                                  # biases
            t = torch.randn(shape, generator=g) * 0.05
        out[name] = t.contiguous()
    return out


def synth_waveglow_mel(B: int, F: int, seed: int) -> torch.Tensor:
    """Log-mel-like input [B, 80, F] (the statistics of synth_batch(logmel_stats=True))."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(B, 80, F, generator=g) * 2.0 - 5.5).clamp_(-11.5, 2.0)


def synth_waveglow_noise(B: int, F: int, seed: int) -> torch.Tensor:
    """N(0, 1) noise [B, 8, 32 F] in WaveGlow.infer's `noise` layout."""
    g = torch.Generator(device="cpu").manual_seed(seed + 7919)
    return torch.randn(B, 8, 32 * F, generator=g)


# ------------------------------------------------------------------------------------------------ inverse STFT / Denoiser
def synth_istft_audio(B: int, N: int, seed: int) -> torch.Tensor:
    """Speech-band test signal [B, N] in [-1, 1]: a few sinusoids with random frequencies, phases and slow amplitude
    envelopes, plus white noise at -40 dB."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    t = torch.arange(N, dtype=torch.float64)[None, None, :] / 22050.0
    f = 80.0 + 3920.0 * torch.rand(B, 6, 1, generator=g, dtype=torch.float64)
    ph = 2 * np.pi * torch.rand(B, 6, 1, generator=g, dtype=torch.float64)
    env = 0.5 + 0.5 * torch.sin(2 * np.pi * (0.5 + 3.0 * torch.rand(B, 6, 1, generator=g, dtype=torch.float64)) * t)
    y = (env * torch.sin(2 * np.pi * f * t + ph)).sum(1) / 6.0
    y = y + 0.01 * torch.randn(B, N, generator=g, dtype=torch.float64)
    return y.clamp(-1.0, 1.0).float()


def synth_istft_spectrum(B: int, F: int, seed: int, n_bins: int = 513):
    """A random, inconsistent (magnitude, phase) pair, each [B, n_bins, F] float32: magnitudes U[0, 2), phases U[-pi, pi),
    non-zero phase at the DC and Nyquist bins included."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    mag = 2.0 * torch.rand(B, n_bins, F, generator=g)
    phase = (2.0 * torch.rand(B, n_bins, F, generator=g) - 1.0) * float(np.pi)
    return mag, phase
