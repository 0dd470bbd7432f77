"""CPU fp32 restatement of WaveGlow.infer (tacotron2/waveglow/glow.py:251-293) with explicit noise, written from the
math rather than from the reference module: the checker of flowtron_b200.waveglow at sizes where the reference itself is
not at hand.  Takes a state_dict in either weight-norm form or plain-weight form."""
from __future__ import annotations

import torch
import torch.nn.functional as F

from flowtron_b200 import synth


def conv_weight(sd, pre):
    """Effective weight of conv `pre`: g * v / |v| (norm over all dims but 0) in weight-norm form, else `weight`."""
    if f"{pre}.weight_g" in sd:
        v, g = sd[f"{pre}.weight_v"].float(), sd[f"{pre}.weight_g"].float()
        return v * (g / v.flatten(1).norm(dim=1).view(-1, 1, 1))
    return sd[f"{pre}.weight"].float()


def _conv(sd, pre, x, **kw):
    return F.conv1d(x, conv_weight(sd, pre), sd[f"{pre}.bias"].float(), **kw)


def wn(sd, pre, audio0, spect, n_layers, C):
    h = _conv(sd, f"{pre}.start", audio0)
    cond = _conv(sd, f"{pre}.cond_layer", spect)
    skip = 0.0
    for i in range(n_layers):
        d = 2 ** i
        x = _conv(sd, f"{pre}.in_layers.{i}", h, dilation=d, padding=d) + cond[:, 2 * C * i: 2 * C * (i + 1)]
        acts = torch.tanh(x[:, :C]) * torch.sigmoid(x[:, C:])
        rs = _conv(sd, f"{pre}.res_skip_layers.{i}", acts)
        if i < n_layers - 1:
            h = h + rs[:, :C]
            skip = skip + rs[:, C:]
        else:
            skip = skip + rs
    return F.conv1d(skip, sd[f"{pre}.end.weight"].float(), sd[f"{pre}.end.bias"].float())


def upsample(sd, mel):
    """ConvTranspose1d(80, 80, 1024, stride=256), trimmed to 256 F samples, grouped by 8: [B, 640, 32 F], channel c*8+j."""
    B, M, Fr = mel.shape
    up = F.conv_transpose1d(mel.float(), sd["upsample.weight"].float(), sd["upsample.bias"].float(), stride=256)[:, :, :256 * Fr]
    return up.view(B, M, 32 * Fr, 8).permute(0, 1, 3, 2).reshape(B, M * 8, 32 * Fr)


def waveglow_infer(sd, mel, noise, sigma, cfg=synth.DEFAULT_WAVEGLOW_CONFIG, lengths=None):
    """mel [B, 80, F], noise [B, 8, 32 F] (WaveGlow.infer's `noise` layout) -> audio [B, 256 F].  With lengths, row b is the
    B=1 result on mel[b, :, :lengths[b]] and zero after 256 lengths[b] samples."""
    B, _, Fr = mel.shape
    if lengths is not None:
        out = torch.zeros(B, 256 * Fr)
        for b, n in enumerate(lengths):
            n = int(n)
            out[b, :256 * n] = waveglow_infer(sd, mel[b:b + 1, :, :n], noise[b:b + 1, :, :32 * n], sigma, cfg)[0]
        return out
    L, C = cfg["WN_config"]["n_layers"], cfg["WN_config"]["n_channels"]
    chans = synth.waveglow_channels(cfg)
    spect = upsample(sd, mel)
    noise = noise.float()
    c = chans[-1][0]
    audio = sigma * noise[:, 8 - c:]
    for k in reversed(range(cfg["n_flows"])):
        c, nh = chans[k]
        out = wn(sd, f"WN.{k}", audio[:, :nh], spect, L, C)
        a1 = (audio[:, nh:] - out[:, :nh]) / torch.exp(out[:, nh:])
        audio = torch.cat([audio[:, :nh], a1], 1)
        w_inv = torch.linalg.inv(sd[f"convinv.{k}.conv.weight"].double().squeeze(-1)).float()
        audio = torch.einsum("ij,bjt->bit", w_inv, audio)
        if k % cfg["n_early_every"] == 0 and k > 0:
            e = cfg["n_early_size"]
            audio = torch.cat([sigma * noise[:, 8 - c - e: 8 - c], audio], 1)
    return audio.permute(0, 2, 1).reshape(B, -1)


def max_log_s(sd, mel, noise, sigma, cfg=synth.DEFAULT_WAVEGLOW_CONFIG):
    """max |log_s| per flow of one inverse pass (how strongly the synthetic `end` weights act)."""
    L, C = cfg["WN_config"]["n_layers"], cfg["WN_config"]["n_channels"]
    chans = synth.waveglow_channels(cfg)
    spect = upsample(sd, mel)
    c = chans[-1][0]
    audio = sigma * noise[:, 8 - c:]
    res = {}
    for k in reversed(range(cfg["n_flows"])):
        c, nh = chans[k]
        out = wn(sd, f"WN.{k}", audio[:, :nh], spect, L, C)
        res[k] = out[:, nh:].abs().max().item()
        a1 = (audio[:, nh:] - out[:, :nh]) / torch.exp(out[:, nh:])
        audio = torch.cat([audio[:, :nh], a1], 1)
        audio = torch.einsum("ij,bjt->bit", torch.linalg.inv(sd[f"convinv.{k}.conv.weight"].double().squeeze(-1)).float(), audio)
        if k % cfg["n_early_every"] == 0 and k > 0:
            e = cfg["n_early_size"]
            audio = torch.cat([sigma * noise[:, 8 - c - e: 8 - c], audio], 1)
    return res
