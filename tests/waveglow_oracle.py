"""Restatement of WaveGlow.infer and of WaveGlow.forward / WaveGlowLoss (tacotron2/waveglow/glow.py:43-58, 196-293),
written from the math rather than from the reference module: the checker of flowtron_b200.waveglow at sizes where the
reference itself is not at hand.  Takes a state_dict in either weight-norm form or plain-weight form.  Infer is a CPU fp32
oracle with explicit noise; forward computes in the dtype of its weights and inputs (fp64 weights give an fp64 oracle) and is
differentiable in the state_dict's tensors."""
from __future__ import annotations

import torch
import torch.nn.functional as F

from flowtron_b200 import synth


def conv_weight(sd, pre):
    """Effective weight of conv `pre` in the dtype of sd: g * v / |v| (norm over all dims but 0) in weight-norm form, else
    `weight`; differentiable in sd's tensors."""
    if f"{pre}.weight_g" in sd:
        v, g = sd[f"{pre}.weight_v"], sd[f"{pre}.weight_g"]
        return v * (g / v.flatten(1).norm(dim=1).view(-1, 1, 1))
    return sd[f"{pre}.weight"]


def wn(sd, pre, audio0, spect, n_layers, C):
    """WN of flow `pre` on audio_0 [B, n_half, T] and the grouped spectrogram -> the end conv's output [B, 2 n_half, T]."""
    def conv(name, x, **kw):
        return F.conv1d(x, conv_weight(sd, f"{pre}.{name}"), sd[f"{pre}.{name}.bias"], **kw)

    h = conv("start", audio0)
    cond = conv("cond_layer", spect)
    skip = 0.0
    for i in range(n_layers):
        d = 2 ** i
        x = conv(f"in_layers.{i}", h, dilation=d, padding=d) + cond[:, 2 * C * i: 2 * C * (i + 1)]
        acts = torch.tanh(x[:, :C]) * torch.sigmoid(x[:, C:])
        rs = conv(f"res_skip_layers.{i}", acts)
        if i < n_layers - 1:
            h = h + rs[:, :C]
            skip = skip + rs[:, C:]
        else:
            skip = skip + rs
    return F.conv1d(skip, sd[f"{pre}.end.weight"], sd[f"{pre}.end.bias"])


def upsample(sd, mel, n):
    """ConvTranspose1d(80, 80, 1024, stride=256), trimmed to n samples, grouped by 8: [B, 640, n / 8], channel c*8+j."""
    B, M, _ = mel.shape
    up = F.conv_transpose1d(mel, sd["upsample.weight"], sd["upsample.bias"], stride=256)[:, :, :n]
    return up.view(B, M, n // 8, 8).permute(0, 1, 3, 2).reshape(B, M * 8, n // 8)


def _infer(sd, mel, noise, sigma, cfg):
    """The inverse pass on fp32 copies of sd, mel and noise: (audio [B, 8, 32 F], max |log_s| per flow)."""
    sd = {k: v.float() for k, v in sd.items()}
    mel, noise = mel.float(), noise.float()
    L, C = cfg["WN_config"]["n_layers"], cfg["WN_config"]["n_channels"]
    chans = synth.waveglow_channels(cfg)
    spect = upsample(sd, mel, 256 * mel.shape[2])
    c = chans[-1][0]
    audio = sigma * noise[:, 8 - c:]
    max_ls = {}
    for k in reversed(range(cfg["n_flows"])):
        c, nh = chans[k]
        out = wn(sd, f"WN.{k}", audio[:, :nh], spect, L, C)
        max_ls[k] = out[:, nh:].abs().max().item()
        a1 = (audio[:, nh:] - out[:, :nh]) / torch.exp(out[:, nh:])
        audio = torch.cat([audio[:, :nh], a1], 1)
        w_inv = torch.linalg.inv(sd[f"convinv.{k}.conv.weight"].double().squeeze(-1)).float()
        audio = torch.einsum("ij,bjt->bit", w_inv, audio)
        if k % cfg["n_early_every"] == 0 and k > 0:
            e = cfg["n_early_size"]
            audio = torch.cat([sigma * noise[:, 8 - c - e: 8 - c], audio], 1)
    return audio, max_ls


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
    return _infer(sd, mel, noise, sigma, cfg)[0].permute(0, 2, 1).reshape(B, -1)


def max_log_s(sd, mel, noise, sigma, cfg=synth.DEFAULT_WAVEGLOW_CONFIG):
    """max |log_s| per flow of one inverse pass (how strongly the synthetic `end` weights act)."""
    return _infer(sd, mel, noise, sigma, cfg)[1]


def waveglow_forward(sd, spect, audio, cfg=synth.DEFAULT_WAVEGLOW_CONFIG):
    """WaveGlow.forward (glow.py:196-245), the z direction: (spect [B, 80, F], audio [B, N]) -> (z [B, 8, N/8], log_s_list,
    log_det_W_list).  Computes in the dtype of sd and the inputs; differentiable in sd's tensors (either weight form)."""
    L, C, G = cfg["WN_config"]["n_layers"], cfg["WN_config"]["n_channels"], cfg["n_group"]
    B, N = audio.shape
    up = upsample(sd, spect, N)
    a = audio.unfold(1, G, G).permute(0, 2, 1)
    out, log_s_list, log_det_W_list = [], [], []
    for k in range(cfg["n_flows"]):
        if k % cfg["n_early_every"] == 0 and k > 0:
            out.append(a[:, :cfg["n_early_size"]])
            a = a[:, cfg["n_early_size"]:]
        W = sd[f"convinv.{k}.conv.weight"]
        a = F.conv1d(a, W)
        log_det_W_list.append(B * (N // G) * torch.logdet(W.squeeze(-1)))
        nh = a.size(1) // 2
        o = wn(sd, f"WN.{k}", a[:, :nh], up, L, C)
        log_s = o[:, nh:]
        a = torch.cat([a[:, :nh], torch.exp(log_s) * a[:, nh:] + o[:, :nh]], 1)
        log_s_list.append(log_s)
    out.append(a)
    return torch.cat(out, 1), log_s_list, log_det_W_list


def waveglow_loss(model_output, sigma=1.0):
    """WaveGlowLoss (glow.py:43-58)."""
    z, log_s_list, log_det_W_list = model_output
    loss = torch.sum(z * z) / (2 * sigma * sigma) - sum(torch.sum(s) for s in log_s_list) - sum(log_det_W_list)
    return loss / z.numel()
