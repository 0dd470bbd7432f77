"""fp64-capable, differentiable restatement of WaveGlow.forward and WaveGlowLoss (tacotron2/waveglow/glow.py:43-58,
196-245), written from the math: the checker of flowtron_b200.waveglow's training direction.  Computes in the dtype of its
weights and inputs (fp64 weights give an fp64 oracle) and takes a state_dict in either weight-norm or plain-weight form."""
from __future__ import annotations

import torch
import torch.nn.functional as F

from flowtron_b200 import synth


def _weight(sd, pre):
    """Effective weight of conv `pre` in the dtype of sd: g * v / |v| (norm over all dims but 0) in weight-norm form, else
    `weight`; differentiable in sd's tensors."""
    if f"{pre}.weight_g" in sd:
        v, g = sd[f"{pre}.weight_v"], sd[f"{pre}.weight_g"]
        return v * (g / v.flatten(1).norm(dim=1).view(-1, 1, 1))
    return sd[f"{pre}.weight"]


def _wn_forward(sd, pre, audio0, spect, n_layers, C):
    def conv(name, x, **kw):
        return F.conv1d(x, _weight(sd, f"{pre}.{name}"), sd[f"{pre}.{name}.bias"], **kw)

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


def waveglow_forward(sd, spect, audio, cfg=synth.DEFAULT_WAVEGLOW_CONFIG):
    """WaveGlow.forward (glow.py:196-245), the z direction: (spect [B, 80, F], audio [B, N]) -> (z [B, 8, N/8], log_s_list,
    log_det_W_list).  Computes in the dtype of sd and the inputs; differentiable in sd's tensors (either weight form)."""
    L, C, G = cfg["WN_config"]["n_layers"], cfg["WN_config"]["n_channels"], cfg["n_group"]
    B, N = audio.shape
    up = F.conv_transpose1d(spect, sd["upsample.weight"], sd["upsample.bias"], stride=256)[:, :, :N]
    up = up.unfold(2, G, G).permute(0, 2, 1, 3).reshape(B, N // G, -1).permute(0, 2, 1)
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
        o = _wn_forward(sd, f"WN.{k}", a[:, :nh], up, L, C)
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
