"""CPU: the WaveGlow oracle against the reference-generated fixtures, the module's state_dict layout, argument checks."""
import json
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from flowtron_b200 import synth
from flowtron_b200._lib import FlowtronB200Error
from flowtron_b200.waveglow import WaveGlow, waveglow_flops

import waveglow_oracle as WO

CFG = synth.DEFAULT_WAVEGLOW_CONFIG


def _gold(tag):
    return dict(np.load(os.path.join(GOLDEN, f"waveglow_{tag}.npz")))


@pytest.mark.parametrize("tag", ["b1", "b2", "f96", "ragged"])
def test_oracle_matches_reference_goldens(tag):
    g = _gold(tag)
    seed, B, Fr = int(g["seed"]), int(g["B"]), int(g["F"])
    sd = synth.synth_waveglow_params(CFG, seed)
    lengths = g["lengths"].tolist() if "lengths" in g else None
    out = WO.waveglow_infer(sd, synth.synth_waveglow_mel(B, Fr, seed), synth.synth_waveglow_noise(B, Fr, seed), float(g["sigma"]),
                            CFG, lengths=lengths)
    ref = torch.from_numpy(g["audio"])
    err = (out - ref).abs().max().item() / ref.abs().max().item()
    assert err <= 1e-5, err
    if lengths is not None:
        assert (out[1, 256 * lengths[1]:] == 0).all()


def test_oracle_plain_weight_form_equals_weight_norm_form():
    sd = synth.synth_waveglow_params(CFG, 5)
    plain = {}
    for k, v in sd.items():
        if k.endswith("weight_g"):
            pre = k[: -len(".weight_g")]
            plain[pre + ".weight"] = WO.conv_weight(sd, pre)
        elif not k.endswith("weight_v"):
            plain[k] = v
    mel, z = synth.synth_waveglow_mel(1, 4, 5), synth.synth_waveglow_noise(1, 4, 5)
    a, b = WO.waveglow_infer(sd, mel, z, 0.6), WO.waveglow_infer(plain, mel, z, 0.6)
    assert (a - b).abs().max().item() <= 1e-5 * a.abs().max().item()


def test_synth_end_weights_make_log_s_act():
    sd = synth.synth_waveglow_params(CFG, 101)
    ls = WO.max_log_s(sd, synth.synth_waveglow_mel(1, 8, 101), synth.synth_waveglow_noise(1, 8, 101), 0.6)
    assert all(0.1 <= v <= 0.6 for v in ls.values()), ls


def test_synth_weight_norm_and_convinv_properties():
    sd = synth.synth_waveglow_params(CFG, 3)
    v, g = sd["WN.0.in_layers.0.weight_v"], sd["WN.0.in_layers.0.weight_g"]
    assert (v.flatten(1).norm(dim=1) - g.flatten()).abs().min() > 1.0          # the fold is not the identity
    for k in range(CFG["n_flows"]):
        W = sd[f"convinv.{k}.conv.weight"].squeeze(-1).double()
        assert torch.allclose(W @ W.T, torch.eye(W.shape[0], dtype=torch.float64), atol=1e-6)
        assert torch.det(W) > 0
    assert synth.synth_waveglow_params(CFG, 3)["WN.3.end.weight"].equal(sd["WN.3.end.weight"])


def test_state_dict_keys_and_shapes_match_reference_both_forms():
    with open(os.path.join(GOLDEN, "waveglow_keys.json")) as f:
        ref = json.load(f)
    m = WaveGlow(**CFG)
    assert {k: list(v.shape) for k, v in m.state_dict().items()} == ref["weight_norm"]
    assert {k: list(v) for k, v in synth.waveglow_param_shapes(CFG, True).items()} == ref["weight_norm"]
    assert {k: list(v) for k, v in synth.waveglow_param_shapes(CFG, False).items()} == ref["plain"]
    sd = synth.synth_waveglow_params(CFG, 9)
    m.load_state_dict(sd, strict=True)
    plain_model = WaveGlow.remove_weightnorm(m)
    plain = {k: v.clone() for k, v in plain_model.state_dict().items()}
    assert {k: list(v.shape) for k, v in plain.items()} == ref["plain"]
    m2 = WaveGlow.remove_weightnorm(WaveGlow(**CFG))
    m2.load_state_dict(plain, strict=True)
    # the folded weight is the oracle's g * v / |v|
    w = m2.WN[2].in_layers[5].weight.detach()
    assert torch.allclose(w, WO.conv_weight(sd, "WN.2.in_layers.5"), rtol=1e-5, atol=1e-7)


def test_cpu_tensors_raise():
    m = WaveGlow(**CFG)
    with pytest.raises(FlowtronB200Error):
        m.infer(torch.zeros(1, 80, 4))
    with pytest.raises(FlowtronB200Error):
        m.infer(torch.zeros(1, 80, 4), noise=torch.zeros(1, 8, 128))


def test_bad_noise_and_lengths_raise():
    m = WaveGlow(**CFG)
    x = torch.zeros(2, 80, 4)
    with pytest.raises(ValueError):
        m.infer(x, noise=torch.zeros(2, 8, 127))
    with pytest.raises(ValueError):
        m.infer(x, noise=torch.zeros(1, 8, 128))
    with pytest.raises(ValueError):
        m.infer(x, noise=torch.zeros(2, 4, 128))
    with pytest.raises(ValueError):
        m.infer(x, lengths=[4])
    with pytest.raises(ValueError):
        m.infer(x, lengths=[4, 5])
    with pytest.raises(ValueError):
        m.infer(x, lengths=[0, 4])
    with pytest.raises(ValueError):
        m.infer(torch.zeros(2, 40, 4))


@pytest.mark.parametrize("override", [dict(n_group=4), dict(WN_config=dict(n_layers=8, n_channels=512, kernel_size=3)),
                                      dict(WN_config=dict(n_layers=8, n_channels=256, kernel_size=5)),
                                      dict(WN_config=dict(n_layers=9, n_channels=256, kernel_size=3)),
                                      dict(n_mel_channels=100)])
def test_unsupported_configs_raise(override):
    with pytest.raises(NotImplementedError):
        WaveGlow(**dict(CFG, **override))


def test_forward_raises():
    with pytest.raises(NotImplementedError):
        WaveGlow(**CFG)((torch.zeros(1, 80, 4), torch.zeros(1, 1024)))


def test_flop_model():
    per_frame = waveglow_flops(1, CFG)
    assert abs((per_frame - 2 * 320 * 20480) / 1e9 - 5.186) < 1e-3
    assert abs(per_frame * 22050 / 256 / 1e9 - 447.8) < 1.0
