"""CPU: the differentiable WaveGlow oracle (tests/waveglow_oracle.py) pinned against the reference-generated training
fixture (tests/make_golden_waveglow_train.py), WaveGlowLoss, and the argument checks of WaveGlow.forward."""
import os

import numpy as np
import pytest
import torch

import waveglow_oracle as O
from conftest import GOLDEN
from flowtron_b200 import synth
from make_golden_waveglow_train import REDUCED_CONFIG, inputs

G = dict(np.load(os.path.join(GOLDEN, "waveglow_train.npz")))


def _rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return ((a - b).norm() / b.norm()).item()


def test_oracle_forward_matches_reference_fixture():
    cfg = synth.DEFAULT_WAVEGLOW_CONFIG
    sd = synth.synth_waveglow_params(cfg, int(G["fwd_seed"]))
    spect, audio = inputs(int(G["fwd_B"]), int(G["fwd_N"]), int(G["fwd_input_seed"]))
    with torch.no_grad():
        z, log_s, log_det = O.waveglow_forward(sd, spect, audio, cfg)
        loss = O.waveglow_loss((z, log_s, log_det), float(G["sigma"]))
    assert _rel(z, G["fwd_z"]) < 1e-5
    for k, t in enumerate(log_s):
        assert _rel(t, G[f"fwd_log_s_{k}"]) < 1e-5, k
    # orthonormal W: logdet is rounding noise times B N / 8 in both runs
    assert (torch.stack(log_det) - torch.from_numpy(G["fwd_log_det_W"])).abs().max().item() < 5e-4
    assert abs(float(loss) - float(G["fwd_loss"])) < 1e-5 * abs(float(G["fwd_loss"]))


def test_oracle_gradients_match_reference_fixture():
    sd = {k: v.requires_grad_(True) for k, v in synth.synth_waveglow_params(REDUCED_CONFIG, int(G["grad_seed"])).items()}
    spect, audio = inputs(int(G["grad_B"]), int(G["grad_N"]), int(G["grad_input_seed"]))
    loss = O.waveglow_loss(O.waveglow_forward(sd, spect, audio, REDUCED_CONFIG), float(G["sigma"]))
    loss.backward()
    assert abs(loss.item() - float(G["grad_loss"])) < 1e-5 * abs(float(G["grad_loss"]))
    names = [str(n) for n in G["grad_names"]]
    assert sorted(names) == sorted(sd)
    for name in names:
        g = sd[name].grad
        ref_norm = float(G[f"grad_norm/{name}"])
        assert abs(g.norm().item() - ref_norm) <= 1e-4 * ref_norm + 1e-12, name
        got = g.flatten()[torch.from_numpy(G[f"grad_idx/{name}"])]
        assert (got - torch.from_numpy(G[f"grad_val/{name}"])).abs().max().item() <= 1e-4 * ref_norm + 1e-12, name


def test_loss_matches_oracle():
    from flowtron_b200.waveglow import WaveGlowLoss
    g = torch.Generator().manual_seed(3)
    z = torch.randn(2, 8, 40, generator=g)
    log_s = [torch.randn(2, 4, 40, generator=g), torch.randn(2, 3, 40, generator=g)]
    log_det = [torch.tensor(0.3), torch.tensor(-1.2)]
    a = WaveGlowLoss(0.6)((z, log_s, log_det))
    b = O.waveglow_loss((z, log_s, log_det), 0.6)
    assert torch.allclose(a, b, rtol=1e-6, atol=0)


def _model():
    from flowtron_b200.waveglow import WaveGlow
    return WaveGlow(**synth.DEFAULT_WAVEGLOW_CONFIG)


@pytest.mark.parametrize("spect_shape, audio_shape", [
    ((2, 80), (2, 2048)),           # spect not 3-D
    ((2, 81, 9), (2, 2048)),        # wrong mel channels
    ((2, 80, 9), (2, 8, 256)),      # audio not 2-D
    ((2, 80, 9), (3, 2048)),        # batch mismatch
    ((0, 80, 9), (0, 2048)),        # empty batch
    ((2, 80, 9), (2, 2044)),        # N % 8
    ((2, 80, 9), (2, 0)),           # N = 0
    ((2, 80, 8), (2, 2056)),        # N > 256 F
])
def test_forward_argument_checks(spect_shape, audio_shape):
    with pytest.raises(ValueError):
        _model()((torch.zeros(spect_shape), torch.zeros(audio_shape)))


def test_forward_rejects_inputs_that_require_grad():
    with pytest.raises(ValueError):
        _model()((torch.zeros(2, 80, 9, requires_grad=True), torch.zeros(2, 2048)))
    with pytest.raises(ValueError):
        _model()((torch.zeros(2, 80, 9), torch.zeros(2, 2048, requires_grad=True)))


def test_forward_on_cpu_tensors_raises():
    from flowtron_b200._lib import FlowtronB200Error
    with pytest.raises(FlowtronB200Error):
        _model()((torch.zeros(2, 80, 9), torch.zeros(2, 2048)))
    with pytest.raises(NotImplementedError):        # there is no CPU implementation of training
        _model()((torch.zeros(2, 80, 9), torch.zeros(2, 2048)))


def test_forward_accepts_n_up_to_256_f_and_rejects_past_the_batch_limit():
    with pytest.raises(ValueError):
        _model()((torch.zeros(129, 80, 9), torch.zeros(129, 2048)))
    from flowtron_b200._lib import FlowtronB200Error
    with pytest.raises(FlowtronB200Error):          # N = 256 F passes the checks and then needs CUDA
        _model()((torch.zeros(1, 80, 8), torch.zeros(1, 2048)))
