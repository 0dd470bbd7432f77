"""GPU: WaveGlow.infer (csrc/waveglow.cu) against the reference-generated fixtures, ragged batches, both weight forms, the
noise contract, CUDA-graph replay and launch count."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, record_parity
from flowtron_b200 import synth

pytestmark = pytest.mark.gpu

CFG = synth.DEFAULT_WAVEGLOW_CONFIG


def _model(seed, plain=False):
    from flowtron_b200.waveglow import WaveGlow
    m = WaveGlow(**CFG)
    m.load_state_dict(synth.synth_waveglow_params(CFG, seed), strict=True)
    if plain:
        m = WaveGlow.remove_weightnorm(m)
    return m.cuda().eval()


def _inputs(g):
    seed, B, Fr = int(g["seed"]), int(g["B"]), int(g["F"])
    return synth.synth_waveglow_mel(B, Fr, seed).cuda(), synth.synth_waveglow_noise(B, Fr, seed).cuda()


def _rel(a, b):
    return (a.cpu() - b.cpu()).abs().max().item() / b.abs().max().item()


@pytest.mark.parametrize("tag", ["b1", "b2", "f96"])
def test_waveglow_matches_reference_goldens(tag):
    from flowtron_b200 import _lib
    g = dict(np.load(os.path.join(GOLDEN, f"waveglow_{tag}.npz")))
    m = _model(int(g["seed"]))
    mel, z = _inputs(g)
    audio = m.infer(mel, sigma=float(g["sigma"]), noise=z)
    torch.cuda.synchronize()
    assert _lib.device_status() == 0
    ref = torch.from_numpy(g["audio"])
    assert tuple(audio.shape) == tuple(ref.shape)
    err = _rel(audio, ref)
    print(f"waveglow {tag} rel err {err:.3e}")
    record_parity(f"waveglow_{tag}", {"audio": err})
    assert err <= 1e-3, err


def test_waveglow_ragged_rows_equal_single_runs():
    g = dict(np.load(os.path.join(GOLDEN, "waveglow_ragged.npz")))
    lengths = g["lengths"].tolist()
    m = _model(int(g["seed"]))
    mel, z = _inputs(g)
    sigma = float(g["sigma"])
    audio = m.infer(mel, sigma=sigma, noise=z, lengths=lengths)
    ref = torch.from_numpy(g["audio"])
    errs = {}
    for b, n in enumerate(lengths):
        errs[f"row{b}"] = _rel(audio[b, :256 * n], ref[b, :256 * n])
        assert errs[f"row{b}"] <= 1e-3, errs
        assert (audio[b, 256 * n:] == 0).all()
        single = m.infer(mel[b:b + 1, :, :n].contiguous(), sigma=sigma, noise=z[b:b + 1, :, :32 * n].contiguous())
        errs[f"row{b}_vs_b1"] = _rel(audio[b, :256 * n], single[0])
        assert errs[f"row{b}_vs_b1"] <= 1e-6, errs
    record_parity("waveglow_ragged", errs)


def test_weight_norm_and_plain_forms_agree():
    mel, z = synth.synth_waveglow_mel(1, 16, 8).cuda(), synth.synth_waveglow_noise(1, 16, 8).cuda()
    a = _model(8).infer(mel, sigma=0.6, noise=z)
    b = _model(8, plain=True).infer(mel, sigma=0.6, noise=z)
    err = _rel(a, b)
    record_parity("waveglow_weight_forms", {"audio": err})
    assert err <= 1e-6, err


def test_default_noise_is_reproducible_and_follows_draw_order():
    m = _model(12)
    B, Fr, Tg = 2, 8, 256
    mel = synth.synth_waveglow_mel(B, Fr, 12).cuda()
    torch.cuda.manual_seed(77)
    a = m.infer(mel, sigma=0.7)
    torch.cuda.manual_seed(77)
    b = m.infer(mel, sigma=0.7)
    assert torch.equal(a, b)
    torch.cuda.manual_seed(77)                                 # the reference's draws: initial, then after flow 8, flow 4
    z = torch.zeros(B, 8, Tg, device="cuda")
    z[:, 4:8] = torch.randn(B, 4, Tg, device="cuda")
    z[:, 2:4] = torch.randn(B, 2, Tg, device="cuda")
    z[:, 0:2] = torch.randn(B, 2, Tg, device="cuda")
    c = m.infer(mel, sigma=0.7, noise=z)
    assert torch.equal(a, c)


def test_cuda_graph_replay_equals_eager_and_launch_count():
    from flowtron_b200 import _lib
    m = _model(13)
    mel, z = synth.synth_waveglow_mel(2, 12, 13).cuda(), synth.synth_waveglow_noise(2, 12, 13).cuda()
    _lib.reset_launch_count()
    eager = m.infer(mel, sigma=0.6, noise=z)
    launches = _lib.launch_count()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        m.infer(mel, sigma=0.6, noise=z)                       # warm the capture stream's scratch
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = m.infer(mel, sigma=0.6, noise=z)
    graph.replay()
    torch.cuda.synchronize()
    assert _lib.device_status() == 0
    assert torch.equal(out, eager)
    assert launches <= CFG["n_flows"] * (2 * CFG["WN_config"]["n_layers"] + 1) + 4, launches
