"""GPU: STFT.inverse / STFT.forward / griffin_lim (csrc/istft.cu) and the WaveGlow Denoiser against the reference-generated
fixtures (tests/make_golden_istft.py), ragged batches against B=1 runs, the Denoiser's bias and state_dict, CUDA-graph
replay and launch counts."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, record_parity
from flowtron_b200 import synth
from oracle import stft_oracle as S

import make_golden_istft as MG
from test_istft_host import istft_case_input

pytestmark = pytest.mark.gpu

WG_CFG = synth.DEFAULT_WAVEGLOW_CONFIG


def _rel(a, ref):
    a, ref = torch.as_tensor(a).double().cpu(), torch.as_tensor(ref).double().cpu()
    return (a - ref).abs().max().item() / ref.abs().max().item()


def _stft(hop, win=1024):
    from flowtron_b200.audio_processing import STFT
    return STFT(1024, hop, win).cuda()


@pytest.fixture(scope="module")
def waveglow():
    from flowtron_b200.waveglow import WaveGlow
    m = WaveGlow(**WG_CFG)
    m.load_state_dict(synth.synth_waveglow_params(WG_CFG, MG.DENOISER["wg_seed"]), strict=True)
    return m.cuda().eval()


@pytest.fixture(scope="module")
def denoiser(waveglow):
    """Denoiser with the fixture's bias_spec, loaded through a strict load_state_dict of the reference's layout."""
    from flowtron_b200.denoiser import Denoiser
    g = np.load(os.path.join(GOLDEN, "denoiser.npz"))
    d = Denoiser(waveglow)
    sd = d.state_dict()
    shapes = {k: tuple(int(x) for x in s if x) for k, s in zip(g["state_keys"].tolist(), g["state_shapes"])}
    assert {k: tuple(v.shape) for k, v in sd.items()} == shapes
    sd["bias_spec"] = torch.from_numpy(g["bias_spec"])
    d.load_state_dict(sd, strict=True)
    return d


@pytest.mark.parametrize("tag", list(MG.ISTFT_CASES))
def test_inverse_matches_reference_fixture(tag):
    from flowtron_b200 import _lib
    g = np.load(os.path.join(GOLDEN, "istft.npz"))
    mag, phase, hop, win = istft_case_input(tag)
    out = _stft(hop, win).inverse(mag.cuda(), phase.cuda())
    torch.cuda.synchronize()
    ref = torch.from_numpy(g[f"{tag}_out"])
    assert tuple(out.shape) == tuple(ref.shape)
    err = _rel(out, ref)
    record_parity(f"stft_inverse_{tag}", {"out": err})
    assert err <= 1e-4, err
    assert _lib.device_status() == 0


@pytest.mark.parametrize("hop", [128, 256, 512])
def test_forward_reconstructs_the_signal(hop):
    from flowtron_b200 import _lib
    y = synth.synth_istft_audio(3, 7001, 50 + hop).cuda()
    stft = _stft(hop)
    rec = stft(y)
    n = (y.shape[1] // hop) * hop
    assert tuple(rec.shape) == (3, 1, n)
    assert stft.magnitude.shape == (3, 513, 1 + y.shape[1] // hop)
    err = _rel(rec[:, 0], y[:, :n])
    record_parity(f"stft_forward_roundtrip_h{hop}", {"out": err})
    assert err <= 1e-5, err
    one = stft.inverse(stft.magnitude[:, :, :1], stft.phase[:, :, :1])
    assert tuple(one.shape) == (3, 1, 0)
    assert _lib.device_status() == 0


def test_ragged_packed_inverse_equals_single_runs():
    from flowtron_b200 import _lib
    hop = 256
    stft = _stft(hop)
    lens = [3000, 5213, 700, 4100, 2571]
    wavs = [synth.synth_istft_audio(1, n, 60 + i)[0].cuda() for i, n in enumerate(lens)]
    F = [1 + n // hop for n in lens]
    so = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int64, device="cuda")
    fo_h = np.concatenate([[0], np.cumsum(F)]).astype(np.int64)
    oo_h = np.concatenate([[0], np.cumsum([(f - 1) * hop for f in F])]).astype(np.int64)
    fo, oo = torch.from_numpy(fo_h).cuda(), torch.from_numpy(oo_h[:-1]).cuda()
    total = int(fo_h[-1])
    mag, ph = torch.empty(total * 513, device="cuda"), torch.empty(total * 513, device="cuda")
    _lib.stft_transform(torch.cat(wavs), so, fo, len(lens), total, stft._window, 1024, hop, mag, ph)
    outs = []
    for _ in range(2):
        out = torch.empty(int(oo_h[-1]), device="cuda")
        _lib.stft_inverse(mag, ph, fo, oo, len(lens), total, stft._window, 1024, hop, out)
        outs.append(out)
    assert torch.equal(outs[0], outs[1])
    for i, w in enumerate(wavs):
        single = stft.forward(w[None])[0, 0]
        assert torch.equal(outs[0][oo_h[i]:oo_h[i + 1]], single), i
    assert _lib.device_status() == 0


@pytest.mark.parametrize("n_iters", list(MG.GL["iters"]))
def test_griffin_lim_matches_reference_fixture(n_iters):
    from flowtron_b200 import _lib
    from flowtron_b200.audio_processing import griffin_lim
    g = np.load(os.path.join(GOLDEN, "griffin_lim.npz"))
    mag, _ = S.stft_transform(synth.synth_istft_audio(MG.GL["B"], MG.GL["N"], MG.GL["seed"]), 1024, MG.GL["hop"], 1024)
    np.random.seed(MG.GL["np_seed"])
    out = griffin_lim(mag.cuda(), _stft(MG.GL["hop"]), n_iters=n_iters)
    torch.cuda.synchronize()
    ref = torch.from_numpy(g[f"out_{n_iters}"])
    assert tuple(out.shape) == tuple(ref.shape)
    err = _rel(out, ref)
    record_parity(f"griffin_lim_{n_iters}", {"out": err})
    assert err <= 1e-3, err
    assert _lib.device_status() == 0


def test_denoiser_bias_matches_reference(waveglow):
    from flowtron_b200.denoiser import Denoiser
    g = np.load(os.path.join(GOLDEN, "denoiser.npz"))
    bias = Denoiser(waveglow).bias_spec
    assert tuple(bias.shape) == (1, 513, 1)
    err = _rel(bias, torch.from_numpy(g["bias_spec"]))
    record_parity("denoiser_bias_spec", {"bias": err})
    assert err <= 1e-3, err


def test_denoiser_matches_reference_fixture(denoiser):
    from flowtron_b200 import _lib
    g = np.load(os.path.join(GOLDEN, "denoiser.npz"))
    audio = torch.from_numpy(np.load(os.path.join(GOLDEN, MG.DENOISER["input"]))["audio"]).cuda()
    errs = {}
    for s in MG.DENOISER["strengths"]:
        out = denoiser(audio, s)
        ref = torch.from_numpy(g[f"out_{s}"])
        assert tuple(out.shape) == tuple(ref.shape)
        errs[f"strength_{s}"] = _rel(out, ref)
    torch.cuda.synchronize()
    record_parity("denoiser_forward", errs)
    assert max(errs.values()) <= 1e-4, errs
    assert _lib.device_status() == 0


def test_denoiser_ragged_rows_equal_single_runs(denoiser):
    from flowtron_b200 import _lib
    lengths = [256 * 40, 256 * 23, 256 * 31 + 77, 256 * 3]
    N = 256 * 41 + 13
    audio = synth.synth_istft_audio(len(lengths), N, 70).cuda()
    out = denoiser(audio, 0.3, lengths=lengths)
    assert tuple(out.shape) == (len(lengths), 1, (N // 256) * 256)
    assert torch.equal(out, denoiser(audio, 0.3, lengths=lengths))
    for b, n in enumerate(lengths):
        m = (n // 256) * 256
        single = denoiser(audio[b:b + 1, :n], 0.3)
        assert torch.equal(out[b, 0, :m], single[0, 0]), b
        assert (out[b, 0, m:] == 0).all(), b
    assert _lib.device_status() == 0


def test_denoiser_normal_mode_follows_cuda_generator(waveglow):
    from flowtron_b200.denoiser import Denoiser
    torch.cuda.manual_seed(5)
    a = Denoiser(waveglow, mode="normal").bias_spec
    torch.cuda.manual_seed(5)
    b = Denoiser(waveglow, mode="normal").bias_spec
    assert torch.equal(a, b)
    torch.cuda.manual_seed(5)
    mel = torch.randn((1, 80, 88), device="cuda")
    c = _stft(256).transform(waveglow.infer(mel, sigma=0.0))[0][:, :, :1]
    assert torch.equal(a, c)
    assert not torch.equal(a, Denoiser(waveglow).bias_spec)
    with pytest.raises(ValueError):
        Denoiser(waveglow, mode="uniform")


def _capture(fn):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = fn()
    graph.replay()
    torch.cuda.synchronize()
    return out


def test_denoiser_graph_replay_and_launch_count(denoiser):
    from flowtron_b200 import _lib
    audio = synth.synth_istft_audio(4, 256 * 60, 80).cuda()
    _lib.reset_launch_count()
    eager = denoiser(audio, 0.1)
    assert _lib.launch_count() == 2
    out = _capture(lambda: denoiser(audio, 0.1))
    assert torch.equal(out, eager)
    assert _lib.device_status() == 0


def test_griffin_lim_graph_replay_and_launch_count():
    from flowtron_b200 import _lib
    from flowtron_b200.audio_processing import griffin_lim
    stft = _stft(256)
    mag, _ = stft.transform(synth.synth_istft_audio(2, 256 * 40, 81).cuda())
    angles = ((torch.rand(mag.shape, generator=torch.Generator().manual_seed(3)) * 2 - 1) * np.pi).cuda()
    n = 5
    _lib.reset_launch_count()
    eager = griffin_lim(mag, stft, n, angles=angles)
    assert _lib.launch_count() == 1 + 2 * n
    out = _capture(lambda: griffin_lim(mag, stft, n, angles=angles))
    assert torch.equal(out, eager)
    assert _lib.device_status() == 0
