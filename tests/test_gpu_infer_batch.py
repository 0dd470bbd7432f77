"""GPU: Flowtron.infer_batch (ragged-batch inference over ft_ar_step_infer) against the reference-generated
fixtures (tests/make_golden_infer_batch.py), B = 1 and equal-length bit-identity with Flowtron.infer, a two-launch batch
against per-row B = 1 runs, padding invariance, CUDA-graph replay, and the chain into WaveGlow and the Denoiser."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, record_parity
from flowtron_b200 import synth

pytestmark = pytest.mark.gpu


def _model(n_flows, seed, n_speakers=1, gate_bias=None, gate_scale=1.0, use_gate=True):
    from flowtron_b200.flowtron import Flowtron
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=n_flows, n_speakers=n_speakers, use_gate_layer=use_gate)
    p = synth.synth_params(cfg, seed)
    if use_gate and gate_bias is not None:
        kb = [k for k in p if k.endswith("gate_layer.linear_layer.bias")][0]
        kw = [k for k in p if k.endswith("gate_layer.linear_layer.weight")][0]
        p[kb] = torch.full_like(p[kb], gate_bias)
        p[kw] = p[kw] * gate_scale
    m = Flowtron(**cfg)
    m.load_state_dict(p, strict=True)
    return m.cuda().eval()


def _batch(seed, B, T, L, n_speakers=1):
    g = torch.Generator().manual_seed(seed)
    res = (torch.randn(B, 80, T, generator=g) * 0.5).cuda()
    text = torch.randint(0, 185, (B, L), generator=g).cuda()
    spk = torch.randint(0, n_speakers, (B,), generator=g).cuda()
    return res, spk, text


def _single(m, res, spk, text, b, n_text, n_frames):
    mel, _ = m.infer(res[b:b + 1, :, :n_frames].contiguous(), spk[b:b + 1], text[b:b + 1, :n_text].contiguous())
    return mel[0]


def _check_attention(attn, n_flows, B, T, L, in_lens, mel_lens):
    assert len(attn) == n_flows
    for a in attn:
        assert tuple(a.shape) == (B, T, L)
        for b in range(B):
            n, k = int(mel_lens[b]), int(in_lens[b])
            assert (a[b, n:] == 0).all() and (a[b, :, k:] == 0).all()
            assert ((a[b, :n].sum(-1) - 1).abs() <= 1e-5).all()


@pytest.mark.parametrize("tag", ["f2", "f3", "t400"])
def test_infer_batch_matches_reference_fixtures(tag):
    from flowtron_b200 import _lib
    g = dict(np.load(os.path.join(GOLDEN, f"infer_ragged_{tag}.npz")))
    n_flows = int(g["cfg_n_flows"])
    m = _model(n_flows, int(g["seed"]), int(g["n_speakers"]), float(g["gate_bias"]), float(g["gate_scale"]))
    in_lens, max_frames = g["in_lens"].tolist(), g["max_frames"].tolist()
    B, T, L = len(in_lens), int(g["T"]), int(g["L"])
    with torch.no_grad():
        mel, mel_lens, attn = m.infer_batch(torch.from_numpy(g["residual"]).cuda(), torch.from_numpy(g["speaker_ids"]).cuda(),
                                            torch.from_numpy(g["text"]).cuda(), in_lens, max_frames=max_frames)
    torch.cuda.synchronize()
    assert _lib.device_status() == 0
    assert tuple(mel.shape) == (B, 80, T) and mel_lens.is_cuda and mel_lens.dtype == torch.int64
    assert mel_lens.cpu().tolist() == g["mel_lens"].tolist()
    ref = torch.from_numpy(g["mel"])
    errs = {}
    for b in range(B):
        n = int(g["mel_lens"][b])
        errs[f"row{b}"] = (mel[b, :, :n].cpu() - ref[b, :, :n]).abs().max().item() / ref[b, :, :n].abs().max().item()
        assert (mel[b, :, n:] == 0).all(), b
    print(f"infer_batch {tag}", mel_lens.tolist(), errs)
    record_parity(f"infer_batch_{tag}", errs)
    assert max(errs.values()) <= 1e-3, errs                 # north-star bar, per row
    _check_attention(attn, n_flows, B, T, L, in_lens, g["mel_lens"])


@pytest.mark.parametrize("n_flows", [2, 3])
@pytest.mark.parametrize("use_gate", [False, True])
def test_b1_is_bit_identical_to_infer(n_flows, use_gate):
    m = _model(n_flows, 61 + n_flows, gate_bias=-0.3 if n_flows == 2 else -6.0, gate_scale=40.0, use_gate=use_gate)
    res, spk, text = _batch(5, 1, 40, 17)
    with torch.no_grad():
        ref, _ = m.infer(res, spk, text)
        mel, mel_lens, _ = m.infer_batch(res, spk, text, [17])
    n = ref.shape[-1]
    assert mel_lens.tolist() == [n]
    assert torch.equal(mel[..., :n], ref)
    assert (mel[..., n:] == 0).all()


def test_equal_length_batch_is_bit_identical_to_infer():
    m = _model(2, 23, use_gate=False)
    res, spk, text = _batch(6, 4, 32, 14)
    with torch.no_grad():
        ref, ref_attn = m.infer(res, spk, text)
        mel, mel_lens, attn = m.infer_batch(res, spk, text, [14] * 4, max_frames=[32] * 4)
    assert mel_lens.tolist() == [32] * 4
    assert torch.equal(mel, ref)
    for a, r in zip(attn, ref_attn):
        assert torch.equal(a, torch.cat(r, 1))


def test_wide_ragged_batch_rows_equal_single_runs():
    """B = 20 (two launches of 16 + 4): every row equals its own B = 1 infer on the unpadded inputs."""
    from flowtron_b200 import _lib
    m = _model(2, 61, gate_bias=-0.3, gate_scale=40.0)
    B, T, L = 20, 40, 24
    res, spk, text = _batch(7, B, T, L)
    g = torch.Generator().manual_seed(8)
    in_lens = torch.randint(3, L + 1, (B,), generator=g).tolist()
    max_frames = torch.randint(8, T + 1, (B,), generator=g).tolist()
    with torch.no_grad():
        mel, mel_lens, attn = m.infer_batch(res, spk, text, in_lens, max_frames=max_frames)
        singles = [_single(m, res, spk, text, b, in_lens[b], max_frames[b]) for b in range(B)]
    torch.cuda.synchronize()
    assert _lib.device_status() == 0
    lens = mel_lens.tolist()
    assert lens == [s.shape[-1] for s in singles], (lens, max_frames)
    errs = {}
    for b, s in enumerate(singles):
        n = lens[b]
        errs[f"row{b}"] = (mel[b, :, :n] - s).abs().max().item() / s.abs().max().item()
        assert (mel[b, :, n:] == 0).all(), b
    record_parity("infer_batch_b20", errs)
    assert max(errs.values()) <= 2e-3, errs
    stopped = sum(n < f for n, f in zip(lens, max_frames))
    assert 0 < stopped < B, (lens, max_frames)             # both gate stops and budget runs are covered
    _check_attention(attn, 2, B, T, L, in_lens, lens)


def test_padding_is_never_used():
    m = _model(3, 62, n_speakers=3, gate_bias=-6.0, gate_scale=40.0)
    B, T, L = 6, 36, 20
    res, spk, text = _batch(9, B, T, L, n_speakers=3)
    in_lens, max_frames = [20, 4, 13, 9, 17, 11], [36, 12, 30, 21, 25, 33]
    g = torch.Generator().manual_seed(10)
    res2, text2 = res.clone(), text.clone()
    for b in range(B):
        res2[b, :, max_frames[b]:] = torch.randn(80, T - max_frames[b], generator=g).cuda() * 3
        text2[b, in_lens[b]:] = torch.randint(0, 185, (L - in_lens[b],), generator=g).cuda()
    assert not torch.equal(res, res2) and not torch.equal(text, text2)
    with torch.no_grad():
        a = m.infer_batch(res, spk, text, in_lens, max_frames=max_frames)
        b = m.infer_batch(res2, spk, text2, torch.tensor(in_lens), max_frames=torch.tensor(max_frames))
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    for x, y in zip(a[2], b[2]):
        assert torch.equal(x, y)


def test_cuda_graph_replay_equals_eager():
    m = _model(2, 61, gate_bias=-0.3, gate_scale=40.0)
    B, T, L = 5, 30, 16
    res, spk, text = _batch(11, B, T, L)
    in_lens = torch.tensor([16, 5, 11, 8, 14], device="cuda")
    max_frames = torch.tensor([30, 12, 25, 18, 9], device="cuda")
    new_res, _, _ = _batch(12, B, T, L)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.no_grad():
        with torch.cuda.stream(s):
            m.infer_batch(res, spk, text, in_lens, max_frames=max_frames)        # warm-up: scratch buffers exist before capture
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            mel_g, lens_g, attn_g = m.infer_batch(res, spk, text, in_lens, max_frames=max_frames)
        res.copy_(new_res)
        graph.replay()
        torch.cuda.synchronize()
        mel_e, lens_e, attn_e = m.infer_batch(new_res, spk, text, in_lens, max_frames=max_frames)
    assert torch.equal(lens_g, lens_e)
    assert torch.equal(mel_g, mel_e)
    for x, y in zip(attn_g, attn_e):
        assert torch.equal(x, y)


def test_end_to_end_into_waveglow_and_denoiser():
    """infer_batch -> WaveGlow.infer(lengths=) -> Denoiser(lengths=): every row equals the same chain at B = 1."""
    from flowtron_b200 import _lib
    from flowtron_b200.denoiser import Denoiser
    from flowtron_b200.waveglow import WaveGlow
    wcfg = synth.DEFAULT_WAVEGLOW_CONFIG
    wg = WaveGlow(**wcfg)
    wg.load_state_dict(synth.synth_waveglow_params(wcfg, 14), strict=True)
    wg = wg.cuda().eval()
    den = Denoiser(wg)
    m = _model(2, 61, gate_bias=-0.3, gate_scale=40.0)
    B, T, L = 4, 36, 18
    res, spk, text = _batch(13, B, T, L)
    in_lens, max_frames = [18, 6, 12, 15], [36, 20, 28, 14]
    noise = synth.synth_waveglow_noise(B, T, 15).cuda()
    sigma = 0.6
    with torch.no_grad():
        mel, mel_lens, _ = m.infer_batch(res, spk, text, in_lens, max_frames=max_frames)
        lens = mel_lens.tolist()
        audio = wg.infer(mel.contiguous(), sigma=sigma, noise=noise, lengths=lens)
        clean = den(audio, 0.1, lengths=[256 * n for n in lens])
        errs = {}
        for b, n in enumerate(lens):
            assert (audio[b, 256 * n:] == 0).all() and (clean[b, 0, 256 * n:] == 0).all(), b
            mel1 = _single(m, res, spk, text, b, in_lens[b], max_frames[b])
            assert mel1.shape[-1] == n
            a1 = wg.infer(mel1[None].contiguous(), sigma=sigma, noise=noise[b:b + 1, :, :32 * n].contiguous())
            c1 = den(a1, 0.1)
            errs[f"mel{b}"] = (mel[b, :, :n] - mel1).abs().max().item() / mel1.abs().max().item()
            errs[f"audio{b}"] = (audio[b, :256 * n] - a1[0]).abs().max().item() / a1.abs().max().item()
            errs[f"denoised{b}"] = (clean[b, 0, :256 * n] - c1[0, 0]).abs().max().item() / c1.abs().max().item()
    torch.cuda.synchronize()
    assert _lib.device_status() == 0
    record_parity("infer_batch_to_audio", errs)
    assert max(v for k, v in errs.items() if k.startswith("mel")) <= 2e-3, errs
    assert max(v for k, v in errs.items() if not k.startswith("mel")) <= 1e-3, errs
