"""GPU: voice conversion and rhythm transfer -- Flowtron.encode(return_attns=True), Flowtron.infer_aligned (over
ft_ar_step_infer with forced alignments) and Flowtron.convert against the reference-generated fixtures (tests/make_golden_convert.py), a
two-launch batch against per-row B = 1 Flowtron.infer(attns=) runs, the identity conversion, padding invariance, CUDA-graph
replay and the chain into WaveGlow and the Denoiser."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, record_parity
from flowtron_b200 import synth

pytestmark = pytest.mark.gpu


def _model(n_flows, seed, n_speakers=2, gate_bias=-10.0):
    from flowtron_b200.flowtron import Flowtron
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=n_flows, n_speakers=n_speakers)
    p = synth.synth_params(cfg, seed)
    kb = [k for k in p if k.endswith("gate_layer.linear_layer.bias")][0]
    p[kb] = torch.full_like(p[kb], gate_bias)
    m = Flowtron(**cfg)
    m.load_state_dict(p, strict=True)
    return m.cuda().eval()


def _fixture(tag):
    g = dict(np.load(os.path.join(GOLDEN, f"convert_{tag}.npz")))
    m = _model(int(g["cfg_n_flows"]), int(g["seed"]), int(g["n_speakers"]), float(g["gate_bias"]))
    return g, m, (lambda k: torch.from_numpy(g[k]).cuda())


def _mels(seed, B, T):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(B, 80, T, generator=g) * 2.0 - 5.5).clamp_(-11.5, 2.0).cuda()


def _alignments(seed, n_flows, B, T, L, in_lens, fill=0.0):
    """Random attention maps [B, T, L] per flow: rows sum to 1 over each utterance's own tokens, `fill` past them."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n_flows):
        a = torch.full((B, T, L), fill)
        for b, n in enumerate(in_lens):
            a[b, :, :n] = torch.softmax(3.0 * torch.randn(T, n, generator=g), -1)
        out.append(a.cuda())
    return out


def _row_errs(x, ref, lens):
    errs = {}
    for b, n in enumerate(lens):
        errs[f"row{b}"] = (x[b, :, :n] - ref[b, :, :n]).abs().max().item() / ref[b, :, :n].abs().max().item()
        assert (x[b, :, n:] == 0).all(), b
    return errs


@pytest.mark.parametrize("tag", ["f2", "f3", "long"])
def test_encode_returns_the_reference_alignments(tag):
    from flowtron_b200 import _lib
    g, m, t = _fixture(tag)
    in_lens, out_lens = g["in_lens"].tolist(), g["out_lens"].tolist()
    z0 = m.encode(t("mel"), t("speaker_ids"), t("text"), in_lens, out_lens)
    z, attns = m.encode(t("mel"), t("speaker_ids"), t("text"), in_lens, out_lens, return_attns=True)
    torch.cuda.synchronize()
    assert _lib.device_status() == 0
    assert torch.equal(z, z0)
    B, _, T = g["mel"].shape
    assert len(attns) == int(g["cfg_n_flows"])
    errs = {}
    for f, a in enumerate(attns):
        assert tuple(a.shape) == (B, T, g["text"].shape[1])
        for b in range(B):
            assert (a[b, out_lens[b]:] == 0).all() and (a[b, :, in_lens[b]:] == 0).all()
        errs[f"attn{f}"] = (a - t(f"attn_{f}")).abs().max().item()
    errs["z"] = (z - t("z")).abs().max().item() / float(np.abs(g["z"]).max())
    record_parity(f"convert_encode_{tag}", errs)
    assert max(errs.values()) <= 2e-3, errs


@pytest.mark.parametrize("tag", ["f2", "f3", "long"])
def test_convert_and_infer_aligned_match_reference_fixtures(tag):
    from flowtron_b200 import _lib
    g, m, t = _fixture(tag)
    in_lens, out_lens = g["in_lens"].tolist(), g["out_lens"].tolist()
    ref_attns = [t(f"attn_{f}") for f in range(int(g["cfg_n_flows"]))]
    conv = m.convert(t("mel"), t("speaker_ids"), t("target_speaker_ids"), t("text"), in_lens, out_lens)
    mel, mel_lens = m.infer_aligned(t("z"), t("target_speaker_ids"), t("text"), in_lens, ref_attns, out_lens)
    torch.cuda.synchronize()
    assert _lib.device_status() == 0
    assert mel_lens.dtype == torch.int64 and mel_lens.tolist() == out_lens
    assert conv.shape == mel.shape == g["mel"].shape
    errs = {f"convert_{k}": v for k, v in _row_errs(conv, t("mel_converted"), out_lens).items()}
    errs.update({f"aligned_{k}": v for k, v in _row_errs(mel, t("mel_converted"), out_lens).items()})
    if "mel_rhythm" in g:                                        # rhythm transfer: a sampled z under the recording's timing
        rhy, _ = m.infer_aligned(t("noise"), t("target_speaker_ids"), t("text"), in_lens, ref_attns, out_lens)
        errs.update({f"rhythm_{k}": v for k, v in _row_errs(rhy, t("mel_rhythm"), out_lens).items()})
    print(f"convert {tag}", errs)
    record_parity(f"convert_{tag}", errs)
    assert max(errs.values()) <= 2e-3, errs


@pytest.mark.parametrize("L", [24, 300])
def test_wide_batch_rows_equal_single_infer_with_attns(L):
    """B = 20 (launches of 16 + 4), three flows: every row equals its own B = 1 Flowtron.infer(attns=) on unpadded inputs."""
    from flowtron_b200 import _lib
    m = _model(3, 62, n_speakers=3)
    B, T = 20, (40 if L <= 256 else 10)
    g = torch.Generator().manual_seed(L)
    res = (torch.randn(B, 80, T, generator=g) * 0.5).cuda()
    text = torch.randint(0, 185, (B, L), generator=g).cuda()
    spk = torch.randint(0, 3, (B,), generator=g).cuda()
    in_lens = torch.randint(3, L + 1, (B,), generator=g).tolist()
    n_frames = torch.randint(4, T + 1, (B,), generator=g).tolist()
    in_lens[5], n_frames[17] = L, T
    attns = _alignments(L + 1, 3, B, T, L, in_lens)
    mel, mel_lens = m.infer_aligned(res, spk, text, in_lens, attns, n_frames)
    with torch.no_grad():
        singles = [m.infer(res[b:b + 1, :, :n_frames[b]].contiguous(), spk[b:b + 1], text[b:b + 1, :in_lens[b]].contiguous(),
                           gate_threshold=1.0, attns=[a[b, :n_frames[b], :in_lens[b]] for a in attns])[0][0] for b in range(B)]
    torch.cuda.synchronize()
    assert _lib.device_status() == 0
    assert mel_lens.tolist() == n_frames == [s.shape[-1] for s in singles]
    errs = {}
    for b, s in enumerate(singles):
        errs[f"row{b}"] = (mel[b, :, :n_frames[b]] - s).abs().max().item() / s.abs().max().item()
        assert (mel[b, :, n_frames[b]:] == 0).all(), b
    errs["rows_bit_identical"] = sum(v == 0.0 for v in errs.values())
    print(f"infer_aligned B=20 L={L}", errs)
    record_parity(f"infer_aligned_b20_L{L}", errs)
    assert max(v for k, v in errs.items() if k.startswith("row") and k != "rows_bit_identical") <= 2e-3, errs


def test_encode_attns_through_the_short_and_long_row_split():
    """Host out_lens on both sides of the 320-frame split: each group's maps are scattered back to their rows and equal the
    row's own B = 1 forward."""
    m = _model(2, 81)
    in_lens, out_lens = [12, 20, 7], [40, 330, 25]
    B, T, L = 3, 330, 20
    mel = _mels(5, B, T)
    g = torch.Generator().manual_seed(6)
    text = torch.randint(0, 185, (B, L), generator=g).cuda()
    spk = torch.tensor([1, 0, 1], device="cuda")
    z, attns = m.encode(mel, spk, text, in_lens, out_lens, return_attns=True)
    assert torch.equal(z, m.encode(mel, spk, text, in_lens, out_lens))
    errs = {}
    with torch.no_grad():
        for b in range(B):
            nl, nt = in_lens[b], out_lens[b]
            out = m(mel[b:b + 1, :, :nt].contiguous(), spk[b:b + 1], text[b:b + 1, :nl].contiguous(),
                    torch.tensor([nl], device="cuda"), torch.tensor([nt], device="cuda"))
            assert torch.equal(z[b, :, :nt], out[0].permute(1, 2, 0)[0]), b
            for f, a in enumerate(attns):
                errs[f"row{b}_attn{f}"] = (a[b, :nt, :nl] - out[3][f][0]).abs().max().item()
                assert (a[b, nt:] == 0).all() and (a[b, :, nl:] == 0).all()
    record_parity("convert_encode_split", errs)
    assert max(errs.values()) <= 1e-6, errs


def test_identity_conversion_returns_the_mel():
    from flowtron_b200 import _lib
    m = _model(3, 82, n_speakers=3)
    in_lens, out_lens = [15, 22, 9, 18, 22], [70, 44, 96, 31, 58]
    B, T, L = 5, 96, 22
    mel = _mels(7, B, T)
    g = torch.Generator().manual_seed(8)
    text = torch.randint(0, 185, (B, L), generator=g).cuda()
    spk = torch.tensor([2, 0, 1, 1, 0], device="cuda")
    back = m.convert(mel, spk, spk, text, in_lens, out_lens)
    other = m.convert(mel, spk, (spk + 1) % 3, text, in_lens, out_lens)
    torch.cuda.synchronize()
    assert _lib.device_status() == 0
    errs = _row_errs(back, mel, out_lens)
    record_parity("convert_identity", errs)
    assert max(errs.values()) <= 2e-3, errs
    for b, n in enumerate(out_lens):                             # another voice: another mel, same length
        assert (other[b, :, :n] - mel[b, :, :n]).abs().max().item() > 0.05 and (other[b, :, n:] == 0).all()


def test_flow_infer_ragged_attention_out_is_the_forced_alignment():
    """Per flow: the returned attention is the given map, in generation order, masked to each row's lengths."""
    m = _model(2, 81)
    B, T, L = 4, 30, 16
    in_lens, n_frames = [16, 5, 11, 8], [30, 12, 25, 18]
    g = torch.Generator().manual_seed(9)
    res = (torch.randn(T, B, 80, generator=g) * 0.5).cuda()
    text = (torch.randn(L, B, 640, generator=g) * 0.3).cuda()
    il, fl = torch.tensor(in_lens, dtype=torch.int32, device="cuda"), torch.tensor(n_frames, dtype=torch.int32, device="cuda")
    attns = _alignments(10, 2, B, T, L, in_lens, fill=0.25)
    text2 = text.clone()
    text2[:, :, 512:] += 0.1                                     # the speaker part of the encoding
    for flow, a in zip(m.flows, attns):
        out, attn, n = flow.infer_ragged(res, text, il, fl, attns=a)
        out2, attn2, _ = flow.infer_ragged(res, text2, il, fl, attns=a)
        assert n.tolist() == n_frames
        want = a.transpose(0, 1).clone()
        for b in range(B):
            want[n_frames[b]:, b] = 0
            want[:, b, in_lens[b]:] = 0
        assert torch.equal(attn, want) and torch.equal(attn2, want)
        assert not torch.equal(out, out2)


def test_padding_is_never_used():
    m = _model(3, 82, n_speakers=3)
    B, T, L = 6, 36, 20
    in_lens, n_frames = [20, 4, 13, 9, 17, 11], [36, 12, 30, 21, 25, 33]
    g = torch.Generator().manual_seed(11)
    res = (torch.randn(B, 80, T, generator=g) * 0.5).cuda()
    text = torch.randint(0, 185, (B, L), generator=g).cuda()
    spk = torch.randint(0, 3, (B,), generator=g).cuda()
    attns = _alignments(12, 3, B, T, L, in_lens)
    res2, text2, attns2 = res.clone(), text.clone(), [a.clone() for a in attns]
    for b in range(B):
        res2[b, :, n_frames[b]:] = 7.0
        text2[b, in_lens[b]:] = torch.randint(0, 185, (L - in_lens[b],), generator=g).cuda()
        for a in attns2:
            a[b, :, in_lens[b]:] = float("nan")
            a[b, n_frames[b]:] = float("inf")
    x = m.infer_aligned(res, spk, text, in_lens, attns, n_frames)
    y = m.infer_aligned(res2, spk, text2, torch.tensor(in_lens), attns2, torch.tensor(n_frames))
    assert torch.isfinite(y[0]).all()
    assert torch.equal(x[0], y[0]) and torch.equal(x[1], y[1])
    # convert: mel frames past out_lens and text padding
    mel = _mels(13, B, T)
    mel2 = mel.clone()
    for b in range(B):
        mel2[b, :, n_frames[b]:] = 3.0
    tgt = (spk + 1) % 3
    assert torch.equal(m.convert(mel, spk, tgt, text, in_lens, n_frames), m.convert(mel2, spk, tgt, text2, in_lens, n_frames))


def test_convert_cuda_graph_replay_equals_eager():
    m = _model(2, 81)
    B, T, L = 5, 30, 16
    g = torch.Generator().manual_seed(14)
    text = torch.randint(0, 185, (B, L), generator=g).cuda()
    spk = torch.tensor([0, 1, 1, 0, 1], device="cuda")
    tgt = 1 - spk
    in_lens = torch.tensor([16, 5, 11, 8, 14], device="cuda")
    out_lens = torch.tensor([30, 12, 25, 18, 9], device="cuda")
    mel, new_mel = _mels(15, B, T), _mels(16, B, T)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        m.convert(mel, spk, tgt, text, in_lens, out_lens)        # warm-up: scratch buffers exist before capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out_g = m.convert(mel, spk, tgt, text, in_lens, out_lens)
    mel.copy_(new_mel)
    graph.replay()
    torch.cuda.synchronize()
    out_e = m.convert(new_mel, spk, tgt, text, in_lens, out_lens)
    assert torch.equal(out_g, out_e)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out_g, out_e)


def test_convert_into_waveglow_and_denoiser():
    from flowtron_b200 import _lib
    from flowtron_b200.denoiser import Denoiser
    from flowtron_b200.waveglow import WaveGlow
    wcfg = synth.DEFAULT_WAVEGLOW_CONFIG
    wg = WaveGlow(**wcfg)
    wg.load_state_dict(synth.synth_waveglow_params(wcfg, 14), strict=True)
    wg = wg.cuda().eval()
    den = Denoiser(wg)
    m = _model(2, 81)
    B, T, L = 4, 36, 18
    in_lens, out_lens = [18, 6, 12, 15], [36, 20, 28, 14]
    g = torch.Generator().manual_seed(17)
    text = torch.randint(0, 185, (B, L), generator=g).cuda()
    spk = torch.tensor([0, 1, 0, 1], device="cuda")
    noise = synth.synth_waveglow_noise(B, T, 15).cuda()
    with torch.no_grad():
        mel = m.convert(_mels(18, B, T), spk, 1 - spk, text, in_lens, out_lens)
        audio = wg.infer(mel.contiguous(), sigma=0.6, noise=noise, lengths=out_lens)
        clean = den(audio, 0.1, lengths=[256 * n for n in out_lens])
    torch.cuda.synchronize()
    assert _lib.device_status() == 0
    assert torch.isfinite(audio).all() and torch.isfinite(clean).all()
    for b, n in enumerate(out_lens):
        assert (audio[b, 256 * n:] == 0).all() and (clean[b, 0, 256 * n:] == 0).all(), b
        assert audio[b, :256 * n].abs().max().item() > 0
