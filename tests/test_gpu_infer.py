"""GPU: Flowtron.infer (persistent inference kernel) vs reference-generated fixtures and the invertibility identity."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, record_parity
from flowtron_b200 import synth

pytestmark = pytest.mark.gpu


def _model(cfg, seed, gate_bias=None, gate_scale=1.0):
    from flowtron_b200.flowtron import Flowtron
    p = synth.synth_params(cfg, seed)
    if gate_bias is not None:
        key = [k for k in p if k.endswith("gate_layer.linear_layer.bias")][0]
        p[key] = torch.full_like(p[key], gate_bias)
        key = [k for k in p if k.endswith("gate_layer.linear_layer.weight")][0]
        p[key] = p[key] * gate_scale
    m = Flowtron(**cfg)
    m.load_state_dict(p, strict=True)
    return m.cuda().eval()


@pytest.mark.parametrize("tag", ["b1", "b1gate", "b4nogate"])
def test_infer_matches_reference_goldens(tag):
    from flowtron_b200 import _lib
    gold = dict(np.load(os.path.join(GOLDEN, f"infer_{tag}.npz")))
    use_gate = bool(gold["use_gate"])
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=int(gold["cfg_n_flows"]), use_gate_layer=use_gate)
    m = _model(cfg, int(gold["seed"]), float(gold["gate_bias"]) if use_gate else None)
    B = int(gold["B"])
    with torch.no_grad():
        mel, attn = m.infer(torch.from_numpy(gold["residual"]).cuda(), torch.zeros(B, dtype=torch.long, device="cuda"),
                            torch.from_numpy(gold["text"]).cuda())
    torch.cuda.synchronize()
    assert _lib.device_status() == 0
    ref = torch.from_numpy(gold["mel"])
    assert tuple(mel.shape) == tuple(ref.shape), (mel.shape, ref.shape)
    err = (mel.cpu() - ref).abs().max().item() / ref.abs().max().item()
    print("infer rel err", err)
    record_parity(f"infer_{tag}", {"mel": err})
    assert err <= 1e-3, err                      # north_star bar


def test_invertibility_forward_of_infer():
    """flowtron.py:932-954: forward(infer(z)) == z (reference docstring: 'order of 1e-5' in fp32; here both directions
    use fp16 tensor-core operands, so the round trip closes to ~1e-3 of |z|)."""
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=2, use_gate_layer=False)
    m = _model(cfg, 3)
    g = torch.Generator().manual_seed(3)
    T, L = 40, 12
    zin = (torch.randn(1, 80, T, generator=g) * 0.5).cuda()
    text = torch.randint(0, 185, (1, L), generator=g).cuda()
    spk = torch.zeros(1, dtype=torch.long, device="cuda")
    with torch.no_grad():
        mel, _ = m.infer(zin, spk, text)
        out = m(mel, spk, text, torch.tensor([L], device="cuda"), torch.tensor([T], device="cuda"))
    z = out[0].permute(1, 2, 0)
    err = (z - zin).abs().max().item() / zin.abs().max().item()
    print("round trip rel err", err)
    record_parity("infer_roundtrip_T40", {"z_roundtrip": err})
    assert err <= 2e-3, err


def test_batched_rows_equal_single_runs():
    """B=3 with a gate (the reference raises there): every row must equal its own B=1 run (SURVEY §3.2)."""
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=2)
    m = _model(cfg, 21, gate_bias=-1.5)
    g = torch.Generator().manual_seed(4)
    B, T, L = 3, 24, 10
    res = (torch.randn(B, 80, T, generator=g) * 0.5).cuda()
    text = torch.randint(0, 185, (B, L), generator=g).cuda()
    spk = torch.zeros(B, dtype=torch.long, device="cuda")
    with torch.no_grad():
        mel_b, _ = m.infer(res, spk, text)
        for b in range(B):
            mel_1, _ = m.infer(res[b:b + 1], spk[b:b + 1], text[b:b + 1])
            n = mel_1.shape[-1]
            ref = mel_1[0]
            got = mel_b[b, :, :n] if mel_b.shape[-1] >= n else None
            assert got is not None
            assert (got - ref).abs().max().item() <= 2e-3 * ref.abs().max().item()


@pytest.mark.parametrize("n_flows, seed, gate_bias, fixture_rows", [
    (2, 61, -0.3, None),                # the steep gates of test_gpu_infer_batch.py
    (3, 62, -6.0, [0, 3, 5]),           # (3 flows: on rows of infer_ragged_f3.npz that stop at different frames)
])
def test_rows_stopping_at_different_frames_equal_single_runs(n_flows, seed, gate_bias, fixture_rows):
    """B=3, a gate that stops the rows at different frames: each row equals its own B=1 run bit for bit and is zero after
    it (a back step flips each row within its own length; later flows see each row's length)."""
    if fixture_rows is None:
        cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=n_flows)
        g = torch.Generator().manual_seed(4)
        B, T, L = 3, 24, 10
        res = (torch.randn(B, 80, T, generator=g) * 0.5).cuda()
        text = torch.randint(0, 185, (B, L), generator=g).cuda()
        spk = torch.zeros(B, dtype=torch.long, device="cuda")
    else:
        gold = np.load(os.path.join(GOLDEN, "infer_ragged_f3.npz"))
        cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=n_flows, n_speakers=int(gold["n_speakers"]))
        res, text, spk = [torch.from_numpy(gold[k][fixture_rows]).cuda() for k in ("residual", "text", "speaker_ids")]
        B = len(fixture_rows)
    m = _model(cfg, seed, gate_bias, gate_scale=40.0)
    with torch.no_grad():
        mel_b, _ = m.infer(res, spk, text)
        singles = [m.infer(res[b:b + 1], spk[b:b + 1], text[b:b + 1])[0][0] for b in range(B)]
    lens = [s.shape[-1] for s in singles]
    assert mel_b.shape[-1] == max(lens) and len(set(lens)) > 1, (mel_b.shape, lens)
    for b, ref in enumerate(singles):
        n = lens[b]
        assert torch.equal(mel_b[b, :, :n], ref) and (mel_b[b, :, n:] == 0).all(), (b, lens)


def test_forced_alignments_attns_argument():
    """Flowtron.infer(..., attns=) (flowtron.py:585-588, 797): with each flow's own attention weights fed back as forced
    alignments the output must equal the free-running result (the context is then the same attn . V), and rolled
    alignments must change it.  Oracle cross-check of the forced branch at a small shape."""
    from flowtron_b200 import _lib
    from oracle import flowtron_oracle as O
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=2, use_gate_layer=False)
    m = _model(cfg, 17)
    g = torch.Generator().manual_seed(9)
    T, L = 24, 11
    res = (torch.randn(1, 80, T, generator=g) * 0.5)
    text = torch.randint(0, 185, (1, L), generator=g)
    spk = torch.zeros(1, dtype=torch.long)
    with torch.no_grad():
        mel0, attn0 = m.infer(res.cuda(), spk.cuda(), text.cuda())
        # attention_weights are returned in flow-application order (last flow first); attns is indexed per flow
        attns = [torch.stack([a[0, 0] for a in aw]) for aw in reversed(attn0)]          # per flow [T, L]
        mel1, attn1 = m.infer(res.cuda(), spk.cuda(), text.cuda(), attns=attns)
        rolled = [torch.zeros_like(a) for a in attns]               # a very different alignment: everything on the last token
        for a in rolled:
            a[:, -1] = 1.0
        mel2, _ = m.infer(res.cuda(), spk.cuda(), text.cuda(), attns=rolled)
        ref2, _ = O.flowtron_infer(synth.synth_params(cfg, 17), res, spk, text, attns=[a.cpu() for a in rolled])
    torch.cuda.synchronize()
    assert _lib.device_status() == 0
    assert (mel1 - mel0).abs().max().item() <= 1e-5 * mel0.abs().max().item()
    for a, b in zip(attn0, attn1):
        assert torch.equal(torch.stack(a), torch.stack(b))
    err = (mel2.cpu() - ref2).abs().max().item() / ref2.abs().max().item()
    moved = (mel2 - mel0).abs().max().item() / ref2.abs().max().item()
    record_parity("infer_forced_attns", {"mel": err, "changed_by": moved})
    assert err <= 1e-3, err
    assert moved > 3 * err, (moved, err)            # the forced alignment is really used
