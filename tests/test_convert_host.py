"""CPU: the forced-alignment argument checks of the flow steps' infer_ragged, the oracle's restatement of Flowtron.convert's
and Flowtron.infer_aligned's contract against the reference-generated fixtures (tests/make_golden_convert.py) and what those fixtures cover."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from flowtron_b200 import synth
from test_batch_args_host import cpu_model  # noqa: F401

TAGS = ["f2", "f3", "long"]


def _load(tag):
    return dict(np.load(os.path.join(GOLDEN, f"convert_{tag}.npz")))


def _params(g):
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=int(g["cfg_n_flows"]), n_speakers=int(g["n_speakers"]))
    p = synth.synth_params(cfg, int(g["seed"]))
    kb = [k for k in p if k.endswith("gate_layer.linear_layer.bias")][0]
    p[kb] = torch.full_like(p[kb], float(g["gate_bias"]))
    return cfg, p


def test_flow_infer_ragged_forced_argument_validation(cpu_model):
    from flowtron_b200._lib import FlowtronB200Error
    lens = torch.tensor([8, 5], dtype=torch.int32)
    for flow in cpu_model.flows:
        with pytest.raises(ValueError):                          # [T, B, L] instead of [B, Ta, L]
            flow.infer_ragged(torch.zeros(8, 2, 80), torch.zeros(6, 2, 640), lens, lens, attns=torch.zeros(8, 2, 6))
        with pytest.raises(ValueError, match="1024"):
            flow.infer_ragged(torch.zeros(8, 2, 80), torch.zeros(1025, 2, 640), lens, lens, attns=torch.zeros(2, 8, 1025))
        with pytest.raises(FlowtronB200Error):
            flow.infer_ragged(torch.zeros(8, 2, 80), torch.zeros(6, 2, 640), lens, lens, attns=torch.zeros(2, 8, 6))


@pytest.mark.parametrize("tag", TAGS)
def test_oracle_convert_matches_reference_fixtures(tag):
    from convert_oracle import flowtron_convert, flowtron_infer_aligned
    g = _load(tag)
    _, p = _params(g)
    torch.set_num_threads(max(1, min(8, os.cpu_count() or 1)))
    t = lambda k: torch.from_numpy(g[k])
    in_lens, out_lens = g["in_lens"].tolist(), g["out_lens"].tolist()
    with torch.no_grad():
        mel, z, attns = flowtron_convert(p, t("mel"), t("speaker_ids"), t("target_speaker_ids"), t("text"), in_lens, out_lens)
    rel = lambda x, ref: (x - ref).abs().max().item() / ref.abs().max().item()
    assert rel(z, t("z")) <= 1e-5
    for f, a in enumerate(attns):
        assert (a - t(f"attn_{f}")).abs().max().item() <= 1e-5, f
    assert rel(mel, t("mel_converted")) <= 1e-5
    if "mel_rhythm" in g:
        with torch.no_grad():
            rhy = flowtron_infer_aligned(p, t("noise"), t("target_speaker_ids"), t("text"), in_lens,
                                         [t(f"attn_{f}") for f in range(len(attns))], out_lens)
        assert rel(rhy, t("mel_rhythm")) <= 1e-5


def test_fixtures_cover_their_cases():
    for tag in TAGS:
        g = _load(tag)
        n_flows, B = int(g["cfg_n_flows"]), len(g["in_lens"])
        assert (g["speaker_ids"] != g["target_speaker_ids"]).all()               # every row changes voice
        assert len(set(g["speaker_ids"].tolist())) >= 2 and len(set(g["target_speaker_ids"].tolist())) >= 2
        assert g["mel"].shape == g["mel_converted"].shape == g["z"].shape
        for b in range(B):
            nt, nl = int(g["out_lens"][b]), int(g["in_lens"][b])
            assert (g["mel_converted"][b, :, nt:] == 0).all() and np.abs(g["mel_converted"][b, :, :nt]).max() > 0
            assert np.abs(g["mel_converted"][b, :, :nt] - g["mel"][b, :, :nt]).max() > 0.1    # the voice matters
            for f in range(n_flows):
                a = g[f"attn_{f}"][b]
                assert (a[nt:] == 0).all() and (a[:, nl:] == 0).all()
                assert np.abs(a[:nt].sum(-1) - 1).max() <= 1e-5
        for f in range(1, n_flows, 2):                                           # a back step's map is not the forward step's
            assert np.abs(g[f"attn_{f}"] - g[f"attn_{f - 1}"]).max() > 1e-3
    for tag in ("f2", "f3"):
        g = _load(tag)
        for k in ("in_lens", "out_lens"):
            assert (np.diff(g[k]) > 0).any() and (np.diff(g[k]) < 0).any(), (tag, k)   # not sorted
    assert int(_load("f2")["cfg_n_flows"]) == 2 and int(_load("f3")["cfg_n_flows"]) == 3
    assert "mel_rhythm" in _load("f2")                                           # z replaced by fresh noise
    g = _load("long")
    assert g["text"].shape[1] > 256 and (g["in_lens"] > 256).all() and g["in_lens"][0] != g["in_lens"][1]
    for tag in TAGS:
        assert os.path.getsize(os.path.join(GOLDEN, f"convert_{tag}.npz")) < 1 << 20

