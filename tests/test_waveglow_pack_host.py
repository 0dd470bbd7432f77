"""CPU: the kernels' packed WaveGlow weights, pinned by sha256 per packed field.  WaveGlow._pack (infer: host weight-norm
fold, fp16 GEMM operands, fp32 inverses of convinv) and WaveGlow._train_params (training: the fp32 layouts built with
differentiable ops) must keep producing these exact bytes, in weight-norm and in plain form, for the shipped config and a
small one without early outputs; so must the fp16 and transposed copies the training kernels read.
`python tests/test_waveglow_pack_host.py` rewrites the table."""
import hashlib
import json
import os

import pytest
import torch

from conftest import GOLDEN
from flowtron_b200 import synth
from flowtron_b200.waveglow import WaveGlow

TABLE = os.path.join(GOLDEN, "waveglow_pack_sha256.json")
CONFIGS = {
    "default": synth.DEFAULT_WAVEGLOW_CONFIG,
    "small": dict(synth.DEFAULT_WAVEGLOW_CONFIG, n_flows=3, n_early_size=0,
                  WN_config=dict(n_layers=2, n_channels=256, kernel_size=3)),
}
FLOW_FIELDS = ("conv_w", "start_w", "start_b", "end_w", "end_b")
LAYER_FIELDS = ("in_w", "in_b", "rs_w", "rs_b")


def _sha(t: torch.Tensor) -> str:
    t = t.detach().cpu().contiguous()
    h = hashlib.sha256(f"{t.dtype}{tuple(t.shape)}".encode())
    h.update(t.view(torch.uint8).numpy().tobytes() if t.numel() else b"")
    return h.hexdigest()


def _model(cfg, plain: bool) -> WaveGlow:
    m = WaveGlow(**cfg)
    m.load_state_dict(synth.synth_waveglow_params(cfg, 77), strict=True)
    return WaveGlow.remove_weightnorm(m) if plain else m


def _train_keys(cfg):
    """The packed fields in FtWaveGlowTrainWeights' order: up_w, up_b, then per flow conv_w .. end_b and its layers."""
    keys = [("up_w",), ("up_b",)]
    for k in range(cfg["n_flows"]):
        keys += [(f, k) for f in FLOW_FIELDS]
        for i in range(cfg["WN_config"]["n_layers"]):
            keys += [(f, k, i) for f in LAYER_FIELDS]
    return keys


def _name(key) -> str:
    return ".".join(str(p) for p in key)


def _pack_table(m: WaveGlow, cfg) -> dict:
    w, keep = m._pack()
    by_ptr = {t.data_ptr(): t for t in keep}
    L = cfg["WN_config"]["n_layers"]
    out = {"up_w": _sha(by_ptr[w.up_w]), "up_b": _sha(by_ptr[w.up_b])}
    for k in range(cfg["n_flows"]):
        for f in ("start_w", "start_b", "end_w", "end_b", "inv_w"):
            out[f"{f}.{k}"] = _sha(by_ptr[getattr(w, f)[k]])
        for i in range(L):
            for f in LAYER_FIELDS:
                out[f"{f}.{k}.{i}"] = _sha(by_ptr[getattr(w, f)[k][i]])
    return out


def _train_table(m: WaveGlow, cfg) -> dict:
    p = m._train_params()
    if not isinstance(p, dict):                     # a flat list in _train_keys order
        p = dict(zip(_train_keys(cfg), p))
    assert list(p) == _train_keys(cfg)
    return {_name(k): _sha(t) for k, t in p.items()}


def _kernel_table(m: WaveGlow) -> dict:
    from flowtron_b200.waveglow import _train_kernel_weights
    return {_name(k): _sha(t) for k, t in _train_kernel_weights(m._train_params()).items()}


def _table(kinds=("pack", "train", "kernel")) -> dict:
    out = {}
    for cname, cfg in CONFIGS.items():
        for form in ("weight_norm", "plain"):
            m = _model(cfg, form == "plain")
            for kind in kinds:
                out[f"{cname}/{form}/{kind}"] = _kernel_table(m) if kind == "kernel" else \
                    (_pack_table if kind == "pack" else _train_table)(m, cfg)
    return out


@pytest.fixture(scope="module")
def table():
    return _table(("pack", "train"))


def _check(got: dict, key: str):
    with open(TABLE) as f:
        ref = json.load(f)
    assert sorted(got) == sorted(ref[key])
    bad = [n for n in ref[key] if got[n] != ref[key][n]]
    assert not bad, bad[:8]


@pytest.mark.parametrize("cname", sorted(CONFIGS))
@pytest.mark.parametrize("form", ["weight_norm", "plain"])
@pytest.mark.parametrize("kind", ["pack", "train"])
def test_packed_weights_are_pinned(table, cname, form, kind):
    key = f"{cname}/{form}/{kind}"
    _check(table[key], key)


@pytest.mark.parametrize("cname", sorted(CONFIGS))
@pytest.mark.parametrize("form", ["weight_norm", "plain"])
def test_training_kernel_copies_are_pinned(cname, form):
    """The fp16 GEMM operands and the backward's transposed in_wT / rs_wT that _WaveGlowTrainFn hands the kernels."""
    _check(_kernel_table(_model(CONFIGS[cname], form == "plain")), f"{cname}/{form}/kernel")


def test_pack_is_cached_per_weight_version():
    m = _model(CONFIGS["small"], False)
    packed = m._pack()
    assert m._pack() is packed
    with torch.no_grad():
        m.WN[1].end.bias.add_(1.0)
    assert m._pack() is not packed


def test_weight_forms_pack_identically(table):
    """The host fold makes both forms of one checkpoint pack bit-identically for infer."""
    for cname in CONFIGS:
        assert table[f"{cname}/weight_norm/pack"] == table[f"{cname}/plain/pack"]


if __name__ == "__main__":
    with open(TABLE, "w") as f:
        json.dump(_table(), f, indent=1, sort_keys=True)
        f.write("\n")
