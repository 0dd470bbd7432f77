"""CPU: the C-ABI library loads and exports every symbol include/flowtron_b200.h declares; the host-side module
mirror keeps the reference's state_dict layout; product code never imports oracle/ and fails loudly on CPU."""
import ctypes
import os
import re

import pytest
import torch

from conftest import ROOT
from flowtron_b200 import synth


def test_library_exports_every_declared_symbol():
    from flowtron_b200 import _lib, build
    path = build.build()
    L = ctypes.CDLL(path)
    hdr = open(os.path.join(ROOT, "include", "flowtron_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    names = set(re.findall(r"\b(ft_[a-z0-9_]+)\s*\(", hdr))
    assert len(names) >= 15
    missing = [n for n in sorted(names) if not hasattr(L, n)]
    assert not missing, missing
    assert _lib.lib().ft_version() >= 100


def test_state_dict_layout_matches_reference_spec():
    from flowtron_b200.flowtron import Flowtron
    for n_flows in (1, 2, 3):
        cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=n_flows)
        m = Flowtron(**cfg)
        spec = synth.param_shapes(cfg)
        sd = m.state_dict()
        assert set(sd.keys()) == set(spec.keys())
        for k, v in sd.items():
            assert tuple(v.shape) == tuple(spec[k]), k
        m.load_state_dict(synth.synth_params(cfg, 3), strict=True)


def test_state_dict_loads_into_reference_and_back():
    """Same keys, order and shapes as the reference Flowtron's state_dict (tests/golden/reference_checks.npz), so
    checkpoints load strictly in both directions."""
    import numpy as np
    from flowtron_b200.flowtron import Flowtron
    ref = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_checks.npz"))
    cfg = dict(synth.DEFAULT_MODEL_CONFIG)
    ours = Flowtron(**cfg)
    ours.load_state_dict(synth.synth_params(cfg, 5), strict=True)
    sd = ours.state_dict()
    assert list(sd.keys()) == [str(k) for k in ref["sd_keys"]]
    assert [",".join(str(d) for d in v.shape) for v in sd.values()] == [str(s) for s in ref["sd_shapes"]]


def test_product_path_fails_loudly_on_cpu():
    from flowtron_b200._lib import FlowtronB200Error
    from flowtron_b200.flowtron import Flowtron
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=1)
    m = Flowtron(**cfg).eval()
    b = synth.synth_batch(2, 8, 6, cfg, 1)
    with pytest.raises(FlowtronB200Error):
        m(b["mel"], b["speaker_ids"], b["text"], b["in_lens"], b["out_lens"])


def test_product_package_never_imports_oracle():
    pkg = os.path.join(ROOT, "flowtron_b200")
    for dp, _, fs in os.walk(pkg):
        for f in fs:
            if f.endswith(".py"):
                src = open(os.path.join(dp, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M), f


def test_encoder_rejects_sizes_the_kernels_are_not_built_for():
    from flowtron_b200.flowtron import Encoder, MaskedInstanceNorm1d
    Encoder(norm_fn=MaskedInstanceNorm1d)
    for kw in (dict(encoder_embedding_dim=256), dict(encoder_n_convolutions=2), dict(encoder_kernel_size=3)):
        with pytest.raises(NotImplementedError):
            Encoder(norm_fn=MaskedInstanceNorm1d, **kw)
    with pytest.raises(NotImplementedError):
        Encoder(norm_fn=torch.nn.BatchNorm1d)


def test_encoder_fails_loudly_on_cpu():
    from flowtron_b200._lib import FlowtronB200Error
    from flowtron_b200.flowtron import Flowtron
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=1)
    m = Flowtron(**cfg).eval()
    b = synth.synth_batch(3, 8, 11, cfg, 2)
    x = m.embedding(b["text"]).transpose(1, 2)
    for call in (lambda: m.encoder(x, b["in_lens"]), lambda: m.encoder.infer(x[:1]),
                 lambda: m.encoder.forward_tokens(b["text"], m.embedding, b["in_lens"]),
                 lambda: m.encoder.infer_tokens(b["text"], m.embedding),
                 lambda: m.encoder.infer_ragged_tokens(b["text"], m.embedding, b["in_lens"])):
        with pytest.raises(FlowtronB200Error):
            call()


def test_validated_defaults_and_no_native_environment_switches():
    """The GPU validation of record (profiles/r2_*) ran with: encoder overlap ON, fused optimizer ON (capturable), layer
    pipeline ON (forward and BPTT), CUDA-graph step ON in bench.py.  The native library reads no environment variable, so
    its schedule is a function of its arguments alone; bench.py's switches are opt-in (DESIGN.md 4.11)."""
    import flowtron_b200.flowtron as F
    assert F.Flowtron.overlap_encoder is True
    src = open(os.path.join(ROOT, "bench.py")).read()
    assert 'os.environ.get("FT_FUSED_OPT", "1")' in src
    csrc = os.path.join(ROOT, "flowtron_b200", "csrc")
    assert not [f for f in sorted(os.listdir(csrc)) if "getenv" in open(os.path.join(csrc, f)).read()]
    assert 'os.environ.get("FT_GRAPH", "1")' in src


def test_flow_step_has_no_hidden_process_state():
    """What ft_ar_step_fwd launches follows from its arguments: the library has no process-wide kernel switch and no
    per-thread side channel for the text-ready event, and Flowtron.forward hands that event to the flows as an argument,
    not through module attributes."""
    from flowtron_b200 import build
    L = ctypes.CDLL(build.build())
    for name in ("ft_set_lstm_half_sm", "ft_ar_step_set_text_ready_event"):
        assert not hasattr(L, name), name
    csrc = os.path.join(ROOT, "flowtron_b200", "csrc")
    per_thread = [(f, line.strip()) for f in sorted(os.listdir(csrc)) for line in open(os.path.join(csrc, f))
                  if "thread_local" in line]
    # the one per-thread variable is the message ft_last_error returns, which is per thread like errno
    assert per_thread == [("api.cu", "static thread_local std::string g_err;")], per_thread
    src = open(os.path.join(ROOT, "flowtron_b200", "flowtron.py")).read()
    assert "_text_event" not in src and "_enc_chunks" not in src


def test_encoder_abi_host_side():
    """ft_encoder_*_bytes are pure host functions: sizes grow with the batch, an unsupported descriptor gives 0 and an error
    string (no GPU needed)."""
    from ctypes import byref
    from flowtron_b200 import _lib
    L = _lib.lib()
    small, big = _lib.encoder_desc(2, 16, True, 0.0), _lib.encoder_desc(32, 160, True, 0.5)
    for fn in (L.ft_encoder_saved_bytes, L.ft_encoder_fwd_scratch_bytes, L.ft_encoder_bwd_scratch_bytes):
        a, b = fn(byref(small)), fn(byref(big))
        assert 0 < a < b
    bad = _lib.encoder_desc(2, 16, True, 0.0)
    bad.C = 256
    assert L.ft_encoder_saved_bytes(byref(bad)) == 0
    assert b"512" in L.ft_last_error()
    # the weight / gradient structs have one pointer per reference parameter of Encoder (flowtron.py:473-490)
    assert sum(k for _, k in _lib.ENC_PARAM_FIELDS) == 20
