"""CPU: the text-length limit of the flow-step kernels (FT_MAX_TEXT_LEN = 1024 tokens) is one constant shared by the C
header, the library and flowtron_b200._lib; the host entry points refuse longer texts before any device work; the
long-text fixtures (tests/make_golden_long_text.py) cover what their tests claim; and the long-text kernels compile
next to the unchanged short-text ones."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT
from flowtron_b200 import synth
from test_batch_args_host import cpu_model  # noqa: F401

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
HAVE_NVCC = os.path.exists(NVCC) or shutil.which("nvcc") is not None


def test_header_library_and_python_constants_agree():
    from flowtron_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "flowtron_b200.h")).read()
    m = re.search(r"#define\s+FT_MAX_TEXT_LEN\s+(\d+)", hdr)
    assert m and int(m.group(1)) == _lib.MAX_TEXT_LEN == 1024
    assert _lib.lib().ft_max_text_len() == _lib.MAX_TEXT_LEN


def test_forward_refuses_texts_over_the_limit_before_the_device_check(cpu_model):
    from flowtron_b200._lib import FlowtronB200Error
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=2)
    for L, err in ((1025, ValueError), (1024, FlowtronB200Error)):        # 1024 passes the length check, then needs CUDA
        b = synth.synth_batch(1, 8, L, cfg, 1)
        with pytest.raises(err) as e:
            cpu_model(b["mel"], b["speaker_ids"], b["text"], b["in_lens"], b["out_lens"])
        if err is ValueError:
            assert "1024" in str(e.value)


def test_infer_refuses_texts_over_the_limit_before_the_device_check(cpu_model):
    from flowtron_b200._lib import FlowtronB200Error
    res, spk = torch.zeros(1, 80, 6), torch.zeros(1, dtype=torch.long)
    with pytest.raises(ValueError, match="1024"):
        cpu_model.infer(res, spk, torch.zeros(1, 1025, dtype=torch.long))
    with pytest.raises(FlowtronB200Error):
        cpu_model.infer(res, spk, torch.zeros(1, 1024, dtype=torch.long))


def test_flow_steps_refuse_texts_over_the_limit(cpu_model):
    step = cpu_model.flows[0]
    text = torch.zeros(1025, 1, 640)
    with pytest.raises(ValueError, match="1024"):
        step(torch.zeros(8, 1, 80), text, None, torch.tensor([8]))
    with pytest.raises(ValueError, match="1024"):
        step.infer(torch.zeros(8, 1, 80), text, None)
    with pytest.raises(ValueError, match="1024"):
        cpu_model.flows[1].infer(torch.zeros(8, 1, 80), text, None)


def test_infer_batch_keeps_its_256_token_cap(cpu_model):
    with pytest.raises(ValueError):
        cpu_model.infer_batch(torch.zeros(1, 80, 6), torch.zeros(1, dtype=torch.long), torch.zeros(1, 257, dtype=torch.long), [9])


def test_long_text_fixtures_cover_their_cases():
    for tag, L, in_lens in (("long400", 400, [400, 290]), ("long1024", 1024, [1024, 700])):
        g = np.load(os.path.join(GOLDEN, f"train_{tag}.npz"))
        assert int(g["L"]) == L and g["in_lens"].tolist() == in_lens and float(g["ctc_weight"]) == 1.0
        assert int(g["with_prior"]) == 1 and int(g["cfg_n_flows"]) == 2
    g = np.load(os.path.join(GOLDEN, "train_long400.npz"))
    assert (g["out_lens"] >= g["in_lens"]).all() and float(g["loss_ctc"]) > 0.0     # a finite CTC loss
    assert int(g["T"]) >= 320                                                        # the attention overlap runs
    g = np.load(os.path.join(GOLDEN, "infer_long1024.npz"))
    assert int(g["L"]) == 1024 and g["mel"].shape[-1] == int(g["T"])               # gate off: every frame
    g = np.load(os.path.join(GOLDEN, "infer_long600gate.npz"))
    assert int(g["L"]) == 600 and g["mel"].shape[-1] < int(g["T"])                 # the gate stops generation


def _ptxas(src, tmp_path):
    r = subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr",
                        "-Xptxas", "-v", "-c", os.path.join(ROOT, "flowtron_b200", "csrc", src), "-o",
                        str(tmp_path / (src + ".o"))], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    out = {}
    for part in r.stderr.split("Compiling entry function")[1:]:
        name = re.match(r"\s*'(\S+)'", part).group(1)
        regs = re.search(r"Used (\d+) registers", part)
        spill = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", part)
        out[name] = (int(regs.group(1)), spill.groups())
    return out


@pytest.mark.skipif(not HAVE_NVCC, reason="nvcc not available")
def test_short_text_training_kernels_keep_their_register_budget(tmp_path):
    """The L <= 256 kernels are the parent's: same registers, no spills (the long-text variants are separate
    instantiations: attn_*_kernel<true>, attn_ctc_long_kernel; the inference kernels' budget is checked in
    test_infer_batch_host.py)."""
    attn = _ptxas("attention.cu", tmp_path)
    assert attn["_ZN2ft15attn_fwd_kernelILb0EEEvNS_13AttnFwdParamsE"] == (96, ("0", "0"))
    assert attn["_ZN2ft15attn_bwd_kernelILb0EEEvNS_13AttnBwdParamsE"] == (126, ("0", "0"))
    ctc = _ptxas("ctc.cu", tmp_path)
    assert ctc["_ZN2ft15attn_ctc_kernelEPKfPKiS3_iiifPfS4_S4_"] == (32, ("0", "0"))
    assert any("attn_ctc_long_kernel" in k for k in ctc)
