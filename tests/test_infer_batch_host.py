"""CPU: the oracle's restatement of Flowtron.infer_batch's contract against the reference-generated
fixtures (tests/make_golden_infer_batch.py), and the register budget of the inference kernels."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT
from flowtron_b200 import synth

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
HAVE_NVCC = os.path.exists(NVCC) or shutil.which("nvcc") is not None


def _params(g):
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=int(g["cfg_n_flows"]), n_speakers=int(g["n_speakers"]))
    p = synth.synth_params(cfg, int(g["seed"]))
    kb = [k for k in p if k.endswith("gate_layer.linear_layer.bias")][0]
    kw = [k for k in p if k.endswith("gate_layer.linear_layer.weight")][0]
    p[kb] = torch.full_like(p[kb], float(g["gate_bias"]))
    p[kw] = p[kw] * float(g["gate_scale"])
    return cfg, p


@pytest.mark.parametrize("tag", ["f2", "f3", "t400"])
def test_oracle_infer_batch_matches_reference_fixtures(tag):
    from infer_batch_oracle import flowtron_infer_batch
    g = dict(np.load(os.path.join(GOLDEN, f"infer_ragged_{tag}.npz")))
    _, p = _params(g)
    torch.set_num_threads(max(1, min(8, os.cpu_count() or 1)))
    with torch.no_grad():
        mel, lens = flowtron_infer_batch(p, torch.from_numpy(g["residual"]), torch.from_numpy(g["speaker_ids"]),
                                         torch.from_numpy(g["text"]), g["in_lens"].tolist(),
                                         max_frames=g["max_frames"].tolist())
    assert lens.tolist() == g["mel_lens"].tolist()
    ref = torch.from_numpy(g["mel"])
    err = (mel - ref).abs().max().item() / ref.abs().max().item()
    assert err <= 1e-5, err


def test_fixtures_cover_gate_stops_and_budgets():
    for tag, need_stops in (("f2", 2), ("f3", 2), ("t400", 0)):
        g = np.load(os.path.join(GOLDEN, f"infer_ragged_{tag}.npz"))
        stopped = int((g["mel_lens"] < g["max_frames"]).sum())
        assert stopped >= need_stops and len(g["mel_lens"]) - stopped >= 2, (tag, g["mel_lens"], g["max_frames"])
        assert (np.diff(g["in_lens"]) > 0).any() and (np.diff(g["in_lens"]) < 0).any()     # not sorted


@pytest.mark.skipif(not HAVE_NVCC, reason="nvcc not available")
def test_infer_kernels_fit_the_register_budget(tmp_path):
    """infer_kernel<batch > 8, long text, forced>: eight instantiations of the persistent kernel, 512 threads each, so 128
    registers at most, and no spills; the finish kernel likewise."""
    r = subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr",
                        "-Xptxas", "-v", "-c", os.path.join(ROOT, "flowtron_b200", "csrc", "infer.cu"), "-o",
                        str(tmp_path / "infer.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    logs = {}
    for part in r.stderr.split("Compiling entry function")[1:]:
        logs[re.match(r"\s*'(\S+)'", part).group(1)] = part
    want = [f"_ZN2ft12infer_kernelILb{a}ELb{b}ELb{c}EEEvNS_11InferParamsE" for a in "01" for b in "01" for c in "01"]
    want.append("_ZN2ft19infer_finish_kernelEPfS0_PKiiiiii")
    assert all(k in logs for k in want), sorted(logs)
    for k in want:
        regs = int(re.search(r"Used (\d+) registers", logs[k]).group(1))
        spill = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", logs[k])
        assert regs <= 128 and spill.groups() == ("0", "0"), logs[k]
