"""CPU: argument checks of style.posterior_mean, the C-ABI declaration of ft_posterior_mean, its
rejections, the register budget of csrc/style.cu, and the float64 restatement behind the style-transfer fixtures
(tests/make_golden_style_transfer.py)."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
HAVE_NVCC = os.path.exists(NVCC) or shutil.which("nvcc") is not None


def test_posterior_mean_argument_validation():
    from flowtron_b200._lib import FlowtronB200Error
    from flowtron_b200.style import posterior_mean
    z = torch.zeros(4, 80, 30)
    lens = [30, 12, 1, 7]
    for kw in (dict(lambd=0.0), dict(lambd=-1.0), dict(lambd=float("nan")), dict(aggregation="time"),
               dict(aggregation="mean")):
        with pytest.raises(ValueError):
            posterior_mean(z, lens, 50, **kw)
    for n in (0, -3, 2.5):
        with pytest.raises(ValueError):
            posterior_mean(z, lens, n)
    for bad in ([30, 12, 1], [30, 12, 0, 7], [30, 31, 1, 7], [30.0, 12.0, 1.0, 7.0]):
        with pytest.raises(ValueError):
            posterior_mean(z, bad, 50)
    with pytest.raises(ValueError):
        posterior_mean(z[0], lens, 50)
    with pytest.raises(ValueError):
        posterior_mean(torch.zeros(4, 129, 30), lens, 50)
    for agg in ("batch", "time_and_batch"):
        with pytest.raises(FlowtronB200Error):
            posterior_mean(z, lens, 50, aggregation=agg)
        with pytest.raises(FlowtronB200Error):
            posterior_mean(z, torch.tensor(lens), 50, aggregation=agg)


def _header_prototype(name):
    hdr = open(os.path.join(ROOT, "include", "flowtron_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    m = re.search(r"\b(\w+)\s+" + name + r"\s*\(([^)]*)\)\s*;", hdr)
    assert m, name
    return m.group(1), [" ".join(a.split()) for a in m.group(2).split(",")]


def test_posterior_mean_abi_matches_header():
    from flowtron_b200 import _lib, build
    L = ctypes.CDLL(build.build())
    assert hasattr(L, "ft_posterior_mean")
    ret, args = _header_prototype("ft_posterior_mean")
    assert ret == "int"

    def ctype(decl):
        if "*" in decl:
            return ctypes.c_void_p
        return {"int": ctypes.c_int, "float": ctypes.c_float}[decl.rsplit(" ", 1)[0]]
    f = _lib.lib().ft_posterior_mean
    assert f.restype is ctypes.c_int
    assert list(f.argtypes) == [ctype(a) for a in args], (args, f.argtypes)


def test_posterior_mean_rejections_set_the_error():
    """The argument checks run before any device work, so they can be exercised without a GPU."""
    from flowtron_b200 import _lib
    f = _lib.lib().ft_posterior_mean
    buf = ctypes.create_string_buffer(64)          # a non-NULL address: never dereferenced, every case is rejected first
    p = ctypes.cast(buf, ctypes.c_void_p)
    cases = [
        (dict(B=0), "B < 1"),
        (dict(n_frames=0), "n_frames < 1"),
        (dict(M=129), "M must lie in"),
        (dict(mode=2), "mode"),
        (dict(T=0), "T < 1"),
    ]
    for over, msg in cases:
        a = dict(T=10, B=2, M=80, n_frames=5, mode=0)
        a.update(over)
        rc = f(p, a["T"], a["B"], a["M"], p, a["n_frames"], a["mode"], 1.0, p, None)
        assert rc != 0 and msg in _lib.lib().ft_last_error().decode(), (over, _lib.lib().ft_last_error())
    assert f(None, 10, 2, 80, p, 5, 0, 1.0, p, None) != 0
    assert "NULL" in _lib.lib().ft_last_error().decode()


def test_fixture_means_restate_the_notebook():
    """The stored means against an independent float64 restatement (explicit tiling by concatenation, as the notebook
    grows each z until it covers n_frames), and the fixtures' coverage of n_frames below, at and above the lengths."""
    e = np.load(os.path.join(GOLDEN, "style_encode.npz"))
    p = np.load(os.path.join(GOLDEN, "style_posterior.npz"))
    z, lens = e["z"].astype(np.float64), e["out_lens"].tolist()
    K = len(lens)
    assert set(p["n_frames"].tolist()) == {30, 120, 300}
    assert min(lens) > 30 and max(lens) == 120 and max(lens) < 300
    for li, lambd in enumerate(p["lambds"].tolist()):
        scale = (K / lambd) / (K / lambd + 1.0)
        for n in p["n_frames"].tolist():
            tiled = []
            for k, t in enumerate(lens):
                row = z[k, :, :t]
                while row.shape[1] < n:
                    row = np.concatenate([row, z[k, :, :t]], axis=1)
                tiled.append(row[:, :n])
            np.testing.assert_allclose(p[f"mu_batch_n{n}_l{li}"], scale * np.mean(tiled, axis=0), rtol=0, atol=1e-12)
            tb = np.mean([z[k, :, :t].mean(axis=1) for k, t in enumerate(lens)], axis=0)[:, None]
            np.testing.assert_allclose(p[f"mu_time_and_batch_n{n}_l{li}"], scale * tb, rtol=0, atol=1e-12)
    pad = np.arange(z.shape[-1])[None, :] >= np.array(lens)[:, None]           # [K, T]
    assert (e["z"].transpose(0, 2, 1)[pad] == 0).all()


@pytest.mark.skipif(not HAVE_NVCC, reason="nvcc not available")
def test_style_kernels_do_not_spill(tmp_path):
    r = subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr",
                        "-Xptxas", "-v", "-c", os.path.join(ROOT, "flowtron_b200", "csrc", "style.cu"), "-o",
                        str(tmp_path / "style.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    parts = r.stderr.split("Compiling entry function")[1:]
    assert len(parts) == 2 and all("posterior_mean" in s.splitlines()[0] for s in parts), r.stderr
    for log in parts:
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", log)
        assert m and m.groups() == ("0", "0"), log
