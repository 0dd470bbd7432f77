"""CPU: the C-ABI declaration of ft_nll_rows /
ft_gmm_nll_rows and their host-side errors, and a numpy restatement of the per-utterance loss terms: their length-weighted
means are FlowtronLoss's batch losses (the oracle's restatement, and the reference's own module where it can be imported)."""
import os
import re

import numpy as np
import pytest
import torch

from conftest import ROOT
from oracle import flowtron_oracle as O
from oracle import ref_shims


def test_abi_symbols_are_declared_and_exported():
    from flowtron_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "flowtron_b200.h")).read()
    L = _lib.lib()
    for sym, n_args in (("ft_nll_rows", 11), ("ft_gmm_nll_rows", 9)):
        m = re.search(r"\bint\s+" + sym + r"\(([^)]*)\)", hdr)
        assert m, sym
        assert len(m.group(1).split(",")) == n_args == len(getattr(L, sym).argtypes), sym
        assert getattr(L, sym).restype is not None
    for fn in ("nll_rows", "gmm_nll_rows"):
        assert callable(getattr(_lib, fn))


def test_abi_rejects_bad_arguments_before_launching():
    """Errors that need no device: reported through ft_last_error, nothing is launched."""
    from ctypes import byref, c_void_p
    from flowtron_b200 import _lib
    L = _lib.lib()
    fake = c_void_p(256)                                        # never dereferenced: every call below fails its checks first
    arr = (c_void_p * 17)(*([256] * 17))
    assert L.ft_nll_rows(fake, arr, 17, None, None, fake, 4, 2, 80, fake, None) != 0
    assert b"16 flows" in L.ft_last_error()
    assert L.ft_nll_rows(fake, arr, 2, fake, None, fake, 4, 2, 80, fake, None) != 0
    assert b"gate_target" in L.ft_last_error()
    assert L.ft_nll_rows(fake, arr, 2, None, None, None, 4, 2, 80, fake, None) != 0
    assert b"NULL" in L.ft_last_error()
    assert L.ft_nll_rows(fake, arr, 2, None, None, fake, 0, 2, 80, fake, None) != 0
    bad = _lib.FtGmmDesc(T=4, B=2, M=80, K=33, per_row=1)
    assert L.ft_gmm_nll_rows(byref(bad), fake, fake, fake, fake, fake, fake, fake, None) != 0
    assert b"32" in L.ft_last_error()
    ok = _lib.FtGmmDesc(T=4, B=2, M=80, K=4, per_row=1)
    assert L.ft_gmm_nll_rows(byref(ok), fake, fake, fake, fake, fake, None, fake, None) != 0
    assert b"NULL" in L.ft_last_error()


# ---------------------------------------------------------------------------------------------- numpy restatement
def rows_restated(z, log_s_list, gate, gate_target, out_lens, sigma=1.0):
    """Per-utterance terms in float64: nll_b = (sum z^2 / (2 sigma^2) - sum log_s) / (n_b M), gate_b = mean BCE."""
    T, B, M = z.shape
    nll, gl = np.zeros(B), np.zeros(B)
    for b in range(B):
        n = int(out_lens[b])
        zz = z[:n, b].astype(np.float64)
        ls = sum(l[:n, b].astype(np.float64).sum() for l in log_s_list)
        nll[b] = ((zz * zz).sum() / (2 * sigma * sigma) - ls) / (n * M)
        x, y = gate[:n, b, 0].astype(np.float64), gate_target[b, :n].astype(np.float64)
        gl[b] = (np.maximum(x, 0) - x * y + np.log1p(np.exp(-np.abs(x)))).mean()
    return nll, gl


def gmm_rows_restated(z, log_s_list, out_lens, mean, log_var, prob):
    """The gm_loss branch per utterance in float64 (flowtron.py:217-231 on one row)."""
    T, B, M = z.shape
    out = np.zeros(B)
    for b in range(B):
        n = int(out_lens[b])
        mu = mean[0 if mean.shape[0] == 1 else b].astype(np.float64)          # [M, K]
        lv = log_var[0 if log_var.shape[0] == 1 else b].astype(np.float64)
        p = prob[b].astype(np.float64)
        d = z[:n, b, :, None].astype(np.float64) - mu[None]
        a = np.log(p)[None, None] - lv[None] / 2 - d * d / (2 * np.exp(lv[None]))
        mx = a.max(-1, keepdims=True)
        lse = mx[..., 0] + np.log(np.exp(a - mx).sum(-1))
        ls = sum(l[:n, b].astype(np.float64).sum() for l in log_s_list)
        out[b] = (-lse.sum() - ls) / (n * M)
    return out


def _random_outputs(seed, B=5, T=23, M=80, n_flows=3, K=4):
    g = np.random.default_rng(seed)
    out_lens = np.array([23, 7, 15, 1, 19][:B])
    z = g.standard_normal((T, B, M)).astype(np.float32)
    log_s = [(0.1 * g.standard_normal((T, B, M))).astype(np.float32) for _ in range(n_flows)]
    gate = (2 * g.standard_normal((T, B, 1))).astype(np.float32)
    gate_target = (np.arange(T)[None, :] >= (out_lens[:, None] - 1)).astype(np.float32)
    mean = g.standard_normal((B, M, K)).astype(np.float32)
    log_var = (0.3 * g.standard_normal((B, M, K))).astype(np.float32)
    prob = g.dirichlet(np.ones(K), B).astype(np.float32)
    return z, log_s, gate, gate_target, out_lens, mean, log_var, prob


@pytest.mark.parametrize("sigma", [1.0, 0.7])
def test_length_weighted_rows_are_the_oracle_batch_loss(sigma):
    z, log_s, gate, gt, out_lens, *_ = _random_outputs(0)
    nll, gl = rows_restated(z, log_s, gate, gt, out_lens, sigma)
    w = out_lens / out_lens.sum()
    t = torch.from_numpy
    bn, bg = O.flowtron_loss((t(z), [t(l) for l in log_s], t(gate)), t(gt), None, t(out_lens), sigma=sigma)
    assert abs((w * nll).sum() - float(bn)) <= 1e-5 * abs(float(bn))
    assert abs((w * gl).sum() - float(bg)) <= 1e-5 * abs(float(bg))


def test_ctc_rows_mean_is_the_oracle_batch_loss():
    g = torch.Generator().manual_seed(3)
    B, T, L, n_flows = 4, 30, 9, 3
    in_lens, out_lens = torch.tensor([9, 4, 7, 2]), torch.tensor([30, 12, 21, 5])
    lps = [torch.randn(B, T, L, generator=g) * 2 - 3 for _ in range(n_flows)]
    batch = float(O.flowtron_ctc_loss((None,) * 4 + (lps,), in_lens, out_lens))
    rows = np.zeros((n_flows, B))
    for f, lp in enumerate(lps):
        if f % 2:                                                # a back step's flipped time, back to natural time
            idx = O.back_step_index(out_lens, T)
            lp = torch.stack([lp[b][idx[:, b]] for b in range(B)])
        for b in range(B):
            rows[f, b] = float(O.attention_ctc_loss(lp[b:b + 1], in_lens[b:b + 1], out_lens[b:b + 1]))
    assert abs(rows.mean() - batch) <= 1e-5 * abs(batch)


def _reference_loss_module():
    if not ref_shims.runnable():
        pytest.skip("the reference modules are not available here")
    return ref_shims.import_flowtron()


def test_length_weighted_rows_are_the_reference_batch_loss():
    F = _reference_loss_module()
    z, log_s, gate, gt, out_lens, *_ = _random_outputs(1)
    nll, gl = rows_restated(z, log_s, gate, gt, out_lens)
    w = out_lens / out_lens.sum()
    t = torch.from_numpy
    out = (t(z), [t(l) for l in log_s], t(gate), None, None, None, None, None)
    ln, lg, _ = F.FlowtronLoss(sigma=1.0, gm_loss=False, gate_loss=True)(out, t(gt), None, t(out_lens))
    assert abs((w * nll).sum() - float(ln)) <= 1e-5 * abs(float(ln))
    assert abs((w * gl).sum() - float(lg)) <= 1e-5 * abs(float(lg))


@pytest.mark.parametrize("shared", [False, True])
def test_length_weighted_mixture_rows_are_the_reference_batch_loss(shared):
    F = _reference_loss_module()
    z, log_s, gate, gt, out_lens, mean, log_var, prob = _random_outputs(2)
    if shared:                                                   # fixed Gaussians: [1, M, K] buffers
        mean, log_var = mean[:1] * 3, np.zeros_like(log_var[:1])
    nll = gmm_rows_restated(z, log_s, out_lens, mean, log_var, prob)
    w = out_lens / out_lens.sum()
    t = torch.from_numpy
    out = (t(z), [t(l) for l in log_s], t(gate), None, None, t(mean), t(log_var), t(prob))
    ln, _, _ = F.FlowtronLoss(sigma=1.0, gm_loss=True, gate_loss=True)(out, t(gt), None, t(out_lens))
    assert abs((w * nll).sum() - float(ln)) <= 1e-5 * abs(float(ln)), ((w * nll).sum(), float(ln))
