"""CPU: the C-ABI declaration of ft_nll_rows / ft_gmm_nll_rows and their host-side errors, and the per-utterance loss
terms as the oracle's FlowtronLoss on each row alone: their length-weighted means are FlowtronLoss's batch losses (the
oracle's, and the reference's own module where it can be imported), and on the oracle's forward of a mixture model they
are the reference's rows."""
import os
import re

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT
from flowtron_b200 import synth
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


# ---------------------------------------------------------------------------------------------- the oracle, row by row
def rows(out, gate_target, out_lens, sigma=1.0, gm_loss=False):
    """Per-utterance (nll [B], gate [B]) in float64: the oracle's FlowtronLoss on each row alone, cut to its own length, as
    tests/make_golden_score.py applies the reference's.  out: a forward output (z, log_s_list, gate, _, _, mean, log_var,
    prob)."""
    z, log_s, gate, _, _, mean, log_var, prob = out
    own = lambda t, b: None if t is None else (t if t.size(0) == 1 else t[b:b + 1]).double()
    nll, gl = np.zeros(len(out_lens)), np.zeros(len(out_lens))
    for b, n in enumerate(out_lens.tolist()):
        cut = lambda t: t[:n, b:b + 1].double()
        row = (cut(z), [cut(l) for l in log_s], cut(gate), None, None, own(mean, b), own(log_var, b), own(prob, b))
        nll[b], gl[b] = (float(v) for v in O.flowtron_loss(row, gate_target[b:b + 1, :n].double(), None, out_lens[b:b + 1],
                                                           sigma=sigma, gm_loss=gm_loss))
    return nll, gl


def _random_outputs(seed, B=5, T=23, M=80, n_flows=3, K=4):
    """A forward output (z, log_s_list, gate, None, None, mean, log_var, prob), gate_target and out_lens, float32."""
    g = np.random.default_rng(seed)
    t = lambda a: torch.from_numpy(a.astype(np.float32))
    out_lens = torch.tensor([23, 7, 15, 1, 19][:B])
    z = t(g.standard_normal((T, B, M)))
    log_s = [t(0.1 * g.standard_normal((T, B, M))) for _ in range(n_flows)]
    gate = t(2 * g.standard_normal((T, B, 1)))
    gate_target = (torch.arange(T)[None, :] >= (out_lens[:, None] - 1)).float()
    mean = t(g.standard_normal((B, M, K)))
    log_var = t(0.3 * g.standard_normal((B, M, K)))
    prob = t(g.dirichlet(np.ones(K), B))
    return (z, log_s, gate, None, None, mean, log_var, prob), gate_target, out_lens


@pytest.mark.parametrize("sigma", [1.0, 0.7])
def test_length_weighted_rows_are_the_oracle_batch_loss(sigma):
    out, gt, out_lens = _random_outputs(0)
    nll, gl = rows(out, gt, out_lens, sigma)
    w = (out_lens / out_lens.sum()).numpy()
    bn, bg = O.flowtron_loss(out, gt, None, out_lens, sigma=sigma)
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


@pytest.mark.parametrize("name", ["score_gmm_learned", "score_gmm_fixed"])
def test_oracle_mixture_rows_match_reference_fixtures(name):
    """The oracle's MelEncoder, mixture and flows on the fixture's padded batch, its loss row by row, against the
    reference's rows (tests/make_golden_score.py)."""
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=int(g["n_flows"]), n_components=int(g["K"]),
               fixed_gaussian=bool(g["fixed_gaussian"]), mean_scale=float(g["mean_scale"]))
    p = synth.synth_gmm_params(cfg, int(g["seed"]))
    t = lambda k: torch.from_numpy(g[k])
    out_lens = t("out_lens")
    with torch.no_grad():
        out = O.flowtron_forward(p, t("mel"), t("speaker_ids"), t("text"), t("in_lens"), out_lens, t("attn_prior"), fast=True)
    gate_target = (torch.arange(g["mel"].shape[2])[None, :] >= (out_lens[:, None] - 1)).float()
    nll, gl = rows(out, gate_target, out_lens, gm_loss=True)
    for key, got in (("nll", nll), ("gate", gl)):
        err = np.abs(got - g[key]) / np.abs(g[key])
        assert err.max() <= 1e-5, (key, err)


def _reference_loss_module():
    if not ref_shims.runnable():
        pytest.skip("the reference modules are not available here")
    return ref_shims.import_flowtron()


def test_length_weighted_rows_are_the_reference_batch_loss():
    F = _reference_loss_module()
    out, gt, out_lens = _random_outputs(1)
    nll, gl = rows(out, gt, out_lens)
    w = (out_lens / out_lens.sum()).numpy()
    ln, lg, _ = F.FlowtronLoss(sigma=1.0, gm_loss=False, gate_loss=True)(out, gt, None, out_lens)
    assert abs((w * nll).sum() - float(ln)) <= 1e-5 * abs(float(ln))
    assert abs((w * gl).sum() - float(lg)) <= 1e-5 * abs(float(lg))


@pytest.mark.parametrize("shared", [False, True])
def test_length_weighted_mixture_rows_are_the_reference_batch_loss(shared):
    F = _reference_loss_module()
    out, gt, out_lens = _random_outputs(2)
    if shared:                                                   # fixed Gaussians: [1, M, K] buffers
        out = out[:5] + (out[5][:1] * 3, torch.zeros_like(out[6][:1]), out[7])
    nll, _ = rows(out, gt, out_lens, gm_loss=True)
    w = (out_lens / out_lens.sum()).numpy()
    ln, _, _ = F.FlowtronLoss(sigma=1.0, gm_loss=True, gate_loss=True)(out, gt, None, out_lens)
    assert abs((w * nll).sum() - float(ln)) <= 1e-5 * abs(float(ln)), ((w * nll).sum(), float(ln))
