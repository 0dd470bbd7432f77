"""CPU checks of the standalone Attention module: the oracle's fp64 restatement (attention_forward, which the flow step uses
too) against the reference's fixtures and against finite differences, the argument checks that run before any device work,
and the state_dict round trip with the reference module."""
from __future__ import annotations

import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import attention_oracle as AO  # noqa: E402
from flowtron_b200 import _lib  # noqa: E402
from flowtron_b200.flowtron import Attention  # noqa: E402
from oracle import flowtron_oracle as O  # noqa: E402
from oracle import ref_shims  # noqa: E402


def _f64(x):
    return None if x is None else x.double()


@pytest.mark.parametrize("name", sorted(AO.CASES))
def test_oracle_matches_reference_fixture(name):
    c = AO.CASES[name]
    ref = np.load(os.path.join(AO.GOLDEN, f"attention_{name}.npz"))
    x = AO.case_inputs(c)
    for k, v in AO.input_sums(x).items():          # the regenerated inputs are the ones the reference ran on
        assert float(ref[k]) == pytest.approx(v, rel=1e-12, abs=1e-9), k
    W = {f"att.{k}": v.double() for k, v in x["W"].items()}
    out, attn, lp = O.attention_forward(W, "att", _f64(x["queries"]), _f64(x["keys"]), x["mask"], _f64(x["prior"]), c["temp"],
                                        attn=_f64(x["attn"]), values=_f64(x["values"]))
    got = {"output": out, "attn": attn}
    if lp is not None:
        got["attn_logprob"] = lp
    assert ("attn_logprob" in ref.files) == (lp is not None)
    for k, t in got.items():
        r = torch.from_numpy(ref[k]).double()
        err = ((t - r).abs().max() / r.abs().max().clamp_min(1e-3)).item()     # (L = 1: attn_logprob is 0 everywhere)
        assert err < 2e-5, (k, err)                 # fp32 rounding of the reference's own computation
    if x["mask"] is not None:
        assert (torch.from_numpy(ref["attn"])[x["mask"][..., 0][:, None, :].expand(-1, c["T"], -1)] == 0).all()


@pytest.mark.parametrize("prior,given", [(False, False), (True, False), (False, True)])
def test_oracle_gradient_matches_finite_differences(prior, given):
    g = torch.Generator().manual_seed(5)
    T, B, L, Dq, E, A = 3, 2, 5, 4, 6, 8
    W = {f"att.{k}.linear_layer.weight": (0.5 * torch.randn(o, i, generator=g, dtype=torch.float64)).requires_grad_()
         for k, (o, i) in zip(AO.PRE, ((A, Dq), (A, E), (A, E), (1, A)))}
    q = torch.randn(T, B, Dq, generator=g, dtype=torch.float64, requires_grad=True)
    k = torch.randn(L, B, E, generator=g, dtype=torch.float64, requires_grad=True)
    v = torch.randn(L, B, E, generator=g, dtype=torch.float64, requires_grad=True)
    mask = ~(torch.arange(L)[None, :] < torch.tensor([5, 3])[:, None])[..., None]
    pr = torch.softmax(torch.randn(B, T, L, generator=g, dtype=torch.float64), 2) if prior else None
    at = torch.softmax(torch.randn(B, T, L, generator=g, dtype=torch.float64), 2).requires_grad_() if given else None
    names = list(W)

    def f(q, k, v, at, *ws):
        out, a, lp = O.attention_forward(dict(zip(names, ws)), "att", q, k, mask, pr, 0.7, attn=at, values=v)
        # padded keys: lp is log(1e-20 + ...) there with a prior, finite; keep every output in the check
        return (out, a) if lp is None else (out, a, lp)

    assert torch.autograd.gradcheck(f, (q, k, v, at, *W.values()), eps=1e-6, atol=1e-6, rtol=1e-5)


# ------------------------------------------------------------------------------------------------ argument checks (no device)
def _module(Dq=80, E=640, A=128):
    torch.manual_seed(0)
    return Attention(n_mel_channels=Dq, n_speaker_dim=E - 512, n_text_channels=512, n_att_channels=A)


def _inputs(T=4, B=2, L=6, Dq=80, E=640):
    return torch.randn(T, B, Dq), torch.randn(L, B, E), torch.randn(L, B, E)


def test_non_prefix_mask_raises():
    q, k, v = _inputs()
    mask = torch.zeros(2, 6, 1, dtype=torch.bool)
    mask[1, 2, 0] = True                           # a hole, valid keys after it
    with pytest.raises(ValueError, match="length mask"):
        _module()(q, k, v, mask=mask)


def test_empty_row_raises():
    q, k, v = _inputs()
    mask = torch.zeros(2, 6, 1, dtype=torch.bool)
    mask[0] = True
    with pytest.raises(ValueError, match="no valid key"):
        _module()(q, k, v, mask=mask)


def test_mask_and_in_lens_raises():
    q, k, v = _inputs()
    with pytest.raises(ValueError, match="not both"):
        _module()(q, k, v, mask=torch.zeros(2, 6, 1, dtype=torch.bool), in_lens=torch.tensor([6, 6]))


def test_text_longer_than_max_raises():
    q, k, v = _inputs(L=_lib.MAX_TEXT_LEN + 1)
    with pytest.raises(ValueError, match="MAX_TEXT_LEN"):
        _module()(q, k, v)


def test_prior_requiring_grad_raises():
    q, k, v = _inputs()
    with pytest.raises(NotImplementedError, match="attn_prior"):
        _module()(q, k, v, attn_prior=torch.rand(2, 4, 6, requires_grad=True))


@pytest.mark.parametrize("dims", [(84, 640, 128), (80, 644, 128), (80, 640, 132)])
def test_unaligned_sizes_raise_at_forward_not_construction(dims):
    Dq, E, A = dims
    m = _module(Dq, E, A)                          # constructing works: AR_Step and checkpoints are unaffected
    q, k, v = _inputs(Dq=Dq, E=E)
    with pytest.raises(NotImplementedError, match="multiples of 8"):
        m(q, k, v)


def test_cpu_tensors_raise():
    q, k, v = _inputs()
    with pytest.raises(_lib.FlowtronB200Error, match="CUDA"):
        _module()(q, k, v)


def test_state_dict_round_trip_with_reference_module():
    if not ref_shims.runnable():
        pytest.skip("the reference modules are not available")
    F = ref_shims.import_flowtron()
    for Dq, E, A in AO.DIMS.values():
        ours = _module(Dq, E, A)
        torch.manual_seed(1)
        ref = F.Attention(n_mel_channels=Dq, n_speaker_dim=E - 512, n_text_channels=512, n_att_channels=A)
        ref.load_state_dict(ours.state_dict(), strict=True)
        back = _module(Dq, E, A)
        for p in back.parameters():
            p.data.zero_()
        back.load_state_dict(ref.state_dict(), strict=True)
        sd = ours.state_dict()
        assert list(sd) == list(ref.state_dict()) == list(back.state_dict())
        assert all(torch.equal(sd[k], back.state_dict()[k]) for k in sd)
