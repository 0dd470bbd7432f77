"""The standalone Attention module on the GPU (ft_attention_fwd / ft_attention_bwd).

* Forward: every case of tests/golden/attention_*.npz (the unmodified reference, fp32 on the CPU) -- output, attn and
  attn_logprob within 1e-3 of the reference relative to each tensor's max |value| (DESIGN §2), at every position, padded keys
  included; attn exactly 0 at padded keys.
* Backward: torch.autograd of the oracle's fp64 attention_forward on the same weights, one upstream gradient at
  a time (output, attn, attn_logprob) and all together: per-tensor relative L2 and cosine for every input and weight, and per
  utterance for d_queries / d_keys / d_values.  Each bar is about 3x the worst value measured on an NVIDIA H100 80GB HBM3
  (700 W), written beside it; none is looser than tests/test_gpu_ar_step_backward.py's bar for the same upstream gradient.
* A forward + backward with CUDA in_lens captures in one CUDA graph without a host synchronisation; frozen weights and
  inputs that do not require grad keep .grad None.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import attention_oracle as AO  # noqa: E402
from conftest import record_parity  # noqa: E402
from flowtron_b200.flowtron import Attention  # noqa: E402
from oracle import flowtron_oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"

FWD_BAR = 1e-3           # measured worst 7.0e-6 (output, default_nomask): the projections are split fp16
# upstream gradient -> bars (inputs rel L2, per-utterance rel L2, weights rel L2), measured worst over GRAD_CASES in the
# comments (NVIDIA H100 80GB HBM3, 700 W).  "all" on the inputs, whole and per utterance, is held to
# test_gpu_ar_step_backward.py's d_mel bar for "all".
BARS = {
    "output": (9.4e-4, 1.1e-3, 9.2e-4),          # 3.1e-4, 3.8e-4, 3.1e-4
    "attn": (9.0e-4, 1.2e-3, 9.2e-4),            # 3.0e-4, 3.9e-4, 3.1e-4
    "attn_logprob": (9.0e-4, 1.2e-3, 9.1e-4),    # 3.0e-4, 3.9e-4, 3.0e-4
    "all": (5.8e-4, 5.8e-4, 9.2e-4),             # 3.1e-4, 3.6e-4, 3.1e-4
}
COS_BAR = 1.5e-7         # 1 - cosine; measured worst 4.9e-8


def _module(c, x):
    Dq, E, A = AO.DIMS[c["dims"]]
    m = Attention(n_mel_channels=Dq, n_speaker_dim=E - 512, n_text_channels=512, n_att_channels=A, temperature=c["temp"])
    m.load_state_dict(x["W"], strict=True)
    return m.to(DEV)


def _cu(t, dtype=None):
    return None if t is None else t.to(DEV, dtype=dtype)


def _rel(a, r):
    return ((a - r).abs().max() / r.abs().max().clamp_min(1e-3)).item()


@pytest.mark.parametrize("name", sorted(AO.CASES))
def test_forward_matches_reference(name):
    c = AO.CASES[name]
    x = AO.case_inputs(c)
    ref = np.load(os.path.join(AO.GOLDEN, f"attention_{name}.npz"))
    m = _module(c, x)
    with torch.no_grad():
        out, attn, lp = m(_cu(x["queries"]), _cu(x["keys"]), _cu(x["values"]), mask=_cu(x["mask"]), attn=_cu(x["attn"]),
                          attn_prior=_cu(x["prior"]))
    torch.cuda.synchronize()
    errs = {"output": _rel(out.cpu(), torch.from_numpy(ref["output"])), "attn": _rel(attn.cpu(), torch.from_numpy(ref["attn"]))}
    if c["given"]:
        assert lp is None
    else:
        errs["attn_logprob"] = _rel(lp.cpu(), torch.from_numpy(ref["attn_logprob"]))
    record_parity(f"attention_fwd/{name}", errs)
    for k, e in errs.items():
        assert e < FWD_BAR, (k, e)
    if x["mask"] is not None and not c["given"]:
        pad = x["mask"][..., 0][:, None, :].expand(-1, c["T"], -1)
        assert (attn.cpu()[pad] == 0).all()
    # in_lens gives the same result as the mask, bit for bit
    if x["lens"] is not None and not c["given"]:
        with torch.no_grad():
            o2, a2, l2 = m(_cu(x["queries"]), _cu(x["keys"]), _cu(x["values"]), attn_prior=_cu(x["prior"]),
                           in_lens=_cu(x["lens"], torch.int32))
        assert torch.equal(o2, out) and torch.equal(a2, attn) and torch.equal(l2, lp)


GRAD_CASES = ["default_ragged", "default_prior", "default_temp", "default_kv", "default_b40", "default_given",
              "ar_ragged", "ar_prior_temp", "ar_given", "ar_l700"]


def _upstream(c, which, out, attn, lp, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    gs = {}
    if which in ("output", "all"):
        gs["output"] = torch.randn(out.shape, generator=g, device=DEV)
    if which in ("attn", "all"):
        gs["attn"] = torch.randn(attn.shape, generator=g, device=DEV)
    if which in ("attn_logprob", "all") and lp is not None:
        gs["attn_logprob"] = torch.randn(lp.shape, generator=g, device=DEV)
    return gs


def _oracle_grads(c, params, q, k, v, at, mask, prior, gs, names):
    """torch.autograd of the fp64 restatement on the same weights and inputs: gradients of sum(gs[o] * o) w.r.t. `names`
    (inputs "queries" / "keys" / "values" / "attn" or parameter names); None where the upstream gradients do not reach."""
    W64 = {n: p.detach().double().requires_grad_() for n, p in params.items()}
    q64, k64 = q.detach().double().requires_grad_(), k.detach().double().requires_grad_()
    v64 = k64 if v is k else v.detach().double().requires_grad_()
    at64 = None if at is None else at.detach().double().requires_grad_()
    o64, a64, l64 = O.attention_forward({f"att.{n}": w for n, w in W64.items()}, "att", q64, k64, mask,
                                        None if prior is None else prior.double(), c["temp"], attn=at64, values=v64)
    outs64 = {"output": o64, "attn": a64, "attn_logprob": l64}
    leaves64 = {"queries": q64, "keys": k64, "values": v64, "attn": at64}
    t64 = [leaves64[n] if n in leaves64 else W64[n] for n in names]
    return torch.autograd.grad([outs64[n] for n in gs], t64, [gs[n].double() for n in gs], allow_unused=True)


def _compare(targets, got, want, params, bars):
    """Per-tensor relative L2 and cosine for every target, per utterance for the inputs; asserts the bars, returns the errors."""
    bar_in, bar_utt, bar_w = bars
    errs = {}
    for n, a, r, t in zip(targets, got, want, targets.values()):
        a = torch.zeros_like(t) if a is None else a           # a path the upstream gradient does not reach: exactly zero
        r = torch.zeros_like(t, dtype=torch.float64) if r is None else r.double()
        assert torch.isfinite(a).all(), n
        a = a.double()
        rn = r.norm().item()
        if rn == 0:
            assert a.abs().max().item() == 0, n
            continue
        rel = ((a - r).norm() / rn).item()
        cos = 1 - torch.nn.functional.cosine_similarity(a.flatten(), r.flatten(), dim=0).item()
        errs[f"{n}/rel"], errs[f"{n}/cos"] = rel, cos
        assert rel < (bar_w if n in params else bar_in), (n, rel)
        assert cos < COS_BAR, (n, cos)
        if n in ("queries", "keys", "values"):
            for b in range(a.size(1)):
                rb = r[:, b].norm().item()
                if rb == 0:
                    assert a[:, b].abs().max().item() == 0, (n, b)
                    continue
                eb = ((a[:, b] - r[:, b]).norm() / rb).item()
                errs[f"{n}/utt_max"] = max(errs.get(f"{n}/utt_max", 0.0), eb)
                assert eb < bar_utt, (n, b, eb)
    return errs


def _run_case(c, x, upstream):
    """Forward + backward of the module on a case with upstream(out, attn, logprob) -> {output name: gradient}; returns
    (targets, gradients, fp64 oracle gradients, parameters, mask)."""
    m = _module(c, x)
    params = dict(m.named_parameters())
    q, k = _cu(x["queries"]).requires_grad_(), _cu(x["keys"]).requires_grad_()
    v = _cu(x["values"]).requires_grad_() if c["kv"] else k
    at = _cu(x["attn"]).requires_grad_() if c["given"] else None
    mask, prior = _cu(x["mask"]), _cu(x["prior"])
    out, attn, lp = m(q, k, v, mask=mask, attn=at, attn_prior=prior)
    gs = upstream(out, attn, lp)
    outs = {"output": out, "attn": attn, "attn_logprob": lp}
    if c["given"]:
        targets = {"attn": at, **({"values": v} if c["kv"] else {"keys": k}),
                   "value.linear_layer.weight": params["value.linear_layer.weight"]}
    else:
        targets = {"queries": q, "keys": k, **({"values": v} if c["kv"] else {}), **params}
    got = torch.autograd.grad([outs[n] for n in gs], list(targets.values()), [gs[n] for n in gs], allow_unused=True)
    want = _oracle_grads(c, params, q, k, v, at, mask, prior, gs, list(targets))
    return targets, got, want, params


@pytest.mark.parametrize("which", ["output", "attn", "attn_logprob", "all"])
@pytest.mark.parametrize("name", GRAD_CASES)
def test_backward_matches_fp64_oracle(name, which):
    c = AO.CASES[name]
    if c["given"] and which == "attn_logprob":
        pytest.skip("no attn_logprob when attn is given")
    x = AO.case_inputs(c)
    targets, got, want, params = _run_case(c, x, lambda o, a, lp: _upstream(c, which, o, a, lp, 1000 + len(name)))
    errs = _compare(targets, got, want, params, BARS[which])
    record_parity(f"attention_bwd/{name}/{which}", errs)
    if x["mask"] is not None and not c["given"]:
        # keys past a row's length get no gradient at all
        dk = got[list(targets).index("keys")]
        for b, n_b in enumerate(x["lens"].tolist()):
            assert dk[n_b:, b].abs().max().item() == 0 if n_b < c["L"] else True


# Upstream gradients far below fp16's normal range (6.1e-5): a mean over B*A*T elements (1.95e-7 each at B = 8, A = 640,
# T = 1000) and randn * 1e-7.  The backward's fp16 operands carry them only through the device loss scale, which must be
# applied before any fp16 rounding, in both branches.
SMALL_CASES = {
    "given_b8_t1000": dict(AO.CASES["ar_given"], B=8, T=1000),
    "ragged": AO.CASES["default_ragged"],
    "ar_prior_temp": AO.CASES["ar_prior_temp"],
}


@pytest.mark.parametrize("kind", ["mean", "randn_1e-7"])
@pytest.mark.parametrize("name", sorted(SMALL_CASES))
def test_backward_small_upstream_gradients(name, kind):
    c = SMALL_CASES[name]
    x = AO.case_inputs(c)

    def upstream(out, attn, lp):
        outs = {"output": out} if c["given"] else {"output": out, "attn": attn, "attn_logprob": lp}
        if kind == "mean":
            return {n: torch.full_like(t, 1.0 / t.numel()) for n, t in outs.items()}
        g = torch.Generator(device=DEV).manual_seed(77)
        return {n: 1e-7 * torch.randn(t.shape, generator=g, device=DEV) for n, t in outs.items()}

    targets, got, want, params = _run_case(c, x, upstream)
    errs = _compare(targets, got, want, params, BARS["output" if c["given"] else "all"])
    record_parity(f"attention_bwd_small/{name}/{kind}", errs)


def test_graph_capture_with_in_lens_no_sync():
    c = AO.CASES["ar_prior_temp"]
    x = AO.case_inputs(c)
    m = _module(c, x)
    lens = torch.tensor([97], dtype=torch.int32, device=DEV)
    q, k = _cu(x["queries"]).requires_grad_(), _cu(x["keys"]).requires_grad_()
    prior = _cu(x["prior"])
    g = torch.Generator(device=DEV).manual_seed(3)
    go, ga, gl = (torch.randn(s, generator=g, device=DEV) for s in ((1, 640, 65), (1, 65, 160), (1, 65, 160)))

    def step():
        out, attn, lp = m(q, k, k, attn_prior=prior, in_lens=lens)
        return (out * go).sum() + (attn * ga).sum() + (lp * gl).sum(), out, attn

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            for t in (q, k, *m.parameters()):
                t.grad = None
            loss, _, _ = step()
            loss.backward()
    torch.cuda.current_stream().wait_stream(s)
    eager = [t.grad.clone() for t in (q, k, *m.parameters())]
    for t in (q, k, *m.parameters()):
        t.grad = None
    graph = torch.cuda.CUDAGraph()
    torch.cuda.set_sync_debug_mode("error")
    try:
        with torch.cuda.graph(graph):
            loss, out, attn = step()
            loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    graph.replay()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.isfinite(out).all() and (attn[0, :, 97:] == 0).all()
    for e, t in zip(eager, (q, k, *m.parameters())):
        err = ((t.grad - e).norm() / e.norm()).item()
        assert err < 1e-6, err                      # same kernels, same data: replay equals the eager step
    # the replayed step meets the fp64 oracle's bars, forward and every gradient, with the ragged in_lens (the oracle's mask is
    # built from the same lengths)
    mask = ~(torch.arange(160, device=DEV)[None, :] < lens[:, None].long())[..., None]
    params = dict(m.named_parameters())
    W64 = {f"att.{n}": p.detach().double() for n, p in params.items()}
    o64, a64, l64 = O.attention_forward(W64, "att", q.detach().double(), k.detach().double(), mask, prior.double(), c["temp"])
    assert _rel(out.detach().double(), o64) < FWD_BAR and _rel(attn.detach().double(), a64) < FWD_BAR
    targets = {"queries": q, "keys": k, **params}
    want = _oracle_grads(c, params, q, k, k, None, mask, prior, {"output": go, "attn": ga, "attn_logprob": gl}, list(targets))
    errs = _compare(targets, [t.grad for t in targets.values()], want, params, BARS["all"])
    record_parity("attention_bwd/graph_replay", errs)


def test_frozen_weights_and_inputs_keep_grad_none():
    c = AO.CASES["default_ragged"]
    x = AO.case_inputs(c)
    m = _module(c, x)
    m.key.linear_layer.weight.requires_grad_(False)
    m.v.linear_layer.weight.requires_grad_(False)
    q = _cu(x["queries"])                                 # does not require grad
    k = _cu(x["keys"]).requires_grad_()
    out, attn, lp = m(q, k, k, mask=_cu(x["mask"]))
    (out.sum() + lp.sum()).backward()
    assert q.grad is None
    assert m.key.linear_layer.weight.grad is None and m.v.linear_layer.weight.grad is None
    assert m.query.linear_layer.weight.grad is not None and m.value.linear_layer.weight.grad is not None
    assert k.grad is not None and torch.isfinite(k.grad).all()
    # forced weights: query / key / v are not used and get no gradient
    m2 = _module(c, x)
    at = _cu(AO.case_inputs(AO.CASES["default_given"])["attn"]).requires_grad_()
    out, a, lp = m2(q, k, k, attn=at)
    assert a is at and lp is None
    out.sum().backward()
    assert at.grad is not None and m2.value.linear_layer.weight.grad is not None
    assert all(getattr(m2, n).linear_layer.weight.grad is None for n in ("query", "key", "v"))
    # no_grad keeps nothing for a backward
    with torch.no_grad():
        out, _, _ = m(q, k, k, mask=_cu(x["mask"]))
    assert out.grad_fn is None
