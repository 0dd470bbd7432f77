"""CPU: pin the data-layer restatements (oracle/data_oracle.py, oracle/stft_oracle.stft_transform, and the closed-form
prior the product's synthetic batches use) against outputs of the reference's own functions (tests/golden/
reference_checks.npz) and against scipy's beta-binomial."""
import os

import numpy as np
import torch

from oracle import data_oracle as D
from flowtron_b200 import synth
from oracle import stft_oracle as S

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def test_closed_form_prior_equals_scipy_loop():
    for P, M, s in [(7, 13, 1.0), (40, 200, 1.0), (23, 61, 0.5), (1, 5, 1.0)]:
        a = synth.beta_binomial_prior(P, M, s)
        b = D.beta_binomial_prior_distribution(P, M, s).numpy()
        assert a.shape == b.shape == (M, P)
        assert np.abs(a - b).max() <= 1e-12 + 1e-9 * np.abs(b).max()


def _ref():
    """Outputs of the reference's own functions on the inputs below (tests/make_golden.py reference_checks_case)."""
    return np.load(os.path.join(GOLDEN, "reference_checks.npz"))


def test_data_oracle_matches_reference_data_py():
    ref = _ref()
    assert torch.equal(torch.from_numpy(ref["prior_11_29"]), D.beta_binomial_prior_distribution(11, 29, 1.0))
    g = torch.Generator().manual_seed(0)
    batch = []
    for F_, P_ in [(29, 11), (40, 17), (5, 17), (33, 3)]:
        batch.append((torch.randn(80, F_, generator=g), torch.LongTensor([F_ % 3]), torch.randint(1, 100, (P_,), generator=g),
                      D.beta_binomial_prior_distribution(P_, F_, 1.0)))
    mine = D.collate(batch, 1, use_attn_prior=True)
    assert len(mine) == 7
    for i, b in enumerate(mine):
        a = torch.from_numpy(ref[f"collate_{i}"])
        assert a.shape == b.shape and torch.equal(a.float(), b.float())


def test_stft_transform_oracle_matches_reference():
    ref = _ref()
    y = torch.rand(2, 3000, generator=torch.Generator().manual_seed(3)) * 1.9 - 0.95
    assert torch.equal(y, torch.from_numpy(ref["stft_y"]))
    m, p = S.stft_transform(y)
    assert torch.allclose(m, torch.from_numpy(ref["stft_mag"]), atol=1e-6)
    assert torch.allclose(p, torch.from_numpy(ref["stft_phase"]), atol=1e-6)


def test_forced_alignment_branch_matches_reference_ar_step_infer():
    """AR_Step.infer / AR_Back_Step.infer with `attns` given (flowtron.py:585-588, 797): oracle vs the reference modules.
    (Flowtron.infer itself cannot be driven with attns in the reference: `reversed(attns)[i]` at :924 raises.)"""
    from oracle import flowtron_oracle as O
    ref = _ref()
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=2, use_gate_layer=False)
    params = synth.synth_params(cfg, 17)
    g = torch.Generator().manual_seed(2)
    T, L = 10, 6
    residual = torch.randn(T, 1, 80, generator=g) * 0.5
    enc = torch.randn(L, 1, 640, generator=g)
    attns = torch.softmax(torch.randn(T, L, generator=g), -1)
    r0, r1 = torch.from_numpy(ref["forced_r0"]), torch.from_numpy(ref["forced_r1"])
    with torch.no_grad():
        o0, _ = O.ar_step_infer(params, O.flow_prefix(0), residual, enc, attns=attns)
        o1, _ = O.ar_back_step_infer(params, "flows.1", residual, enc, attns=attns)
    assert (r0 - o0).abs().max().item() <= 1e-5 * r0.abs().max().item()
    assert (r1 - o1).abs().max().item() <= 1e-5 * r1.abs().max().item()
