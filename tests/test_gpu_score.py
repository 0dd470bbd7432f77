"""GPU: Flowtron.score (per-utterance NLL, gate and attention-CTC losses; ft_nll_rows, ft_gmm_nll_rows, ft_attn_ctc_loss)
against the reference's FlowtronLoss applied one utterance at a time (tests/make_golden_score.py), against FlowtronLoss on
the same batch, row by row against B = 1 calls, under CUDA-graph replay, at 1024 tokens; and Flowtron.test_invertibility."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, record_parity
from flowtron_b200 import synth

pytestmark = pytest.mark.gpu


def _model(n_flows, seed, K=0, fixed=True, mean_scale=0.0, use_gate=True):
    from flowtron_b200.flowtron import Flowtron
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=n_flows, use_gate_layer=use_gate)
    if K > 1:
        cfg.update(n_components=K, fixed_gaussian=fixed, mean_scale=mean_scale)
        p = synth.synth_gmm_params(cfg, seed)
    else:
        p = synth.synth_params(cfg, seed)
    m = Flowtron(**cfg)
    m.load_state_dict(p, strict=True)
    return m.cuda().eval()


def _fixture(name):
    gold = dict(np.load(os.path.join(GOLDEN, name + ".npz")))
    if "attn_prior" not in gold:                 # large priors are not stored: the generator's own rule rebuilds them
        B, _, T = gold["mel"].shape
        L = gold["text"].shape[1]
        prior = np.zeros((B, T, L), np.float32)
        for b, (nl, n) in enumerate(zip(gold["in_lens"], gold["out_lens"])):
            prior[b, :n, :nl] = synth.beta_binomial_prior(int(nl), int(n)).astype(np.float32)
        gold["attn_prior"] = prior
    return gold


def _fixture_model(gold):
    return _model(int(gold["n_flows"]), int(gold["seed"]), int(gold["K"]), bool(gold["fixed_gaussian"]),
                  float(gold["mean_scale"]))


def _inputs(gold):
    return (torch.from_numpy(gold["mel"]).cuda(), torch.from_numpy(gold["speaker_ids"]).cuda(),
            torch.from_numpy(gold["text"]).cuda(), gold["in_lens"].tolist(), gold["out_lens"].tolist(),
            torch.from_numpy(gold["attn_prior"]).cuda())


def _rel_errors(got, ref):
    """|got - ref| / |ref| per entry; an entry the reference zeroes (an infinite CTC cost, zero_infinity) must be 0."""
    got, ref = got.detach().cpu().double().numpy(), np.asarray(ref, np.float64)
    assert got.shape == ref.shape, (got.shape, ref.shape)
    zero = ref == 0
    assert (got[zero] == 0).all(), (got, ref)
    return np.abs(got - ref)[~zero] / np.abs(ref[~zero])


@pytest.mark.parametrize("name", ["score_f2", "score_f3", "score_gmm_learned", "score_gmm_fixed", "score_l1024"])
def test_rows_match_reference_fixtures(name):
    from flowtron_b200 import _lib
    gold = _fixture(name)
    model = _fixture_model(gold)
    mel, spk, text, in_lens, out_lens, prior = _inputs(gold)
    model.train()                               # score runs with eval semantics in any mode
    try:
        s = model.score(mel, spk, text, in_lens, out_lens, prior)
    finally:
        model.eval()
    torch.cuda.synchronize()
    assert _lib.device_status() == 0
    assert not any(v.requires_grad for v in s.values())
    errs = {k: _rel_errors(s[k], gold[k]) for k in ("nll", "gate", "ctc")}
    record_parity(f"score_{name}", {k: float(v.max()) if v.size else 0.0 for k, v in errs.items()})
    print(name, {k: f"{v.max():.2e}" for k, v in errs.items() if v.size})
    for k, v in errs.items():
        assert (v <= 1e-3).all(), (k, v)


@pytest.mark.parametrize("n_flows, K, fixed", [(2, 0, True), (3, 0, True), (2, 4, False), (3, 8, True)])
def test_length_weighted_rows_equal_flowtron_loss(n_flows, K, fixed):
    from flowtron_b200.flowtron import FlowtronLoss
    model = _model(n_flows, 700 + n_flows + K, K, fixed, 3.0 if fixed else 0.0)
    B, T, L = 9, 120, 30
    b = synth.synth_batch(B, T, L, synth.DEFAULT_MODEL_CONFIG, 800 + n_flows, with_prior=True, logmel_stats=True)
    cu = {k: v.cuda() for k, v in b.items()}
    with torch.no_grad():
        out = model(cu["mel"], cu["speaker_ids"], cu["text"], cu["in_lens"], cu["out_lens"], cu["attn_prior"])
        crit = FlowtronLoss(sigma=1.0, gm_loss=K > 1, gate_loss=True, use_ctc_loss=True, ctc_loss_weight=1.0)
        loss, gate_loss, loss_ctc = crit(out, cu["gate_target"], cu["in_lens"], cu["out_lens"])
        s = model.score(cu["mel"], cu["speaker_ids"], cu["text"], cu["in_lens"], cu["out_lens"], cu["attn_prior"])
        s_gt = model.score(cu["mel"], cu["speaker_ids"], cu["text"], cu["in_lens"], cu["out_lens"], cu["attn_prior"],
                           gate_target=cu["gate_target"])
    w = cu["out_lens"].double() / cu["out_lens"].sum()
    got = {"loss": float((w * s["nll"].double()).sum()), "gate_loss": float((w * s["gate"].double()).sum()),
           "loss_ctc": float(s["ctc"].double().mean())}
    ref = {"loss": float(loss), "gate_loss": float(gate_loss), "loss_ctc": float(loss_ctc)}
    errs = {k: abs(got[k] - ref[k]) / abs(ref[k]) for k in got}
    record_parity(f"score_batch_f{n_flows}_k{K}", errs)
    assert max(errs.values()) <= 1e-5, (errs, got, ref)
    for k in ("nll", "gate", "ctc"):                 # the collate's gate target is what gate_target=None builds
        assert torch.equal(s[k], s_gt[k]), k


@pytest.fixture(scope="module")
def ragged40():
    """B = 40 (two launches of at most 32), lengths on both sides of _ATTN_OVERLAP_MIN_T."""
    from flowtron_b200.flowtron import _ATTN_OVERLAP_MIN_T
    assert _ATTN_OVERLAP_MIN_T == 320
    g = torch.Generator().manual_seed(41)
    B, T, L = 40, 420, 60
    out_lens = torch.randint(60, T + 1, (B,), generator=g)
    out_lens[:4] = torch.tensor([T, 319, 320, 60])
    in_lens = torch.randint(8, L + 1, (B,), generator=g)
    in_lens[0] = L
    b = synth.synth_batch(B, T, L, dict(synth.DEFAULT_MODEL_CONFIG), 42, out_lens=out_lens, in_lens=in_lens,
                          with_prior=True, logmel_stats=True)
    return {k: v.cuda() for k, v in b.items()}


@pytest.mark.parametrize("n_flows", [2, 3])
def test_rows_equal_single_utterance_calls(ragged40, n_flows):
    from flowtron_b200 import _lib
    model = _model(n_flows, 900 + n_flows)
    b = ragged40
    il, ol = b["in_lens"].tolist(), b["out_lens"].tolist()
    assert min(ol) < 320 <= max(ol)
    with torch.no_grad():
        s = model.score(b["mel"], b["speaker_ids"], b["text"], il, ol, b["attn_prior"])
        singles = [model.score(b["mel"][i:i + 1, :, :n], b["speaker_ids"][i:i + 1], b["text"][i:i + 1, :nl], [nl], [n],
                               b["attn_prior"][i:i + 1, :n, :nl]) for i, (nl, n) in enumerate(zip(il, ol))]
    torch.cuda.synchronize()
    assert _lib.device_status() == 0
    mismatched = []
    for i, one in enumerate(singles):
        for k in ("nll", "gate"):
            if not torch.equal(s[k][i:i + 1], one[k]):
                mismatched.append((i, ol[i], k, float(s[k][i]), float(one[k][0])))
        if not torch.equal(s["ctc"][:, i:i + 1], one["ctc"]):
            mismatched.append((i, ol[i], "ctc", s["ctc"][:, i].tolist(), one["ctc"][:, 0].tolist()))
    record_parity(f"score_rows_vs_b1_f{n_flows}", {"mismatched": len(mismatched)})
    assert not mismatched, mismatched[:6]


def test_deterministic_graph_replay_and_memory(ragged40):
    model = _model(2, 950)
    b = {k: v[:12] for k, v in ragged40.items()}
    g = torch.Generator().manual_seed(43)
    B, T, L = 12, 300, 48
    static = {"mel": b["mel"][:, :, :T].contiguous(), "spk": b["speaker_ids"].clone(), "text": b["text"][:, :L].contiguous(),
              "in_lens": torch.randint(5, L + 1, (B,), generator=g).cuda(),
              "out_lens": torch.randint(40, T + 1, (B,), generator=g).cuda()}
    call = lambda: model.score(static["mel"], static["spk"], static["text"], static["in_lens"], static["out_lens"])
    first, second = call(), call()
    for k in ("nll", "gate", "ctc"):
        assert torch.equal(first[k], second[k]), k
        assert not first[k].requires_grad
    torch.cuda.synchronize()
    del first, second
    m0 = torch.cuda.memory_allocated()
    r = call()
    torch.cuda.synchronize()
    del r
    assert torch.cuda.memory_allocated() == m0
    torch.cuda.set_sync_debug_mode("error")             # CUDA lengths: not one host synchronisation
    try:
        call()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        call()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = call()
    for rep in range(2):
        mel = (torch.randn(B, 80, T, generator=g) * 2.0 - 5.5).clamp_(-11.5, 2.0).cuda()
        text = torch.randint(0, 185, (B, L), generator=g).cuda()
        static["mel"].copy_(mel)
        static["text"].copy_(text)
        static["in_lens"].copy_(torch.randint(1, L + 1, (B,), generator=g).cuda())
        static["out_lens"].copy_(torch.randint(1, T + 1, (B,), generator=g).cuda())
        graph.replay()
        eager = call()
        torch.cuda.synchronize()
        for k in ("nll", "gate", "ctc"):
            assert torch.equal(captured[k], eager[k]), (rep, k)
    del graph


def test_invertibility_of_infer_and_forward():
    """Flowtron.test_invertibility on the model and input of test_gpu_infer.py::test_invertibility_forward_of_infer, at
    that test's bar (2e-3 of max |z|)."""
    model = _model(2, 3, use_gate=False)
    g = torch.Generator().manual_seed(3)
    T, L = 40, 12
    zin = (torch.randn(1, 80, T, generator=g) * 0.5).cuda()
    text = torch.randint(0, 185, (1, L), generator=g).cuda()
    spk = torch.zeros(1, dtype=torch.long, device="cuda")
    err = model.test_invertibility(zin, spk, text)
    rel = float(err) / zin.abs().max().item()
    record_parity("score_test_invertibility", {"mean_abs_err_rel": rel})
    assert err.dim() == 0 and 0 < rel <= 2e-3, rel
    model3 = _model(3, 5, use_gate=False)                  # an odd number of flows: compared front to front
    rel3 = float(model3.test_invertibility(zin, spk, text)) / zin.abs().max().item()
    assert 0 < rel3 <= 2e-3, rel3
