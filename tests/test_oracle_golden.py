"""CPU: pin the oracle restatement against fixtures generated from the reference itself
(tests/make_golden.py, tests/make_golden_gmm.py), SURVEY.md §8c."""
import numpy as np
import pytest
import torch

from golden_fixtures import grad_sample_index, load
from oracle import flowtron_oracle as O
from oracle import stft_oracle as S
from flowtron_b200 import synth


def _valid_mask_T(out_lens, T):
    return (torch.arange(T)[:, None] < out_lens[None, :])


@pytest.mark.parametrize("tag", ["cfg1", "f2prior", "f2ragged"])
def test_train_forward_loss_grads_match_reference(tag):
    gold = load(f"train_{tag}.npz")
    n_flows, B, T, L = (int(gold[k]) for k in ("cfg_n_flows", "B", "T", "L"))
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=n_flows)
    p = {k: v.requires_grad_(True) for k, v in synth.synth_params(cfg, int(gold["seed"])).items()}
    # same call pattern as tests/make_golden.py (synth_batch re-sorts rows by text length)
    batch = synth.synth_batch(B, T, L, cfg, int(gold["seed"]),
                              out_lens={"cfg1": [128, 100], "f2prior": [96, 61, 80],
                                        "f2ragged": [64, 1, 33, 64, 17]}[tag],
                              with_prior=bool(gold["with_prior"]))
    assert np.array_equal(batch["out_lens"].numpy(), gold["out_lens"])
    out = O.flowtron_forward(p, batch["mel"], batch["speaker_ids"], batch["text"], batch["in_lens"],
                             batch["out_lens"], batch["attn_prior"])
    z, log_s_list, gate, attns, lps = out[:5]
    vm = _valid_mask_T(batch["out_lens"], T)
    # valid positions are the contract (pad independence, SURVEY §8a row 3); pads agree too here
    def close(a, b, tol=2e-5):
        a, b = torch.as_tensor(a), torch.as_tensor(b)
        err = (a - b).abs().max().item()
        assert err <= tol * max(1.0, b.abs().max().item()), err
    close(z.detach()[vm], torch.from_numpy(gold["z"])[vm])
    close(gate.detach()[vm], torch.from_numpy(gold["gate"])[vm])
    for i in range(n_flows):
        close(log_s_list[i].detach()[vm], torch.from_numpy(gold[f"log_s_{i}"])[vm])
        vmb = vm.t()
        close(attns[i].detach()[vmb], torch.from_numpy(gold[f"attn_{i}"])[vmb])
        lp_o, lp_g = lps[i].detach()[vmb], torch.from_numpy(gold[f"attn_logprob_{i}"])[vmb]
        fin = torch.isfinite(lp_g)
        close(lp_o[fin], lp_g[fin], 1e-4)
    nll, gl = O.flowtron_loss(out, batch["gate_target"], batch["in_lens"], batch["out_lens"])
    assert abs(float(nll.detach()) - float(gold["nll"])) < 1e-5
    assert abs(float(gl.detach()) - float(gold["gate_loss"])) < 1e-5
    (nll + gl).sum().backward()
    for name, t in p.items():
        g = t.grad.reshape(-1)
        gn = float(gold[f"gnorm::{name}"])
        assert abs(float(g.double().norm()) - gn) <= 2e-3 * gn + 1e-7, name
        samp = g[grad_sample_index(name, g.numel())]
        ref = torch.from_numpy(gold[f"gsamp::{name}"])
        assert (samp - ref).abs().max().item() <= 2e-3 * (ref.abs().max().item() + gn / np.sqrt(g.numel())) + 1e-8, name


def test_train_forward_matches_reference_at_baseline_shape():
    """cfg-2 shape (T=1000, L=150, prior on, log-mel statistics): oracle forward + losses vs the reference fixture."""
    gold = load("train_t1000.npz")
    n_flows, B, T, L = (int(gold[k]) for k in ("cfg_n_flows", "B", "T", "L"))
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=n_flows)
    p = synth.synth_params(cfg, int(gold["seed"]))
    batch = synth.synth_batch(B, T, L, cfg, int(gold["seed"]), out_lens=[1000, 873, 640, 512], in_lens=[150, 134, 98, 79],
                              with_prior=True, logmel_stats=True)
    assert np.array_equal(batch["out_lens"].numpy(), gold["out_lens"]) and np.array_equal(batch["in_lens"].numpy(), gold["in_lens"])
    with torch.no_grad():
        out = O.flowtron_forward(p, batch["mel"], batch["speaker_ids"], batch["text"], batch["in_lens"], batch["out_lens"],
                                 batch["attn_prior"], fast=True)
        nll, gl = O.flowtron_loss(out, batch["gate_target"], batch["in_lens"], batch["out_lens"])
    vm = _valid_mask_T(batch["out_lens"], T)
    for name, a, b in [("z", out[0], gold["z"]), ("gate", out[2], gold["gate"]), ("log_s_0", out[1][0], gold["log_s_0"]),
                       ("log_s_1", out[1][1], gold["log_s_1"])]:
        b = torch.from_numpy(b)
        err = (a[vm] - b[vm]).abs().max().item() / max(1.0, b[vm].abs().max().item())
        assert err <= 5e-5, (name, err)
    for i in range(n_flows):
        n0 = int(batch["out_lens"][0])
        assert (out[3][i][0, :n0] - torch.from_numpy(gold[f"attn_{i}_b0"])[:n0]).abs().max().item() <= 5e-5
    assert abs(float(nll) - float(gold["nll"])) < 1e-4 * abs(float(gold["nll"]))
    assert abs(float(gl) - float(gold["gate_loss"])) < 1e-4


def test_ctc_branch_matches_reference():
    """FlowtronLoss with use_ctc_loss (flowtron.py:245-274, 155-182): oracle loss_ctc and the gradients of
    nll + gate + ctc vs the reference fixture (2 flows: one forward, one back step; prior on)."""
    gold = load("train_f2ctc.npz")
    n_flows, B, T, L = (int(gold[k]) for k in ("cfg_n_flows", "B", "T", "L"))
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=n_flows)
    p = {k: v.requires_grad_(True) for k, v in synth.synth_params(cfg, int(gold["seed"])).items()}
    batch = synth.synth_batch(B, T, L, cfg, int(gold["seed"]), out_lens=[80, 47, 66], with_prior=True)
    out = O.flowtron_forward(p, batch["mel"], batch["speaker_ids"], batch["text"], batch["in_lens"], batch["out_lens"],
                             batch["attn_prior"])
    nll, gl = O.flowtron_loss(out, batch["gate_target"], batch["in_lens"], batch["out_lens"])
    ctc = O.flowtron_ctc_loss(out, batch["in_lens"], batch["out_lens"])
    assert abs(float(ctc.detach()) - float(gold["loss_ctc"])) <= 1e-5 * abs(float(gold["loss_ctc"]))
    (nll + gl + float(gold["ctc_weight"]) * ctc).sum().backward()
    for name, t in p.items():
        g = t.grad.reshape(-1)
        gn = float(gold[f"gnorm::{name}"])
        assert abs(float(g.double().norm()) - gn) <= 2e-3 * gn + 1e-7, name


@pytest.mark.parametrize("name", ["gmm_f2_fixed", "gmm_f3_learned", "gmm_b1_learned", "gmm_b1_fixed"])
def test_mixture_prior_matches_reference(name):
    """Flowtron with n_components > 1 and FlowtronLoss(gm_loss=True) (tests/make_golden_gmm.py): the oracle's MelEncoder
    embedding, mixture and losses against the reference's, padded frames holding random values."""
    gold = load(f"{name}.npz")
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=int(gold["n_flows"]), n_components=int(gold["K"]),
               fixed_gaussian=bool(gold["fixed_gaussian"]), mean_scale=float(gold["mean_scale"]))
    p = synth.synth_gmm_params(cfg, int(gold["seed"]))
    t = lambda k: torch.from_numpy(gold[k])
    with torch.no_grad():
        emb = O.mel_encoder_forward(p, t("mel"), t("out_lens"))
        out = O.flowtron_forward(p, t("mel"), t("speaker_ids"), t("text"), t("in_lens"), t("out_lens"),
                                 t("attn_prior") if int(gold["with_prior"]) else None, fast=True)
        losses = O.flowtron_loss(out, t("gate_target"), t("in_lens"), t("out_lens"), gm_loss=True)
        if int(gold["ctc"]):
            losses += (O.flowtron_ctc_loss(out, t("in_lens"), t("out_lens")),)
    for key, got in (("mel_embedding", emb), ("mean", out[5]), ("log_var", out[6]), ("prob", out[7])):
        ref = t(key)
        assert got.shape == ref.shape, key
        assert (got - ref).abs().max().item() <= 1e-5 * max(ref.abs().max().item(), 1e-30), key
    for key, got in zip(("loss", "gate_loss", "loss_ctc"), losses):
        assert abs(float(got) - float(gold[key])) <= 1e-5 * abs(float(gold[key])), key


@pytest.mark.parametrize("tag", ["b1", "b1gate", "b4nogate", "b1_t400", "b4nogate_t400"])
def test_infer_matches_reference(tag):
    gold = load(f"infer_{tag}.npz")
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=int(gold["cfg_n_flows"]), use_gate_layer=bool(gold["use_gate"]))
    p = synth.synth_params(cfg, int(gold["seed"]))
    if bool(gold["use_gate"]):
        key = [k for k in p if k.endswith("gate_layer.linear_layer.bias")][0]
        p[key] = torch.full_like(p[key], float(gold["gate_bias"]))
    B = int(gold["B"])
    with torch.no_grad():
        mel, _ = O.flowtron_infer(p, torch.from_numpy(gold["residual"]), torch.zeros(B, dtype=torch.long),
                                  torch.from_numpy(gold["text"]))
    ref = torch.from_numpy(gold["mel"])
    assert mel.shape == ref.shape
    assert (mel - ref).abs().max().item() <= 1e-4 * max(1.0, ref.abs().max().item())


def test_lstm_fast_equals_explicit():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(17, 3, 40, generator=g)
    w_ih, w_hh = torch.randn(64, 40, generator=g) * 0.2, torch.randn(64, 16, generator=g) * 0.2
    b1, b2 = torch.randn(64, generator=g) * 0.1, torch.randn(64, generator=g) * 0.1
    a = O.lstm_layer_explicit(x, w_ih, w_hh, b1, b2)
    b = O.lstm_layer_fast(x, w_ih, w_hh, b1, b2)
    assert (a - b).abs().max().item() < 1e-5


def test_invertibility_identity():
    """flowtron.py:932-954 (identity only; the shipped method is broken, SURVEY §4)."""
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=2, use_gate_layer=False)
    p = synth.synth_params(cfg, 3)
    g = torch.Generator().manual_seed(3)
    T, L = 24, 10
    zin = torch.randn(1, 80, T, generator=g) * 0.5
    text = torch.randint(0, 185, (1, L), generator=g)
    spk = torch.zeros(1, dtype=torch.long)
    with torch.no_grad():
        mel, _ = O.flowtron_infer(p, zin, spk, text)
        # forward uses the packed/masked encoder; with B=1 and full length it equals Encoder.infer
        out = O.flowtron_forward(p, mel, spk, text, torch.tensor([L]), torch.tensor([T]))
    z = out[0].permute(1, 2, 0)
    assert (z - zin).abs().max().item() < 1e-4


def test_back_step_index_is_involution():
    lens = torch.tensor([7, 1, 4, 10])
    idx = O.back_step_index(lens, 10)
    back = torch.gather(idx, 0, idx)
    assert torch.equal(back, torch.arange(10)[:, None].expand(10, 4))


def test_mel_frontend_matches_reference():
    gold = load("mel.npz")
    basis = S.slaney_mel_basis(22050, 1024, 80, 0.0, 8000.0)
    assert np.allclose(basis, gold["mel_basis"], atol=1e-7)
    for k in ("demo", "noise", "short", "quiet"):
        m = S.mel_spectrogram(torch.from_numpy(gold[f"y_{k}"]))
        ref = torch.from_numpy(gold[f"mel_{k}"])
        assert m.shape == ref.shape
        assert (m - ref).abs().max().item() < 1e-4, k


def test_beta_binomial_prior_matches_scipy():
    P, M = 9, 14
    ours = synth.beta_binomial_prior(P, M)
    ref = O.beta_binomial_prior(P, M)
    assert np.allclose(ours, ref, rtol=1e-9, atol=1e-12)


def test_radam_oracle_matches_reference_trajectory():
    """oracle.radam_oracle vs the unmodified reference RAdam + clip_grad_norm_ (tests/golden/radam.npz)."""
    from oracle import radam_oracle as R
    g = load("radam.npz")
    n = int(g["n_steps"])
    ps = [torch.from_numpy(g[f"p0_{i}"]) for i in range(3)]
    ms = [torch.zeros_like(p) for p in ps]
    vs = [torch.zeros_like(p) for p in ps]
    for s in range(n):
        grads = [torch.from_numpy(g[f"g{s}_{i}"]) for i in range(3)]
        total, coef = R.clip_coef(grads, float(g["max_norm"]))
        assert abs(float(total) - float(g[f"norm{s}"])) <= 1e-6 * float(total)
        for i in range(3):
            ps[i], ms[i], vs[i] = R.radam_step(ps[i], grads[i] * coef, ms[i], vs[i], s + 1, lr=1e-3, weight_decay=1e-6)
            torch.testing.assert_close(ps[i], torch.from_numpy(g[f"p{s + 1}_{i}"]), rtol=2e-6, atol=1e-7)
    for i in range(3):
        torch.testing.assert_close(ms[i], torch.from_numpy(g[f"m_{i}"]), rtol=2e-6, atol=1e-8)
        torch.testing.assert_close(vs[i], torch.from_numpy(g[f"v_{i}"]), rtol=2e-6, atol=1e-10)
