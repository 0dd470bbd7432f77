"""H100: Flowtron with the Gaussian-mixture prior (n_components > 1) against the reference fixtures of
tests/make_golden_gmm.py (MelEncoder embedding, mean / log_var / prob, the three losses, gradients), the mixture-NLL kernels
and the mel encoder against the float64 oracle, the mel encoder's 64-row slicing, padding independence, train-mode dropout,
a CUDA-graph training step and inference on a mixture model."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from flowtron_b200 import synth
from oracle import flowtron_oracle as O

pytestmark = pytest.mark.gpu

CASES = ["gmm_f2_fixed", "gmm_f3_learned", "gmm_b1_learned", "gmm_b1_fixed"]


def _case(name):
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=int(g["n_flows"]), n_components=int(g["K"]),
               fixed_gaussian=bool(g["fixed_gaussian"]), mean_scale=float(g["mean_scale"]))
    return g, cfg, synth.synth_gmm_params(cfg, int(g["seed"]))


def _model(cfg, params):
    from flowtron_b200.flowtron import Flowtron
    m = Flowtron(**cfg)
    m.load_state_dict(params, strict=True)
    return m.cuda()


def _inputs(g):
    t = lambda k: torch.from_numpy(g[k]).cuda()
    return dict(mel=t("mel"), speaker_ids=t("speaker_ids"), text=t("text"), in_lens=t("in_lens"), out_lens=t("out_lens"),
                gate_target=t("gate_target"), attn_prior=t("attn_prior") if int(g["with_prior"]) else None)


def _run(model, g, d):
    from flowtron_b200.flowtron import FlowtronLoss
    emb = {}
    h = model.mel_encoder.register_forward_hook(lambda m, i, o: emb.__setitem__("x", o.detach().clone()))
    out = model(d["mel"], d["speaker_ids"], d["text"], d["in_lens"], d["out_lens"], d["attn_prior"])
    h.remove()
    ctc = bool(int(g["ctc"]))
    crit = FlowtronLoss(sigma=1.0, gm_loss=True, gate_loss=True, use_ctc_loss=ctc, ctc_loss_weight=1.0 if ctc else 0.0)
    losses = crit(out, d["gate_target"], d["in_lens"], d["out_lens"])
    return emb["x"], out, losses


def _rel(a, b):
    return (a.detach().float().cpu() - b).abs().max().item() / max(b.abs().max().item(), 1e-30)


@pytest.mark.parametrize("name", CASES)
def test_matches_reference_fixtures(name):
    g, cfg, params = _case(name)
    model = _model(cfg, params).eval()
    d = _inputs(g)
    mel_before = d["mel"].clone()
    emb, out, (loss, gate_loss, loss_ctc) = _run(model, g, d)
    torch.cuda.synchronize()
    assert torch.equal(d["mel"], mel_before)                           # the caller's mel is not written
    for key, t in (("mel_embedding", emb), ("mean", out[5]), ("log_var", out[6]), ("prob", out[7])):
        ref = torch.from_numpy(g[key])
        assert t.shape == ref.shape, key
        if ref.abs().max() > 0:
            assert _rel(t, ref) < 1e-3, (key, _rel(t, ref))
        else:
            assert t.abs().max().item() == 0.0, key
    for key, t in (("loss", loss), ("gate_loss", gate_loss), ("loss_ctc", loss_ctc)):
        ref = float(g[key])
        assert abs(float(t.sum()) - ref) <= 1e-4 * max(abs(ref), 1e-6), (key, float(t.sum()), ref)
    (loss + gate_loss + loss_ctc).sum().backward()
    torch.cuda.synchronize()
    named = dict(model.named_parameters())
    for k in [f[len("gidx_"):] for f in g.files if f.startswith("gidx_")]:
        gr = named[k].grad
        assert gr is not None, k
        if k.endswith(".0.conv.bias"):
            # a bias in front of an instance norm has a zero gradient; the reference's is rounding noise (~1e-8 of the weight's)
            assert gr.norm().item() <= 1e-3 * named[k.replace(".bias", ".weight")].grad.norm().item(), k
            continue
        got = gr.reshape(-1)[torch.from_numpy(g[f"gidx_{k}"]).long().cuda()].double().cpu()
        ref = torch.from_numpy(g[f"grad_{k}"]).double()
        cos = torch.dot(got, ref) / (got.norm() * ref.norm())
        assert cos >= 0.9999, (k, float(cos))
        assert (got - ref).abs().max() <= 1e-2 * ref.abs().max(), (k, float((got - ref).abs().max() / ref.abs().max()))
        assert abs(gr.norm().item() / float(g[f"gnorm_{k}"]) - 1.0) <= 1e-2, k


@pytest.mark.parametrize("K", [2, 8, 32])
@pytest.mark.parametrize("per_row", [True, False])
def test_mixture_kernels_match_float64(K, per_row):
    from flowtron_b200.flowtron import _GmmNllFn
    g = torch.Generator().manual_seed(K * 2 + per_row)
    T, B, M = 70, 3, 80
    lens = torch.tensor([70, 33, 1])
    Bm = B if per_row else 1
    z = torch.randn(T, B, M, generator=g, dtype=torch.float64) * 2
    mean = torch.randn(Bm, M, K, generator=g, dtype=torch.float64) * 2
    log_var = torch.rand(Bm, M, K, generator=g, dtype=torch.float64) * 40 - 20          # [-20, 20]
    prob = torch.softmax(torch.randn(B, K, generator=g, dtype=torch.float64) * 3, dim=1)
    # the restatement runs on the fp32-rounded inputs the kernels see
    z, mean, log_var, prob = (t.float().double() for t in (z, mean, log_var, prob))
    z[T - 1, 2] = float("nan")                                                        # past row 2's length: ignored
    leaves = [t.clone().requires_grad_(True) for t in (z, mean, log_var, prob)]
    ref, _ = O.flowtron_loss((torch.nan_to_num(leaves[0]), [], None, None, None, *leaves[1:]), None, None, lens,
                             gate_loss=False, gm_loss=True)
    ref.backward()
    cu = [t.detach().float().cuda().requires_grad_(per_row or i in (0, 3)) for i, t in enumerate((z, mean, log_var, prob))]
    got = _GmmNllFn.apply(cu[0], lens.cuda(), cu[1], cu[2], cu[3])
    got.backward()
    torch.cuda.synchronize()
    assert abs(got.item() - ref.item()) <= 1e-5 * abs(ref.item()), (got.item(), ref.item())
    valid = (torch.arange(T)[:, None] < lens[None, :])[..., None].expand(T, B, M)
    dz_ref = torch.where(valid, leaves[0].grad, torch.zeros(()))
    assert torch.isfinite(cu[0].grad).all() and (cu[0].grad.cpu()[~valid] == 0).all()
    checks = [("dz", cu[0].grad, dz_ref), ("dprob", cu[3].grad, leaves[3].grad)]
    if per_row:
        checks += [("dmean", cu[1].grad, leaves[1].grad), ("dlog_var", cu[2].grad, leaves[2].grad)]
    for key, a, b in checks:
        assert _rel(a, b) < 1e-4, (key, _rel(a, b))
    # fixed summation order: a second call is bit-identical
    again = _GmmNllFn.apply(cu[0].detach(), lens.cuda(), cu[1].detach(), cu[2].detach(), cu[3].detach())
    assert again.item() == got.item()


def test_batch_of_70_runs_as_64_plus_6_and_matches_the_restatement():
    g, cfg, params = _case("gmm_f3_learned")
    model = _model(cfg, params).eval()
    B, T = 70, 24
    gen = torch.Generator().manual_seed(5)
    lens = torch.randint(3, T + 1, (B,), generator=gen)
    lens[17] = T
    mel = torch.randn(B, 80, T, generator=gen) * 2 - 4
    with torch.no_grad():
        emb = model.mel_encoder(mel.cuda(), lens.cuda())
        ref = O.mel_encoder_forward({k: v.double() for k, v in params.items()}, mel.double(), lens)
        assert _rel(emb, ref) < 1e-3, _rel(emb, ref)
        # the whole batch's longest row divides every slice: row 0..63 of the 70-row run equal a 64-row run only up to that scale
        head = model.mel_encoder(mel[:64].cuda(), lens[:64].cuda())
    scale = float(lens[:64].max()) / float(lens.max())
    assert torch.allclose(emb[:64], head * scale, rtol=1e-5, atol=1e-7)
    # flows over 70 rows (32 + 32 + 6 launches) with the prior: finite losses
    from flowtron_b200.flowtron import FlowtronLoss
    b = synth.synth_batch(B, T, 8, cfg, 9, out_lens=lens.tolist())
    d = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in b.items()}
    out = model(d["mel"], d["speaker_ids"], d["text"], d["in_lens"], d["out_lens"])
    loss, gl, _ = FlowtronLoss(gm_loss=True)(out, d["gate_target"], d["in_lens"], d["out_lens"])
    assert torch.isfinite(loss).all() and out[5].shape == (B, 80, 4)


def test_padded_frames_are_ignored():
    g, cfg, params = _case("gmm_f2_fixed")
    model = _model(cfg, params).eval()
    d = _inputs(g)
    with torch.no_grad():
        e0, o0, l0 = _run(model, g, d)
        pad = torch.arange(d["mel"].size(2), device="cuda")[None, None, :] >= d["out_lens"][:, None, None]
        d2 = dict(d, mel=d["mel"].masked_fill(pad, float("nan")))
        keep = d2["mel"].clone()
        e1, o1, l1 = _run(model, g, d2)
    assert torch.equal(e0, e1) and torch.equal(o0[7], o1[7]) and torch.equal(l0[0], l1[0])
    assert torch.equal(d2["mel"].isnan(), keep.isnan()) and torch.equal(d2["mel"].nan_to_num(), keep.nan_to_num())


def _train_setup(name="gmm_f3_learned"):
    from flowtron_b200.flowtron import FlowtronLoss
    from flowtron_b200.radam import RAdam
    g, cfg, params = _case(name)
    model = _model(cfg, params).train()
    d = _inputs(g)
    crit = FlowtronLoss(sigma=1.0, gm_loss=True, gate_loss=True)
    opt = RAdam(model.parameters(), lr=1e-4, weight_decay=1e-6, capturable=True)
    return g, model, d, crit, opt


def test_train_mode_dropout_is_seeded_and_training_lowers_the_loss():
    g, model, d, crit, opt = _train_setup()
    enc = model.mel_encoder
    with torch.no_grad():
        enc.eval()
        e_eval = enc(d["mel"], d["out_lens"])
        enc.train()
        rng0 = enc._rng_state(d["mel"].device).clone()
        e1 = enc(d["mel"], d["out_lens"])
        enc._rng.copy_(rng0)
        e2 = enc(d["mel"], d["out_lens"])
        e3 = enc(d["mel"], d["out_lens"])
        enc.p_dropout = 0.0
        e_nodrop = enc(d["mel"], d["out_lens"])
        enc.p_dropout = 0.5
    assert torch.equal(e1, e2) and not torch.equal(e2, e3)
    assert not torch.allclose(e1, e_eval) and torch.allclose(e_nodrop, e_eval, rtol=0, atol=0)
    model.encoder.p_dropout = enc.p_dropout = 0.0                      # a fixed objective for the descent check
    for grp in opt.param_groups:
        grp["lr"] = 1e-3
    losses = []
    for _ in range(6):
        opt.zero_grad()
        out = model(d["mel"], d["speaker_ids"], d["text"], d["in_lens"], d["out_lens"], d["attn_prior"])
        nll, gl, _ = crit(out, d["gate_target"], d["in_lens"], d["out_lens"])
        (nll + gl).sum().backward()
        opt.clip_grad_norm_(1.0)
        opt.step()
        losses.append(float(nll))
    assert all(np.isfinite(losses)) and losses[-1] < losses[0], losses
    assert all(torch.isfinite(p).all() for p in model.parameters())


def test_training_step_replays_bit_identically_from_a_cuda_graph():
    g, model, d, crit, opt = _train_setup("gmm_f2_fixed")
    loss_static = torch.zeros((), device="cuda")

    def body():
        opt.zero_grad()
        out = model(d["mel"], d["speaker_ids"], d["text"], d["in_lens"], d["out_lens"], d["attn_prior"])
        nll, gl, _ = crit(out, d["gate_target"], d["in_lens"], d["out_lens"])
        loss = (nll + gl).sum()
        loss.backward()
        opt.clip_grad_norm_(1.0)
        opt.step()
        loss_static.copy_(loss.detach())

    for _ in range(2):
        body()
    torch.cuda.synchronize()
    rngs = [model.mel_encoder._rng_state(d["mel"].device), model.encoder._rng_state(d["mel"].device)]
    graph = torch.cuda.CUDAGraph()
    opt.zero_grad()
    torch.cuda.synchronize()
    with torch.cuda.graph(graph):
        body()
    torch.cuda.synchronize()
    # the loss and the gradients depend on the weights and the dropout states only: restore both before each replay
    snap = {k: v.clone() for k, v in model.state_dict().items()}
    rng0 = [r.clone() for r in rngs]
    runs = []
    for _ in range(2):
        model.load_state_dict(snap)
        for r, r0 in zip(rngs, rng0):
            r.copy_(r0)
        graph.replay()
        torch.cuda.synchronize()
        runs.append((loss_static.clone(), [p.grad.clone() for p in model.parameters() if p.grad is not None]))
    assert torch.isfinite(runs[0][0])
    assert torch.equal(runs[0][0], runs[1][0])
    assert len(runs[0][1]) == len(list(model.parameters()))
    # the mixture's gradients are bit-identical; the mel encoder's split-K weight-gradient GEMMs and instance-norm affines add
    # atomically (as the text encoder's and the flows' do), so its gradients agree to rounding
    names = [n for n, p in model.named_parameters()]
    for n, a, b in zip(names, runs[0][1], runs[1][1]):
        if n.startswith("gaussian_mixture."):
            assert torch.equal(a, b), n
        elif n.startswith("mel_encoder."):
            assert (a - b).abs().max() <= 1e-3 * max(a.abs().max().item(), 1e-30), n


def test_inference_ignores_the_mixture_modules():
    from flowtron_b200.flowtron import Flowtron
    g, cfg, params = _case("gmm_f3_learned")
    gm = _model(cfg, params).eval()
    base_cfg = dict(cfg, n_components=0)
    base = Flowtron(**base_cfg)
    base.load_state_dict({k: v for k, v in params.items() if not k.startswith(("mel_encoder.", "gaussian_mixture."))}, strict=True)
    base = base.cuda().eval()
    gen = torch.Generator().manual_seed(3)
    residual = torch.randn(2, 80, 30, generator=gen).cuda()
    text = torch.randint(1, cfg["n_text"], (2, 9), generator=gen).cuda()
    spk = torch.zeros(2, dtype=torch.long, device="cuda")
    with torch.no_grad():
        a, _ = gm.infer(residual[:1], spk[:1], text[:1], gate_threshold=1.1)
        b, _ = base.infer(residual[:1], spk[:1], text[:1], gate_threshold=1.1)
        lens = torch.tensor([9, 6])
        ab = gm.infer_batch(residual, spk, text, lens, gate_threshold=1.1)
        bb = base.infer_batch(residual, spk, text, lens, gate_threshold=1.1)
    assert torch.equal(a, b)
    for x, y in zip(ab if isinstance(ab, (tuple, list)) else [ab], bb if isinstance(bb, (tuple, list)) else [bb]):
        if torch.is_tensor(x):
            assert torch.equal(x, y)
