"""GPU: texts longer than 256 tokens, up to FT_MAX_TEXT_LEN = 1024.  Training (forward, FlowtronLoss with the prior and
CTC, backward) and Flowtron.infer against reference-generated fixtures (tests/make_golden_long_text.py); the attention-CTC
kernel's several-states-per-thread variant against torch's nn.CTCLoss restatement; the invertibility identity and the
text encoder at L = 1024.  Bars are those of the short-text tests (test_gpu_flowtron_train.py, test_gpu_infer.py,
test_gpu_ctc.py, test_gpu_encoder.py)."""
import pytest
import torch

from conftest import record_parity
from golden_fixtures import grad_sample_index, load
from oracle import flowtron_oracle as O
from flowtron_b200 import synth

pytestmark = pytest.mark.gpu


def rel_err(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-12)


@pytest.mark.parametrize("tag", ["long400", "long1024"])
def test_training_matches_reference_goldens(tag):
    """long400: shared-memory attention kernels past 256 keys, the attention overlap (T = 420) and a finite CTC loss over
    801 states; long1024: the global-row attention kernels (L > 672)."""
    from flowtron_b200 import _lib
    from flowtron_b200.flowtron import Flowtron, FlowtronLoss
    gold = load(f"train_{tag}.npz")
    n_flows, B, T, L = (int(gold[k]) for k in ("cfg_n_flows", "B", "T", "L"))
    w = float(gold["ctc_weight"])
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=n_flows)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    model = Flowtron(**cfg)
    model.load_state_dict(synth.synth_params(cfg, int(gold["seed"])), strict=True)
    model = model.cuda().train()
    model.encoder.p_dropout = 0.0
    batch = synth.synth_batch(B, T, L, cfg, int(gold["seed"]), out_lens=gold["out_lens"].tolist(),
                              in_lens=gold["in_lens"].tolist(), with_prior=bool(gold["with_prior"]))
    cu = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in batch.items()}
    out = model(cu["mel"], cu["speaker_ids"], cu["text"], cu["in_lens"], cu["out_lens"], cu["attn_prior"])
    z, log_s_list, gate, attns, lps = out[:5]
    crit = FlowtronLoss(sigma=1.0, gate_loss=True, use_ctc_loss=True, ctc_loss_weight=w)
    nll, gl, ctc = crit(out, cu["gate_target"], cu["in_lens"], cu["out_lens"])
    (nll + gl + ctc * w).sum().backward()
    torch.cuda.synchronize()
    assert _lib.device_status() == 0

    vm = (torch.arange(T)[:, None] < batch["out_lens"][None, :])
    st = int(gold.get("t_stride", 1))           # per-frame outputs stored at every st-th frame
    vs = vm[::st]
    errs = {"z": rel_err(z.detach().cpu()[::st][vs], torch.from_numpy(gold["z"])[vs]),
            "gate": rel_err(gate.detach().cpu()[::st][vs], torch.from_numpy(gold["gate"])[vs])}
    for i in range(n_flows):
        errs[f"log_s_{i}"] = rel_err(log_s_list[i].detach().cpu()[::st][vs], torch.from_numpy(gold[f"log_s_{i}"])[vs])
        if f"attn_{i}" in gold:
            errs[f"attn_{i}"] = rel_err(attns[i].detach().cpu()[:, ::st][vs.t()], torch.from_numpy(gold[f"attn_{i}"])[vs.t()])
            errs[f"attn_logprob_{i}"] = rel_err(lps[i].detach().cpu()[:, ::st][vs.t()],
                                                torch.from_numpy(gold[f"attn_logprob_{i}"])[vs.t()])
        else:                                   # one utterance's attention stored
            a0 = attns[i][0, ::st].detach().cpu()
            n0 = int(vs[:, 0].sum())
            errs[f"attn_{i}_b0"] = rel_err(a0[:n0], torch.from_numpy(gold[f"attn_{i}_b0"])[:n0])
    errs["nll"] = abs(float(nll) - float(gold["nll"])) / abs(float(gold["nll"]))
    errs["gate_loss"] = abs(float(gl) - float(gold["gate_loss"])) / abs(float(gold["gate_loss"]))
    ref_ctc = float(gold["loss_ctc"])
    errs["loss_ctc"] = abs(float(ctc) - ref_ctc) / max(abs(ref_ctc), 1e-6) if ref_ctc != 0.0 else abs(float(ctc))

    # gradients: norm and the fixture's 32 sampled entries of every parameter, 1e-2 relative (the floor 1e-4 of the
    # largest gradient norm covers tensors whose gradient is analytically ~0, as in test_gpu_flowtron_train.py)
    gmax = max(float(gold[f"gnorm::{n}"]) for n, _ in model.named_parameters())
    worst_norm, worst_samp, worst = 0.0, 0.0, ""
    for name, p in model.named_parameters():
        g = p.grad.detach().reshape(-1).cpu()
        gn = float(gold[f"gnorm::{name}"])
        e_norm = abs(float(g.double().norm()) - gn) / (gn + 1e-4 * gmax)
        r = torch.from_numpy(gold[f"gsamp::{name}"]).double()
        s = g[grad_sample_index(name, g.numel())].double()
        e_samp = float((s - r).norm()) / (float(r.norm()) + 1e-4 * gmax)
        worst_norm = max(worst_norm, e_norm)
        if e_samp > worst_samp:
            worst_samp, worst = e_samp, name
    errs["grad_norm_worst"], errs["grad_samples_worst"] = worst_norm, worst_samp
    print(f"train_{tag} errors:", {k: f"{v:.2e}" for k, v in errs.items()}, "worst sampled gradient:", worst)
    record_parity(f"train_{tag}", errs)
    bad = {k: v for k, v in errs.items() if not k.startswith("grad") and not v <= 1e-3}
    assert not bad, bad
    assert worst_norm <= 1e-2 and worst_samp <= 1e-2, (worst_norm, worst_samp, worst)


@pytest.mark.parametrize("L", [272, 513, 1024])
@pytest.mark.parametrize("time_reversed", [False, True])
def test_ctc_kernel_long_texts_match_torch_ctc(L, time_reversed):
    from flowtron_b200 import _lib
    from flowtron_b200.flowtron import AttentionCTCLoss
    g = torch.Generator().manual_seed(L)
    T = L + 48
    in_lens = torch.tensor([L, L - 37, 5, L // 2])
    out_lens = torch.tensor([T, T - 20, 9, L // 2 - 3])            # last row: fewer frames than tokens -> inf -> zero_infinity
    B = len(in_lens)
    lp_nat = (torch.randn(B, T, L, generator=g) * 2.0 - 3.0)
    ref_in = lp_nat.clone().requires_grad_(True)
    ref = O.attention_ctc_loss(ref_in, in_lens, out_lens, -1.0)
    ref.backward()
    if time_reversed:
        idx = O.back_step_index(out_lens, T)
        lp_dev = torch.zeros_like(lp_nat)
        for b in range(B):
            lp_dev[b][idx[:, b]] = lp_nat[b]
    else:
        lp_dev = lp_nat
    x = lp_dev.cuda().requires_grad_(True)
    loss = AttentionCTCLoss(blank_logprob=-1)(None, in_lens.cuda(), out_lens.cuda(), x[:, None], time_reversed=time_reversed)
    loss.backward()
    torch.cuda.synchronize()
    assert _lib.device_status() == 0
    gx = x.grad.cpu()
    if time_reversed:
        idx = O.back_step_index(out_lens, T)
        gx = torch.stack([gx[b][idx[:, b]] for b in range(B)])
    e_loss = abs(float(loss) - float(ref)) / abs(float(ref))
    e_grad = (gx - ref_in.grad).abs().max().item() / ref_in.grad.abs().max().item()
    record_parity(f"ctc_kernel_L{L}_rev{int(time_reversed)}", {"loss": e_loss, "grad": e_grad})
    # the log-space sums run over ~L + T steps: fp32 rounding of alpha + beta + nll (|nll| ~ 1e3-1e4) sets the gradient bar
    assert e_loss <= 1e-5 and e_grad <= 2e-3, (e_loss, e_grad)


def _infer_model(cfg, seed, gate_bias=None):
    from flowtron_b200.flowtron import Flowtron
    p = synth.synth_params(cfg, seed)
    if gate_bias is not None:
        key = [k for k in p if k.endswith("gate_layer.linear_layer.bias")][0]
        p[key] = torch.full_like(p[key], gate_bias)
    m = Flowtron(**cfg)
    m.load_state_dict(p, strict=True)
    return m.cuda().eval()


@pytest.mark.parametrize("tag", ["long1024", "long600gate"])
def test_infer_matches_reference_goldens(tag):
    from flowtron_b200 import _lib
    gold = load(f"infer_{tag}.npz")
    use_gate = bool(gold["use_gate"])
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=int(gold["cfg_n_flows"]), use_gate_layer=use_gate)
    m = _infer_model(cfg, int(gold["seed"]), float(gold["gate_bias"]) if use_gate else None)
    B = int(gold["B"])
    with torch.no_grad():
        mel, _ = m.infer(torch.from_numpy(gold["residual"]).cuda(), torch.zeros(B, dtype=torch.long, device="cuda"),
                         torch.from_numpy(gold["text"]).cuda())
    torch.cuda.synchronize()
    assert _lib.device_status() == 0
    ref = torch.from_numpy(gold["mel"])
    assert tuple(mel.shape) == tuple(ref.shape), (mel.shape, ref.shape)
    err = (mel.cpu() - ref).abs().max().item() / ref.abs().max().item()
    record_parity(f"infer_{tag}", {"mel": err})
    assert err <= 1e-3, err


def test_invertibility_forward_of_infer_1024_tokens():
    """forward(infer(z)) == z at L = 1024 (test_gpu_infer.py's identity).  T = 360 >= 320 also runs the training forward's
    attention overlap on the global-row attention kernel."""
    from flowtron_b200 import _lib
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=2, use_gate_layer=False)
    m = _infer_model(cfg, 3)
    g = torch.Generator().manual_seed(4)
    T, L = 360, 1024
    zin = (torch.randn(1, 80, T, generator=g) * 0.5).cuda()
    text = torch.randint(0, 185, (1, L), generator=g).cuda()
    spk = torch.zeros(1, dtype=torch.long, device="cuda")
    with torch.no_grad():
        mel, attn = m.infer(zin, spk, text)
        out = m(mel, spk, text, torch.tensor([L], device="cuda"), torch.tensor([T], device="cuda"))
    torch.cuda.synchronize()
    assert _lib.device_status() == 0
    assert len(attn) == 2 and len(attn[0]) == T and attn[0][0].shape[-1] == L
    z = out[0].permute(1, 2, 0)
    err = (z - zin).abs().max().item() / zin.abs().max().item()
    record_parity("infer_roundtrip_L1024", {"z_roundtrip": err})
    assert err <= 2e-3, err


def _encoder_model(seed):
    from flowtron_b200.flowtron import Flowtron
    cfg = dict(synth.DEFAULT_MODEL_CONFIG)
    m = Flowtron(**cfg)
    params = synth.synth_params(cfg, seed)
    m.load_state_dict(params, strict=True)
    return m.cuda(), params


@pytest.mark.parametrize("lens", [[1024, 700], None])
def test_encoder_1024_tokens_forward_and_backward(lens):
    """The text encoder has no length limit of its own: at L = 1024, masked (ragged lengths) and unmasked (inference
    path forward; full lengths backward), against the oracle restatement and fp32 autograd through it."""
    m, p = _encoder_model(6)
    B, L = 2, 1024
    x = torch.randn(B, 512, L, generator=torch.Generator().manual_seed(13)) * 0.7
    m.eval()
    with torch.no_grad():
        if lens is None:
            ours = m.encoder.infer(x.cuda())
            ref = O.encoder_forward(p, x, None, infer=True)
        else:
            ours = m.encoder(x.cuda(), torch.tensor(lens).cuda())
            ref = O.encoder_forward(p, x, torch.tensor(lens))
    e_fwd = rel_err(ours, ref)
    assert e_fwd < 1e-3, e_fwd

    in_lens = torch.tensor(lens if lens is not None else [L] * B)
    m.train()
    m.encoder.p_dropout = 0.0
    w_out = torch.randn(B, L, 512, generator=torch.Generator().manual_seed(99)) * 0.05
    xc = x.cuda().requires_grad_(True)
    out = m.encoder(xc, in_lens.cuda())
    (out * w_out.cuda()).sum().backward()
    ours = {"x": xc.grad.cpu()}
    for n, q in m.encoder.named_parameters():
        ours["encoder." + n] = q.grad.cpu()
    pr = {k: v.clone().requires_grad_(k.startswith("encoder.")) for k, v in p.items()}
    xr = x.clone().requires_grad_(True)
    ref_out = O.encoder_forward(pr, xr, in_lens)
    (ref_out * w_out[:, :ref_out.shape[1]]).sum().backward()
    ref = {"x": xr.grad}
    ref.update({k: v.grad for k, v in pr.items() if k.startswith("encoder.")})
    worst_norm, worst_cos, worst = 0.0, 1.0, ""
    wscale = ref["encoder.convolutions.0.0.conv.weight"].double().norm().item()
    for k, r in ref.items():
        o, r = ours[k].double(), r.double()
        if k.endswith("conv.bias"):             # zero gradient in front of an instance norm: rounding noise on both sides
            assert o.norm().item() < 1e-3 * wscale, (k, o.norm().item(), wscale)
            continue
        ne = (o - r).norm().item() / max(r.norm().item(), 1e-30)
        cos = (o * r).sum().item() / max(o.norm().item() * r.norm().item(), 1e-30)
        if ne > worst_norm:
            worst_norm, worst = ne, k
        worst_cos = min(worst_cos, cos)
    record_parity(f"encoder_L1024_{'masked' if lens else 'full'}", {"fwd": e_fwd, "rel_l2_worst": worst_norm,
                                                                    "cos_worst": worst_cos})
    assert worst_norm < 1e-2 and worst_cos > 0.9999, (worst, worst_norm, worst_cos)
