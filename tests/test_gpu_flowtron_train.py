"""GPU parity (through the C ABI): Flowtron.forward + FlowtronLoss + backward vs fixtures generated from the
reference itself (tests/golden/train_*.npz) and vs the CPU oracle.  Tolerance: 1e-3 of the tensor's max |value|
(north_star: 'within 1e-3 relative fp32') for z / log_s / gate / attn / attn_logprob on VALID positions;
losses 1e-4 relative... (see each assert); gradients 1e-2 relative per tensor."""
import pytest
import torch

from conftest import record_parity
from golden_fixtures import load
from flowtron_b200 import synth

pytestmark = pytest.mark.gpu

OUT_LENS = {"cfg1": [128, 100], "f2prior": [96, 61, 80], "f2ragged": [64, 1, 33, 64, 17]}


def build_model(cfg, seed, device="cuda"):
    from flowtron_b200.flowtron import Flowtron
    model = Flowtron(**cfg)
    model.load_state_dict(synth.synth_params(cfg, seed), strict=True)
    return model.to(device).eval()


def rel_err(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-12)


@pytest.mark.parametrize("tag", ["cfg1", "f2prior", "f2ragged"])
def test_forward_loss_backward_match_reference_goldens(tag):
    from flowtron_b200 import _lib
    from flowtron_b200.flowtron import FlowtronLoss
    gold = load(f"train_{tag}.npz")
    n_flows, B, T, L = (int(gold[k]) for k in ("cfg_n_flows", "B", "T", "L"))
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=n_flows)
    # any torch GEMM or convolution left on the path runs in true fp32 for a parity test
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    model = build_model(cfg, int(gold["seed"]))
    batch = synth.synth_batch(B, T, L, cfg, int(gold["seed"]), out_lens=OUT_LENS[tag], with_prior=bool(gold["with_prior"]))
    dev = "cuda"
    cu = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in batch.items()}
    model.train()
    model.encoder.p_dropout = 0.0      # the (random) encoder dropout disabled, like the golden generator
    for p in model.parameters():
        p.requires_grad_(True)
    out = model(cu["mel"], cu["speaker_ids"], cu["text"], cu["in_lens"], cu["out_lens"], cu["attn_prior"])
    z, log_s_list, gate, attns, lps = out[:5]
    crit = FlowtronLoss(sigma=1.0, gate_loss=True)
    nll, gl, _ = crit(out, cu["gate_target"], cu["in_lens"], cu["out_lens"])
    (nll + gl).sum().backward()
    torch.cuda.synchronize()
    assert _lib.device_status() == 0

    vm = (torch.arange(T)[:, None] < batch["out_lens"][None, :])
    errs = {}
    errs["z"] = rel_err(z.detach().cpu()[vm], torch.from_numpy(gold["z"])[vm])
    errs["gate"] = rel_err(gate.detach().cpu()[vm], torch.from_numpy(gold["gate"])[vm])
    for i in range(n_flows):
        errs[f"log_s_{i}"] = rel_err(log_s_list[i].detach().cpu()[vm], torch.from_numpy(gold[f"log_s_{i}"])[vm])
        errs[f"attn_{i}"] = rel_err(attns[i].detach().cpu()[vm.t()], torch.from_numpy(gold[f"attn_{i}"])[vm.t()])
        errs[f"attn_logprob_{i}"] = rel_err(lps[i].detach().cpu()[vm.t()], torch.from_numpy(gold[f"attn_logprob_{i}"])[vm.t()])
    errs["nll"] = abs(float(nll) - float(gold["nll"])) / abs(float(gold["nll"]))
    errs["gate_loss"] = abs(float(gl) - float(gold["gate_loss"])) / abs(float(gold["gate_loss"]))
    print("forward errors:", {k: f"{v:.2e}" for k, v in errs.items()})
    record_parity(f"train_{tag}_forward", errs)
    bad = {k: v for k, v in errs.items() if not v <= 1e-3}
    assert not bad, bad

    # ---- gradients.  Backward tensor-core operands are bf16 (8-bit significand): per-element noise of a few 1e-3
    # relative is inherent, so the gate is per tensor: norm within 1e-2 of the reference's (fixture) and cosine
    # >= 0.999 / relative L2 <= 4e-2 against the full CPU-oracle gradient (the oracle is pinned to the reference in
    # tests/test_oracle_golden.py).  Tensors whose true gradient is analytically ~0 (conv biases feeding an
    # instance norm) are compared on an absolute scale.
    from oracle import flowtron_oracle as O
    op = {k: v.clone().requires_grad_(True) for k, v in synth.synth_params(cfg, int(gold["seed"])).items()}
    oout = O.flowtron_forward(op, batch["mel"], batch["speaker_ids"], batch["text"], batch["in_lens"], batch["out_lens"],
                              batch["attn_prior"], fast=True)
    onll, ogl = O.flowtron_loss(oout, batch["gate_target"], batch["in_lens"], batch["out_lens"])
    (onll + ogl).sum().backward()
    _assert_grads_match(f"train_{tag}", model, op, {n: float(gold[f"gnorm::{n}"]) for n, _ in model.named_parameters()})


def _assert_grads_match(tag, model, op, gnorm):
    """Every parameter gradient of `model` against the CPU oracle's (op[name].grad): norm within 1e-2 of gnorm[name],
    relative L2 <= 4e-2 and cosine >= 0.999."""
    gmax = max(gnorm.values())
    rows, bad = [], {}
    for name, p in model.named_parameters():
        g = p.grad.detach().reshape(-1).double().cpu()
        r = op[name].grad.reshape(-1).double()
        gn = gnorm[name]
        e_norm = abs(float(g.norm()) - gn) / (gn + 1e-4 * gmax)
        rel_l2 = float((g - r).norm()) / (float(r.norm()) + 1e-4 * gmax)
        cos = float((g @ r) / (g.norm() * r.norm() + 1e-30)) if gn > 1e-4 * gmax else 1.0
        rows.append((name, e_norm, rel_l2, cos))
        if not (e_norm <= 1e-2 and rel_l2 <= 4e-2 and cos >= 0.999):   # tightened once the fp16-scaled backward landed
            bad[name] = (e_norm, rel_l2, cos)
    rows.sort(key=lambda x: -x[2])
    record_parity(f"{tag}_grads", {"norm_err_worst": max(r[1] for r in rows), "rel_l2_worst": max(r[2] for r in rows),
                                   "cos_worst": min(r[3] for r in rows), "worst_tensor": rows[0][0]})
    print("worst grads (name, norm err, rel L2, cosine):", [(n, f"{a:.1e}", f"{b:.1e}", f"{c:.5f}") for n, a, b, c in rows[:8]])
    assert not bad, bad


@pytest.mark.parametrize("T", [77, 200, 250, 347])
def test_chunked_schedules_match_oracle(T):
    """The flow steps' chunked schedules (csrc/ar_step.cu) at the shapes where they change: lstm layers 0/1 run in 100-step
    chunks, one chunk apart (T = 77: one chunk; 200: two; 250: a ragged 50-step tail), and from T = 320 on the attention
    LSTM runs in 256-step chunks under its attention (347 = 256 + 91).  Forward outputs and every parameter gradient of a
    training step against the CPU oracle, at the bars of the reference-golden test above."""
    from flowtron_b200 import _lib
    from flowtron_b200.flowtron import FlowtronLoss
    from oracle import flowtron_oracle as O
    B, L, seed = 5, 12, 9
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=2)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    model = build_model(cfg, seed).train()
    model.encoder.p_dropout = 0.0
    batch = synth.synth_batch(B, T, L, cfg, seed, with_prior=True)
    cu = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in batch.items()}
    out = model(cu["mel"], cu["speaker_ids"], cu["text"], cu["in_lens"], cu["out_lens"], cu["attn_prior"])
    nll, gl, _ = FlowtronLoss(sigma=1.0, gate_loss=True)(out, cu["gate_target"], cu["in_lens"], cu["out_lens"])
    (nll + gl).sum().backward()
    torch.cuda.synchronize()
    assert _lib.device_status() == 0

    op = {k: v.clone().requires_grad_(True) for k, v in synth.synth_params(cfg, seed).items()}
    oout = O.flowtron_forward(op, batch["mel"], batch["speaker_ids"], batch["text"], batch["in_lens"], batch["out_lens"],
                              batch["attn_prior"], fast=True)
    onll, ogl = O.flowtron_loss(oout, batch["gate_target"], batch["in_lens"], batch["out_lens"])
    (onll + ogl).sum().backward()
    vm = (torch.arange(T)[:, None] < batch["out_lens"][None, :])
    errs = {"z": rel_err(out[0].detach().cpu()[vm], oout[0].detach()[vm]),
            "gate": rel_err(out[2].detach().cpu()[vm], oout[2].detach()[vm])}
    for i in range(cfg["n_flows"]):
        errs[f"log_s_{i}"] = rel_err(out[1][i].detach().cpu()[vm], oout[1][i].detach()[vm])
        errs[f"attn_{i}"] = rel_err(out[3][i].detach().cpu()[vm.t()], oout[3][i].detach()[vm.t()])
    errs["nll"] = abs(float(nll) - float(onll)) / abs(float(onll))
    record_parity(f"chunked_t{T}_forward", errs)
    bad = {k: v for k, v in errs.items() if not v <= 1e-3}
    assert not bad, bad
    _assert_grads_match(f"chunked_t{T}", model, op, {n: float(op[n].grad.norm()) for n, _ in model.named_parameters()})


def test_zero_init_identity_flow():
    """Known-answer test from the reference's own init (flowtron.py:652-653): conv.weight = conv.bias = 0
    => z == mel and log_s == 0 exactly."""
    from flowtron_b200.flowtron import Flowtron
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=2)
    torch.manual_seed(0)
    model = Flowtron(**cfg).cuda().eval()
    batch = synth.synth_batch(3, 40, 12, cfg, 11, out_lens=[40, 7, 22])
    cu = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in batch.items()}
    with torch.no_grad():
        out = model(cu["mel"], cu["speaker_ids"], cu["text"], cu["in_lens"], cu["out_lens"])
    z = out[0].permute(1, 2, 0)
    assert torch.equal(z, cu["mel"])
    assert all(float(ls.abs().max()) == 0.0 for ls in out[1])


def test_pad_independence():
    """Valid outputs must not depend on pad contents (SURVEY §8a row 3)."""
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=2)
    model = build_model(cfg, 77)
    batch = synth.synth_batch(3, 48, 16, cfg, 5, out_lens=[48, 20, 31])
    cu = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in batch.items()}
    mel2 = cu["mel"].clone()
    T = 48
    tm = (torch.arange(T, device="cuda")[None, :] >= cu["out_lens"][:, None])
    mel2 = torch.where(tm[:, None, :], torch.full_like(mel2, 3.7), mel2)
    with torch.no_grad():
        a = model(cu["mel"], cu["speaker_ids"], cu["text"], cu["in_lens"], cu["out_lens"])
        b = model(mel2, cu["speaker_ids"], cu["text"], cu["in_lens"], cu["out_lens"])
    vm = ~tm.t()
    assert torch.equal(a[0][vm], b[0][vm])
    for x, y in zip(a[1], b[1]):
        assert torch.equal(x[vm], y[vm])


def test_two_stream_half_batches_equal_single_stream():
    """Flowtron.forward splits B >= 8 into two half batches on two CUDA streams (64-SM recurrence kernels running
    concurrently).  Utterances are independent, so outputs and parameter gradients must equal the single-stream run."""
    from flowtron_b200.flowtron import FlowtronLoss
    torch.backends.cudnn.allow_tf32 = False
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=2)
    batch = synth.synth_batch(8, 40, 14, cfg, 21, with_prior=True)
    cu = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in batch.items()}
    res = []
    for n_streams in (1, 2):
        model = build_model(cfg, 31)
        model.train()
        model.encoder.p_dropout = 0.0
        model.n_streams = n_streams
        out = model(cu["mel"], cu["speaker_ids"], cu["text"], cu["in_lens"], cu["out_lens"], cu["attn_prior"])
        nll, gl, _ = FlowtronLoss()(out, cu["gate_target"], cu["in_lens"], cu["out_lens"])
        (nll + gl).sum().backward()
        torch.cuda.synchronize()
        res.append((out, float(nll), {n: p.grad.clone() for n, p in model.named_parameters()}))
    (o1, n1, g1), (o2, n2, g2) = res
    assert (o1[0] - o2[0]).abs().max().item() <= 1e-5 * o1[0].abs().max().item()
    assert (o1[2] - o2[2]).abs().max().item() <= 1e-4
    for a, b in zip(o1[3], o2[3]):
        assert (a - b).abs().max().item() <= 1e-5
    assert abs(n1 - n2) <= 1e-5 * abs(n1)
    gmax = max(v.norm().item() for v in g1.values())
    for k in g1:
        d = (g1[k] - g2[k]).norm().item()
        assert d <= 2e-3 * (g1[k].norm().item() + 1e-4 * gmax), (k, d)   # wgrad sums are split differently (fp32 sums of fp16 products)


def test_batches_larger_than_a_launch_are_chunked():
    """B > max_kernel_batch runs as consecutive launches of at most max_kernel_batch utterances; rows must equal the
    unchunked result."""
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=2)
    model = build_model(cfg, 13)
    batch = synth.synth_batch(6, 24, 10, cfg, 3)
    cu = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in batch.items()}
    with torch.no_grad():
        a = model(cu["mel"], cu["speaker_ids"], cu["text"], cu["in_lens"], cu["out_lens"])
        model.max_kernel_batch = 4
        b = model(cu["mel"], cu["speaker_ids"], cu["text"], cu["in_lens"], cu["out_lens"])
    assert torch.equal(a[0], b[0]) and torch.equal(a[2], b[2])
    for x, y in zip(a[1] + a[3], b[1] + b[3]):
        assert torch.equal(x, y)


def test_encoder_streams_and_overlap_equal_serial():
    """Flowtron.overlap_encoder (the whole encoder on its own stream underneath the first flow's attention LSTM, joined
    inside ft_ar_step_fwd by the text-ready event) only changes scheduling: outputs are bit-identical and gradients equal
    up to the order of atomic accumulation.  Repeated a few times so a missing dependency would have a chance to show."""
    from flowtron_b200.flowtron import FlowtronLoss
    torch.backends.cudnn.allow_tf32 = False
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=2)
    batch = synth.synth_batch(6, 64, 20, cfg, 23, with_prior=True, in_lens=[20, 20, 17, 11, 9, 5])
    cu = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in batch.items()}

    def run(overlap):
        model = build_model(cfg, 37)
        model.train()
        model.encoder.p_dropout = 0.0
        model.overlap_encoder = overlap
        out = model(cu["mel"], cu["speaker_ids"], cu["text"], cu["in_lens"], cu["out_lens"], cu["attn_prior"])
        nll, gl, _ = FlowtronLoss()(out, cu["gate_target"], cu["in_lens"], cu["out_lens"])
        (nll + gl).sum().backward()
        torch.cuda.synchronize()
        return out, float(nll), {n: p.grad.clone() for n, p in model.named_parameters()}

    o1, n1, g1 = run(False)
    gmax = max(v.norm().item() for v in g1.values())
    for rep in range(4):
        o2, n2, g2 = run(True)
        assert torch.equal(o1[0], o2[0]) and torch.equal(o1[2], o2[2]), rep
        for a, b in zip(o1[1] + o1[3] + o1[4], o2[1] + o2[3] + o2[4]):
            assert torch.equal(a, b), rep
        assert abs(n1 - n2) <= 1e-6 * abs(n1)                  # the loss sums use float atomics
        for k in g1:
            d = (g1[k] - g2[k]).norm().item()
            # schedules differ only in the order of fp32 atomic accumulation (attention reductions, split-K weight
            # gradients); tensors that are small sums of large partials see a few 1e-4 of their own norm
            assert d <= 1e-3 * (g1[k].norm().item() + 1e-4 * gmax), (rep, k, d)


def test_batch_above_32_runs_as_32_plus_8_and_matches_split_runs():
    """A B = 40 batch runs as a 32-utterance and an 8-utterance flow launch (cfg 3 runs B = 64 per GPU as 32 + 32): rows
    must equal the same utterances run as two B = 20 batches, and the backward must produce the same gradients as the sum
    of the two halves."""
    from flowtron_b200 import _lib
    from flowtron_b200.flowtron import FlowtronLoss
    torch.backends.cudnn.allow_tf32 = False
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=2)
    batch = synth.synth_batch(40, 150, 16, cfg, 41, with_prior=True)
    cu = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in batch.items()}

    def run(sl):
        model = build_model(cfg, 43)
        model.train()
        model.encoder.p_dropout = 0.0
        Lp = int(cu["in_lens"][sl].max())
        out = model(cu["mel"][sl], cu["speaker_ids"][sl], cu["text"][sl][:, :Lp].contiguous(), cu["in_lens"][sl], cu["out_lens"][sl],
                    cu["attn_prior"][sl][:, :, :Lp].contiguous())
        nll, gl, _ = FlowtronLoss()(out, cu["gate_target"][sl], cu["in_lens"][sl], cu["out_lens"][sl])
        n = cu["out_lens"][sl].sum().float()
        ((nll + gl).sum() * n).backward()                       # un-normalised: the two halves' gradients add up to the whole
        torch.cuda.synchronize()
        return out, {k: p.grad.clone() for k, p in model.named_parameters()}

    full, gf = run(slice(0, 40))
    a, ga = run(slice(0, 20))
    b, gb = run(slice(20, 40))
    assert _lib.device_status() == 0
    T = 150
    vm = (torch.arange(T, device="cuda")[:, None] < cu["out_lens"][None, :])
    for part, sl in ((a, slice(0, 20)), (b, slice(20, 40))):
        ez = (full[0][:, sl] - part[0])[vm[:, sl]].abs().max().item() / full[0].abs().max().item()
        assert ez <= 1e-3, ez
    gmax = max(v.norm().item() for v in gf.values())
    for k in gf:
        d = (gf[k] - (ga[k] + gb[k])).norm().item()
        assert d <= 2e-2 * (gf[k].norm().item() + 1e-3 * gmax), (k, d, gf[k].norm().item())


def test_ar_step_rejects_more_than_32_utterances_per_call():
    """A flow step called directly takes at most 32 utterances (Flowtron.forward splits larger batches itself)."""
    from flowtron_b200 import _lib
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=2)
    step = build_model(cfg, 5).flows[0]
    T, B, L = 16, 33, 8
    E = cfg["n_text_dim"] + cfg["n_speaker_dim"]
    mel = torch.randn(T, B, cfg["n_mel_channels"], device="cuda")
    text = torch.randn(L, B, E, device="cuda")
    mask = torch.zeros(B, L, 1, dtype=torch.bool, device="cuda")
    out_lens = torch.full((B,), T, dtype=torch.long, device="cuda")
    with torch.no_grad(), pytest.raises(_lib.FlowtronB200Error, match="batch > 32"):
        step(mel, text, mask, out_lens)
    torch.cuda.synchronize()
    assert _lib.device_status() == 0
