"""GPU parity of the Encoder kernels (ft_encoder_fwd / ft_encoder_bwd, csrc/encoder.cu) against the CPU oracle's restatement of
flowtron.py:467-525 (forward) and against fp32 autograd through that restatement (backward).  Forward bar: 1e-3 of the tensor's
max |value| (north star); gradients: SURVEY 8d (norm 1e-2 relative, cosine 0.9999)."""
import pytest
import torch

from conftest import record_parity
from oracle import flowtron_oracle as O
from flowtron_b200 import synth

pytestmark = pytest.mark.gpu


def _model(seed):
    from flowtron_b200.flowtron import Flowtron
    cfg = dict(synth.DEFAULT_MODEL_CONFIG)
    m = Flowtron(**cfg)
    params = synth.synth_params(cfg, seed)
    m.load_state_dict(params, strict=True)
    return m.cuda(), params


def _x(B, L, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, 512, L, generator=g) * 0.7


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-12)


@pytest.mark.parametrize("B,L,lens", [(5, 37, [37, 30, 22, 9, 1]), (32, 150, None), (1, 50, [50]), (48, 64, None), (72, 40, None)])
def test_encoder_forward_matches_oracle(B, L, lens):
    m, p = _model(3)
    m.eval()
    x = _x(B, L, 11)
    if lens is None:
        g = torch.Generator().manual_seed(5)
        lens = sorted(torch.randint(max(1, L // 3), L + 1, (B,), generator=g).tolist(), reverse=True)
        lens[0] = L
    in_lens = torch.tensor(lens)
    with torch.no_grad():
        ours = m.encoder(x.cuda(), in_lens.cuda())
        ref = O.encoder_forward(p, x, in_lens)
    assert ours.shape == ref.shape
    err = rel(ours, ref)
    record_parity(f"encoder_fwd_B{B}_L{L}", {"out": err})
    assert err < 1e-3, err
    # padded positions are exactly zero (pad_packed_sequence)
    for b, n in enumerate(lens):
        assert float(ours[b, n:].abs().max()) == 0.0 if n < L else True


def test_encoder_infer_matches_oracle():
    m, p = _model(4)
    m.eval()
    x = _x(4, 41, 12)
    with torch.no_grad():
        ours = m.encoder.infer(x.cuda())
        ref = O.encoder_forward(p, x, None, infer=True)
    err = rel(ours, ref)
    record_parity("encoder_infer_B4", {"out": err})
    assert err < 1e-3, err


@pytest.mark.parametrize("B,L,lens", [(4, 29, [29, 20, 11, 3]), (1, 33, [33]), (32, 120, None), (72, 40, None)])
def test_encoder_backward_matches_fp32_autograd(B, L, lens):
    m, p = _model(6)
    m.train()
    m.encoder.p_dropout = 0.0
    x = _x(B, L, 13)
    if lens is None:
        g = torch.Generator().manual_seed(7)
        lens = sorted(torch.randint(L // 3, L + 1, (B,), generator=g).tolist(), reverse=True)
        lens[0] = L
    in_lens = torch.tensor(lens)
    g = torch.Generator().manual_seed(99)
    w_out = torch.randn(B, L, 512, generator=g) * 0.05
    # ours
    xc = x.cuda().requires_grad_(True)
    for q in m.encoder.parameters():
        q.grad = None
    out = m.encoder(xc, in_lens.cuda())
    (out * w_out.cuda()).sum().backward()
    ours = {"x": xc.grad.cpu()}
    for n, q in m.encoder.named_parameters():
        ours["encoder." + n] = q.grad.cpu()
    # fp32 autograd through the oracle restatement
    pr = {k: v.clone().requires_grad_(k.startswith("encoder.")) for k, v in p.items()}
    xr = x.clone().requires_grad_(True)
    ref_out = O.encoder_forward(pr, xr, in_lens)
    (ref_out * w_out[:, :ref_out.shape[1]]).sum().backward()
    ref = {"x": xr.grad}
    for k, v in pr.items():
        if k.startswith("encoder."):
            ref[k] = v.grad
    worst_norm, worst_cos, worst = 0.0, 1.0, ""
    wscale = ref["encoder.convolutions.0.0.conv.weight"].double().norm().item()
    for k, r in ref.items():
        o = ours[k].double()
        r = r.double()
        if k.endswith("conv.bias"):
            # a bias in front of an instance norm has an identically zero gradient (the norm removes the mean): both sides
            # are rounding noise; ours must be negligible next to the same layer's weight gradient
            assert o.norm().item() < 1e-3 * wscale, (k, o.norm().item(), wscale)
            continue
        ne = (o - r).norm().item() / max(r.norm().item(), 1e-30)
        cos = (o * r).sum().item() / max(o.norm().item() * r.norm().item(), 1e-30)
        if ne > worst_norm:
            worst_norm, worst = ne, k
        worst_cos = min(worst_cos, cos)
    record_parity(f"encoder_bwd_B{B}_L{L}", {"rel_l2_worst": worst_norm, "cos_worst": worst_cos, "worst_tensor": worst})
    assert worst_norm < 1e-2 and worst_cos > 0.9999, (worst, worst_norm, worst_cos)


def test_encoder_dropout_is_random_scaled_and_consistent_in_backward():
    """Training-mode dropout (flowtron.py:502, p = 0.5): about half the activations of a block survive, scaled by 2; a second
    forward draws different masks; backward uses the mask of its own forward (gradient is zero where the output is zero)."""
    m, _ = _model(8)
    m.train()
    B, L = 6, 40
    x = _x(B, L, 14).cuda().requires_grad_(True)
    in_lens = torch.tensor([40, 33, 30, 21, 12, 5]).cuda()
    o1 = m.encoder(x, in_lens)
    o2 = m.encoder(x, in_lens)
    assert (o1 - o2).abs().max() > 1e-3
    o1.sum().backward()
    assert torch.isfinite(x.grad).all() and x.grad.abs().max() > 0
    # gradient w.r.t. masked-out input positions is exactly zero (masked_fill before the first convolution)
    for b, n in enumerate(in_lens.tolist()):
        if n < L:
            assert float(x.grad[b, :, n:].abs().max()) == 0.0


def test_encoder_token_path_equals_embedding_then_encoder():
    """ft_encoder_fwd_tokens / ft_encoder_bwd_tokens (embedding gather / scatter fused into the encoder kernels) against the
    two-step path nn.Embedding -> Encoder kernels: identical forward, embedding gradient equal up to atomic-add order."""
    m, _ = _model(9)
    m.train()
    m.encoder.p_dropout = 0.0
    g = torch.Generator().manual_seed(21)
    B, L = 7, 33
    tokens = torch.randint(0, m.embedding.num_embeddings, (B, L), generator=g).cuda()
    in_lens = torch.tensor([33, 30, 30, 21, 12, 5, 2]).cuda()
    w_out = (torch.randn(B, L, 512, generator=g) * 0.05).cuda()

    def run(fused):
        for q in m.parameters():
            q.grad = None
        out = m.encoder.forward_tokens(tokens, m.embedding, in_lens) if fused else m.encoder(m.embedding(tokens).transpose(1, 2), in_lens)
        (out * w_out).sum().backward()
        return out.detach(), m.embedding.weight.grad.clone(), m.encoder.lstm.weight_ih_l0.grad.clone()
    o1, e1, w1 = run(True)
    o2, e2, w2 = run(False)
    assert torch.equal(o1, o2)
    assert (e1 - e2).norm().item() <= 1e-5 * e2.norm().item() and e2.norm().item() > 0
    assert (w1 - w2).norm().item() <= 1e-5 * w2.norm().item()
    # rows of tokens that only occur at masked positions get no gradient
    used = set(tokens[torch.arange(L, device="cuda")[None, :] < in_lens[:, None]].tolist())
    unused = [t for t in range(m.embedding.num_embeddings) if t not in used]
    assert float(e1[unused].abs().max()) == 0.0


def test_encoder_batch_above_64_equals_calls_of_at_most_64():
    """The kernels take at most 64 utterances per call: B = 72 runs as 64 + 8 rows, and in eval mode every row equals, bit for
    bit, the same rows run as batches of 64 and 8 (embedded-input and token forms)."""
    m, _ = _model(10)
    m.eval()
    B, L = 72, 40
    g = torch.Generator().manual_seed(15)
    x = _x(B, L, 16).cuda()
    tokens = torch.randint(0, m.embedding.num_embeddings, (B, L), generator=g).cuda()
    in_lens = torch.randint(1, L + 1, (B,), generator=g)
    in_lens[0] = L
    in_lens = in_lens.cuda()
    with torch.no_grad():
        full = m.encoder(x, in_lens)
        parts = torch.cat([m.encoder(x[:64], in_lens[:64]), m.encoder(x[64:], in_lens[64:])])
        full_t = m.encoder.infer_ragged_tokens(tokens, m.embedding, in_lens)
        parts_t = torch.cat([m.encoder.infer_ragged_tokens(tokens[:64], m.embedding, in_lens[:64]),
                             m.encoder.infer_ragged_tokens(tokens[64:], m.embedding, in_lens[64:])])
    assert full.shape == (B, L, 512) and torch.equal(full, parts)
    assert torch.equal(full_t, parts_t)


def test_flowtron_train_step_above_64_utterances():
    """Flowtron.forward + backward at B = 72: the encoder (token form) runs as 64 + 8 rows, the flows as 32-row launches."""
    from flowtron_b200 import _lib
    from flowtron_b200.flowtron import FlowtronLoss
    m, _ = _model(11)
    m.train()
    m.encoder.p_dropout = 0.0
    batch = synth.synth_batch(72, 16, 10, synth.DEFAULT_MODEL_CONFIG, 17)
    cu = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in batch.items()}
    out = m(cu["mel"], cu["speaker_ids"], cu["text"], cu["in_lens"], cu["out_lens"])
    nll, gl, _ = FlowtronLoss()(out, cu["gate_target"], cu["in_lens"], cu["out_lens"])
    (nll + gl).sum().backward()
    torch.cuda.synchronize()
    assert _lib.device_status() == 0
    assert out[0].shape[1] == 72 and torch.isfinite(out[0]).all()
    for p in (m.embedding.weight, m.encoder.lstm.weight_ih_l0, m.encoder.convolutions[0][0].conv.weight):
        assert torch.isfinite(p.grad).all() and p.grad.abs().max() > 0
