"""GPU, BASELINE.json full sizes (configs[1]: B=32, T=1000, L<=160; configs[3]: T=1000 inference): size-independent
properties (SURVEY.md §4 invariants) of the forward pass and the inverse.  The training step at these sizes (forward
outputs, losses and every parameter gradient, eager and replayed from one CUDA graph) is compared with the fp64 oracle,
one utterance at a time, in tests/test_gpu_train_step_oracle.py."""
import pytest
import torch

from conftest import record_parity
from flowtron_b200 import synth

pytestmark = pytest.mark.gpu

B, T = 32, 1000


def _batch(seed=1234, with_prior=True):
    cfg = dict(synth.DEFAULT_MODEL_CONFIG)
    out_lens, in_lens = synth.ljs_like_lengths(B, T, seed)
    L = int(in_lens.max())
    b = synth.synth_batch(B, T, L, cfg, seed, out_lens=out_lens.tolist(), in_lens=in_lens.tolist(), with_prior=with_prior,
                          logmel_stats=True)
    return cfg, {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in b.items()}


def _model(cfg, seed=None):
    from flowtron_b200.flowtron import Flowtron
    m = Flowtron(**cfg)
    if seed is not None:
        m.load_state_dict(synth.synth_params(cfg, seed), strict=True)
    return m.cuda().eval()


def test_fullsize_zero_init_identity():
    """Reference init (flowtron.py:652-653): conv = 0 => z == mel bit-exactly and log_s == 0, at B=32, T=1000."""
    cfg, cu = _batch(with_prior=True)
    torch.manual_seed(0)
    m = _model(cfg)
    with torch.no_grad():
        out = m(cu["mel"], cu["speaker_ids"], cu["text"], cu["in_lens"], cu["out_lens"], cu["attn_prior"])
    assert torch.equal(out[0].permute(1, 2, 0), cu["mel"])
    assert all(float(ls.abs().max()) == 0.0 for ls in out[1])
    for a in out[3]:                                    # attention rows of valid frames sum to 1, mass only on valid keys
        vm = (torch.arange(T, device="cuda")[None, :] < cu["out_lens"][:, None])
        s = a.sum(-1)[vm]
        assert (s - 1).abs().max().item() < 1e-4
        km = (torch.arange(a.shape[-1], device="cuda")[None, :] >= cu["in_lens"][:, None])
        assert float(a.masked_select(km[:, None, :].expand_as(a)).abs().max()) == 0.0


def test_fullsize_batch_split_consistency_and_loss():
    """Utterances are independent: rows of the B=32 run equal the same rows run as two B=16 batches (exercises the
    recurrence kernels at two batch sizes at T=1000); the fused loss reductions equal the torch formula."""
    from flowtron_b200.flowtron import FlowtronLoss
    cfg, cu = _batch(with_prior=False)
    m = _model(cfg, seed=5)
    with torch.no_grad():
        enc_in = (cu["mel"], cu["speaker_ids"], cu["text"], cu["in_lens"], cu["out_lens"])
        full = m(*enc_in)
        vm = (torch.arange(T, device="cuda")[:, None] < cu["out_lens"][None, :])
        for b0, b1 in ((0, 16), (16, 32)):
            sl = slice(b0, b1)
            Lp = int(cu["in_lens"][sl].max())           # the collate pads text to the sub-batch's own max length
            part = m(cu["mel"][sl], cu["speaker_ids"][sl], cu["text"][sl][:, :Lp].contiguous(), cu["in_lens"][sl], cu["out_lens"][sl])
            z_f, z_p = full[0][:, sl], part[0]
            ez = (z_f - z_p)[vm[:, sl]].abs().max().item() / z_f.abs().max().item()
            els = max((full[1][i][:, sl] - part[1][i])[vm[:, sl]].abs().max().item() / full[1][i].abs().max().item() for i in range(2))
            record_parity(f"fullsize_split_{b0}", {"z": ez, "log_s": els})
            assert ez <= 1e-3 and els <= 1e-3, (ez, els)      # same rows, two batch sizes: within the forward parity bar
        nll, gl, _ = FlowtronLoss(sigma=1.0)(full, cu["gate_target"], cu["in_lens"], cu["out_lens"])
        mask = vm.float()[..., None]
        n = mask.sum()
        ref = ((full[0] * mask) ** 2).sum() / 2 - sum((ls * mask).sum() for ls in full[1])
        ref = ref / (n * 80)
        assert abs(float(nll) - float(ref)) <= 1e-4 * abs(float(ref))
        gp = (full[2] * mask)[..., 0].permute(1, 0)
        gref = (torch.nn.functional.binary_cross_entropy_with_logits(gp, cu["gate_target"], reduction="none").permute(1, 0)
                * mask[:, :, 0]).sum() / n
        assert abs(float(gl) - float(gref)) <= 1e-4 * abs(float(gref))


def test_fullsize_invertibility_T1000():
    """forward(infer(z)) == z at T = 1000 (BASELINE configs[3] length), B = 1."""
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, use_gate_layer=False)
    m = _model(cfg, seed=3)
    g = torch.Generator().manual_seed(1)
    L = 100
    zin = (torch.randn(1, 80, T, generator=g) * 0.5).cuda()
    text = torch.randint(0, 185, (1, L), generator=g).cuda()
    spk = torch.zeros(1, dtype=torch.long, device="cuda")
    with torch.no_grad():
        mel, _ = m.infer(zin, spk, text)
        out = m(mel, spk, text, torch.tensor([L], device="cuda"), torch.tensor([T], device="cuda"))
    z = out[0].permute(1, 2, 0)
    err = (z - zin).abs().max().item() / zin.abs().max().item()
    print("T=1000 round trip rel err", err)
    record_parity("fullsize_invertibility_T1000", {"z_roundtrip": err})
    assert torch.isfinite(mel).all()
    assert err <= 2e-3, err       # both directions within 1e-3 of the fp32 reference (test_gpu_baseline_shapes) => 2e-3
