"""CPU: the flow-step oracle (oracle/flowtron_oracle.py ar_step_forward / ar_back_step_forward) as an fp64 gradient oracle.

tests/test_gpu_ar_step_backward.py compares the CUDA flow step's backward with torch.autograd of these functions in fp64.
Here the oracle's own gradient is pinned by finite differences at a toy size (ragged frame and text lengths down to 1,
with and without a prior, temperature 1 and 0.5), and the fp64 oracle is checked to compute the same function as the fp32
one that tests/test_oracle_golden.py pins against the reference.  A silent cast to fp32 anywhere on the way would fail
the gradient check (fp32 rounding is far above its tolerance at eps = 1e-6) or the dtype checks below."""
import pytest
import torch

from flowtron_b200 import synth
from oracle import flowtron_oracle as O

TOY = dict(synth.DEFAULT_MODEL_CONFIG, n_hidden=4, n_attn_channels=4, n_mel_channels=2, n_text_dim=2, n_speaker_dim=2)


def _prior(out_lens, in_lens, T, L, dtype):
    prior = torch.zeros(len(out_lens), T, L, dtype=dtype)
    for b, (t, l) in enumerate(zip(out_lens.tolist(), in_lens.tolist())):
        prior[b, :t, :l] = torch.from_numpy(synth.beta_binomial_prior(l, t)).to(dtype)
    return prior


def _case(cfg, n_flows, B, T, L, out_lens, in_lens, dtype, seed=3):
    """Weights of flow n_flows - 1 (gated: the last flow), inputs and masks."""
    cfg = dict(cfg, n_flows=n_flows)
    i = n_flows - 1
    pre = f"flows.{i}"
    p = {k: v for k, v in synth.synth_params(cfg, seed, dtype=dtype).items() if k.startswith(pre + ".")}
    g = torch.Generator().manual_seed(seed)
    out_lens, in_lens = torch.tensor(out_lens), torch.tensor(in_lens)
    M, E = cfg["n_mel_channels"], cfg["n_text_dim"] + cfg["n_speaker_dim"]
    mel = torch.randn(T, B, M, generator=g).to(dtype)
    text = (0.5 * torch.randn(L, B, E, generator=g)).to(dtype)
    mask = ~(torch.arange(L)[None, :] < in_lens[:, None])[..., None]
    return pre, p, mel, text, mask, out_lens, in_lens


@pytest.mark.parametrize("temperature", [1.0, 0.5])
@pytest.mark.parametrize("with_prior", [True, False])
@pytest.mark.parametrize("back", [False, True], ids=["ar_step", "ar_back_step"])
def test_oracle_flow_step_gradcheck(back, with_prior, temperature):
    """d(weighted sum of z, log_s, gate, attn, attn_logprob on valid positions) / d(mel, text, every weight) of one flow step
    agrees with central differences over the full Jacobian (torch.autograd.gradcheck, fp64)."""
    B, T, L = 3, 5, 4
    pre, p, mel, text, mask, out_lens, in_lens = _case(TOY, 2 if back else 1, B, T, L, [5, 1, 3], [4, 2, 1], torch.float64)
    assert f"{pre}{'.ar_step' if back else ''}.gate_layer.linear_layer.weight" in p
    prior = _prior(out_lens, in_lens, T, L, torch.float64) if with_prior else None
    names = list(p)
    vt = (torch.arange(T)[:, None] < out_lens[None, :]).to(torch.float64)            # [T,B] valid frames
    vk = (torch.arange(L)[None, :] < in_lens[:, None]).to(torch.float64)             # [B,L] valid keys
    vtl = vt.t()[:, :, None] * vk[:, None, :]                                         # [B,T,L]
    g = torch.Generator().manual_seed(7)
    w = [torch.randn(T, B, TOY["n_mel_channels"], generator=g, dtype=torch.float64) * vt[..., None],
         torch.randn(T, B, TOY["n_mel_channels"], generator=g, dtype=torch.float64) * vt[..., None],
         torch.randn(T, B, 1, generator=g, dtype=torch.float64) * vt[..., None],
         torch.randn(B, T, L, generator=g, dtype=torch.float64) * vtl,
         torch.randn(B, T, L, generator=g, dtype=torch.float64) * vtl]
    fn = O.ar_back_step_forward if back else O.ar_step_forward

    def f(mel, text, *weights):
        outs = fn(dict(zip(names, weights)), pre, mel, text, mask, out_lens, prior, temperature)
        return sum((o * wi).sum() for o, wi in zip(outs, w))

    inputs = [t.clone().requires_grad_(True) for t in [mel, text, *p.values()]]
    assert torch.autograd.gradcheck(f, inputs, eps=1e-6, atol=1e-7, rtol=1e-5)


@pytest.mark.parametrize("back", [False, True], ids=["ar_step", "ar_back_step"])
def test_fp64_oracle_matches_fp32_oracle_at_full_size(back):
    """At the real widths (H = 1024, A = 640), the fp64 oracle on fp32-valued inputs keeps fp64 end to end (outputs and
    gradients) and, rounded to fp32, is the fp32 oracle's function: every output within 2e-6 of its max |value|."""
    B, T, L = 2, 6, 5
    res = {}
    for dtype in (torch.float32, torch.float64):
        pre, p, mel, text, mask, out_lens, in_lens = _case(synth.DEFAULT_MODEL_CONFIG, 2 if back else 1, B, T, L, [6, 3], [5, 2],
                                                           dtype, seed=11)
        prior = _prior(out_lens, in_lens, T, L, dtype)
        mel.requires_grad_(True)
        fn = O.ar_back_step_forward if back else O.ar_step_forward
        outs = fn(p, pre, mel, text, mask, out_lens, prior, 0.5)
        vt = (torch.arange(T)[:, None] < out_lens[None, :])
        vk = (torch.arange(L)[None, :] < in_lens[:, None])
        (d_mel,) = torch.autograd.grad(outs[0][vt].sum() + outs[4].masked_fill(~vk[:, None, :], 0).sum(), [mel])
        for o in (*outs, d_mel):
            assert o.dtype == dtype
        vtl = vt.t()[:, :, None] & vk[:, None, :]
        res[dtype] = [outs[0][vt], outs[1][vt], outs[2][vt], outs[3][vtl], outs[4][vtl], d_mel]
    for i, (a, b) in enumerate(zip(res[torch.float32], res[torch.float64])):
        err = (a.double() - b).abs().max().item() / b.abs().max().item()
        assert err <= 2e-6, (i, err)
