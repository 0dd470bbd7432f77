"""GPU: style transfer by posterior sampling -- Flowtron.encode and style.posterior_mean (ft_posterior_mean) against the
reference-generated fixtures (tests/make_golden_style_transfer.py), float64 restatements, CUDA-graph replay, and the
chain into Flowtron.infer, WaveGlow.infer and the Denoiser."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, record_parity
from flowtron_b200 import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def enc():
    return dict(np.load(os.path.join(GOLDEN, "style_encode.npz")))


@pytest.fixture(scope="module")
def post():
    return dict(np.load(os.path.join(GOLDEN, "style_posterior.npz")))


@pytest.fixture(scope="module")
def model(enc):
    from flowtron_b200.flowtron import Flowtron
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=2)
    p = synth.synth_params(cfg, int(enc["seed"]))
    key = [k for k in p if k.endswith("gate_layer.linear_layer.bias")][0]
    p[key] = torch.full_like(p[key], float(enc["gate_bias"]))
    m = Flowtron(**cfg)
    m.load_state_dict(p, strict=True)
    return m.cuda().eval()


def _inputs(enc):
    return (torch.from_numpy(enc["mel"]).cuda(), torch.from_numpy(enc["speaker_ids"]).cuda(),
            torch.from_numpy(enc["text"]).cuda(), enc["in_lens"].tolist(), enc["out_lens"].tolist())


def test_encode_padded_batch_matches_reference(model, enc):
    from flowtron_b200 import _lib
    mel, spk, text, in_lens, out_lens = _inputs(enc)
    model.train()                                   # encode runs without dropout and without autograd state in any mode
    try:
        z = model.encode(mel, spk, text, in_lens, out_lens)
    finally:
        model.eval()
    torch.cuda.synchronize()
    assert _lib.device_status() == 0
    assert tuple(z.shape) == tuple(enc["z"].shape) and not z.requires_grad
    ref = torch.from_numpy(enc["z"])
    zmax = ref.abs().max().item()
    errs = {}
    for b, n in enumerate(out_lens):
        errs[f"row{b}"] = (z[b, :, :n].cpu() - ref[b, :, :n]).abs().max().item() / zmax
        assert (z[b, :, n:] == 0).all(), b
    record_parity("style_encode_batch", errs)
    assert max(errs.values()) <= 1e-3, errs


def test_encode_rows_equal_single_runs(model, enc):
    """Each row of the padded batch against encode on its own unpadded inputs (the reference notebook's B = 1 loop)."""
    mel, spk, text, in_lens, out_lens = _inputs(enc)
    with torch.no_grad():
        zb = model.encode(mel, spk, text, torch.tensor(in_lens, device="cuda"), torch.tensor(out_lens, device="cuda"))
        singles = [model.encode(mel[b:b + 1, :, :n].contiguous(), spk[b:b + 1], text[b:b + 1, :nl].contiguous(), [nl], [n])
                   for b, (nl, n) in enumerate(zip(in_lens, out_lens))]
    zmax = max(s.abs().max().item() for s in singles)
    diff = max((zb[b, :, :n] - s[0]).abs().max().item() for b, (n, s) in enumerate(zip(out_lens, singles)))
    identical = all(torch.equal(zb[b, :, :n], s[0]) for b, (n, s) in enumerate(zip(out_lens, singles)))
    record_parity("style_encode_rows_vs_b1", {"max_abs_diff": diff, "rel_diff": diff / zmax, "bit_identical": int(identical)})
    print(f"batched vs B = 1 encode: max |diff| {diff:.3e} ({diff / zmax:.3e} of max |z|), bit-identical {identical}")
    assert diff <= 1e-5 * zmax, (diff, zmax)


def test_encode_rows_on_both_sides_of_the_attention_overlap_threshold(model):
    """A batch padded to >= 320 frames runs the attention LSTM's input projection as a separate GEMM, a shorter one folds it
    into the recurrence.  With host lengths, encode runs the rows under 320 frames as their own launch, so every row equals
    its B = 1 run; with CUDA lengths the batch runs as one launch and those rows differ by rounding only."""
    from flowtron_b200.flowtron import _ATTN_OVERLAP_MIN_T
    assert _ATTN_OVERLAP_MIN_T == 320
    g = torch.Generator().manual_seed(31)
    out_lens, in_lens = [400, 150, 330, 90, 319, 320], [40, 20, 35, 12, 30, 33]
    B, T, L = len(out_lens), max(out_lens), max(in_lens)
    mel = (torch.randn(B, 80, T, generator=g) * 2.0 - 5.5).clamp_(-11.5, 2.0).cuda()
    text = torch.randint(0, 185, (B, L), generator=g).cuda()
    spk = torch.zeros(B, dtype=torch.long, device="cuda")
    z_host = model.encode(mel, spk, text, in_lens, out_lens)
    z_dev = model.encode(mel, spk, text, torch.tensor(in_lens, device="cuda"), torch.tensor(out_lens, device="cuda"))
    singles = [model.encode(mel[b:b + 1, :, :n], spk[b:b + 1], text[b:b + 1, :nl], [nl], [n])
               for b, (nl, n) in enumerate(zip(in_lens, out_lens))]
    zmax = max(s.abs().max().item() for s in singles)
    host = {b: (z_host[b, :, :n] - s[0]).abs().max().item() / zmax for b, (n, s) in enumerate(zip(out_lens, singles))}
    dev = {b: (z_dev[b, :, :n] - s[0]).abs().max().item() / zmax for b, (n, s) in enumerate(zip(out_lens, singles))}
    record_parity("style_encode_overlap_threshold", {"host_lens_max": max(host.values()), "cuda_lens_max": max(dev.values()),
                                                     **{f"cuda_lens_row{b}_len{out_lens[b]}": v for b, v in dev.items()}})
    for b, n in enumerate(out_lens):
        assert torch.equal(z_host[b, :, :n], singles[b][0]), (b, n, host[b])
        assert (z_host[b, :, n:] == 0).all() and (z_dev[b, :, n:] == 0).all(), b
        if n >= _ATTN_OVERLAP_MIN_T:                     # same path as the B = 1 run either way
            assert torch.equal(z_dev[b, :, :n], singles[b][0]), (b, n, dev[b])
    assert max(dev.values()) <= 1e-3, dev


@pytest.mark.parametrize("aggregation", ["batch", "time_and_batch"])
def test_posterior_mean_matches_fixtures(enc, post, aggregation):
    from flowtron_b200.style import posterior_mean
    z = torch.from_numpy(enc["z"]).cuda()
    lens_host = enc["out_lens"].tolist()
    lens_dev = torch.tensor(lens_host, device="cuda")
    errs = {}
    for li, lambd in enumerate(post["lambds"].tolist()):
        for n in post["n_frames"].tolist():
            ref = torch.from_numpy(post[f"mu_{aggregation}_n{n}_l{li}"])
            for tag, lens in (("host", lens_host), ("dev", lens_dev)):
                mu = posterior_mean(z, lens, n, lambd=lambd, aggregation=aggregation)
                assert tuple(mu.shape) == (1, 80, n if aggregation == "batch" else 1)
                errs[f"n{n}_l{li}_{tag}"] = (mu[0].double().cpu() - ref).abs().max().item() / ref.abs().max().item()
    record_parity(f"style_posterior_{aggregation}", errs)
    assert max(errs.values()) <= 1e-6, errs


def _posterior_f64(z, lens, n_frames, lambd, aggregation):
    K = z.shape[0]
    zd = z.double()
    if aggregation == "batch":
        mean = torch.stack([zd[k][:, torch.arange(n_frames, device=z.device) % int(t)] for k, t in enumerate(lens)]).mean(0)
    else:
        mean = torch.stack([zd[k, :, :int(t)].mean(1) for k, t in enumerate(lens)]).mean(0)[:, None]
    ratio = K / lambd
    return (ratio * mean / (ratio + 1.0))[None]


@pytest.mark.parametrize("K", [1, 7, 40])
def test_posterior_mean_random_against_float64(K):
    from flowtron_b200.style import posterior_mean
    g = torch.Generator().manual_seed(100 + K)
    T = 150
    lens = torch.randint(1, T + 1, (K,), generator=g)
    lens[0] = 1                                         # a one-frame utterance
    if K > 1:
        lens[1] = T
    zt = (torch.randn(T, K, 80, generator=g) * 1.5 + 0.3).cuda()      # encode's storage order
    z = zt.permute(1, 2, 0)                             # [K, 80, T] view, read without a copy
    zc = z.contiguous()                                 # and a contiguous [K, 80, T] tensor
    errs = {}
    for n in sorted({1, 29, int(lens[-1]), T, 401}):    # n == a row's length (and == T)
        for agg in ("batch", "time_and_batch"):
            for lambd in (1e-4, 0.5):
                ref = _posterior_f64(z, lens.tolist(), n, lambd, agg)
                for tag, zz in (("view", z), ("contig", zc)):
                    mu = posterior_mean(zz, lens.cuda(), n, lambd=lambd, aggregation=agg)
                    errs[f"{agg}_n{n}_l{lambd}_{tag}"] = (mu.double() - ref).abs().max().item() / ref.abs().max().item()
    record_parity(f"style_posterior_random_K{K}", {"max": max(errs.values())})
    assert max(errs.values()) <= 1e-6, {k: v for k, v in errs.items() if v > 1e-6}


def test_cuda_graph_replay_equals_eager(model, enc):
    """encode + posterior_mean (both aggregations) captured in one CUDA graph with CUDA length tensors."""
    from flowtron_b200.style import posterior_mean
    mel, spk, text, in_lens, out_lens = _inputs(enc)
    in_d, out_d = torch.tensor(in_lens, device="cuda"), torch.tensor(out_lens, device="cuda")
    new_mel = (torch.randn(mel.shape, generator=torch.Generator().manual_seed(5)) * 2.0 - 5.5).clamp_(-11.5, 2.0).cuda()

    def chain():
        z = model.encode(mel, spk, text, in_d, out_d)
        return z, posterior_mean(z, out_d, 150), posterior_mean(z, out_d, 150, aggregation="time_and_batch")

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        chain()                                         # warm-up: scratch buffers exist before capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        zg, mbg, mtg = chain()
    mel.copy_(new_mel)
    graph.replay()
    torch.cuda.synchronize()
    ze, mbe, mte = chain()
    torch.cuda.synchronize()
    assert torch.equal(zg, ze) and torch.equal(mbg, mbe) and torch.equal(mtg, mte)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(zg, ze) and torch.equal(mbg, mbe) and torch.equal(mtg, mte)


def test_infer_from_fixture_residual_matches_reference(model, post):
    from flowtron_b200 import _lib
    res = torch.from_numpy(post["infer_residual"]).cuda()
    text = torch.from_numpy(post["infer_text"]).cuda()
    with torch.no_grad():
        mel, _ = model.infer(res, torch.zeros(1, dtype=torch.long, device="cuda"), text)
    torch.cuda.synchronize()
    assert _lib.device_status() == 0
    ref = torch.from_numpy(post["infer_mel"])
    assert tuple(mel.shape) == tuple(ref.shape), (mel.shape, ref.shape)
    err = (mel.cpu() - ref).abs().max().item() / ref.abs().max().item()
    record_parity("style_infer", {"mel": err})
    assert err <= 1e-3, err


def test_style_transfer_chain_to_audio(model, enc):
    """encode -> posterior_mean -> infer and infer_batch (the mean broadcast over the rows) -> WaveGlow.infer -> Denoiser."""
    from flowtron_b200 import _lib
    from flowtron_b200.denoiser import Denoiser
    from flowtron_b200.style import posterior_mean
    from flowtron_b200.waveglow import WaveGlow
    wcfg = synth.DEFAULT_WAVEGLOW_CONFIG
    wg = WaveGlow(**wcfg)
    wg.load_state_dict(synth.synth_waveglow_params(wcfg, 14), strict=True)
    wg = wg.cuda().eval()
    den = Denoiser(wg)
    mel, spk, text, in_lens, out_lens = _inputs(enc)
    g = torch.Generator().manual_seed(8)
    n_frames, sigma = 48, 0.5
    new_text = torch.randint(0, 185, (2, 14), generator=g).cuda()
    with torch.no_grad():
        z = model.encode(mel, spk, text, in_lens, out_lens)
        for agg in ("batch", "time_and_batch"):
            mu = posterior_mean(z, out_lens, n_frames, aggregation=agg)
            res = mu + sigma * torch.randn(2, 80, n_frames, generator=g).cuda()
            m1, _ = model.infer(res[:1], spk[:1], new_text[:1])
            mb, lens, _ = model.infer_batch(res, spk[:2], new_text, [14, 9])
            assert m1.shape[-1] == n_frames and lens.tolist() == [n_frames, n_frames]
            assert (mb[0] - m1[0]).abs().max().item() <= 2e-3 * m1.abs().max().item()
            audio = wg.infer(mb.contiguous(), sigma=0.6, noise=synth.synth_waveglow_noise(2, n_frames, 15).cuda())
            clean = den(audio, 0.01)
            assert audio.shape[-1] == 256 * n_frames and torch.isfinite(clean).all()
    torch.cuda.synchronize()
    assert _lib.device_status() == 0
