"""H100: synthesis from the Gaussian-mixture prior.  Flowtron.mixture against the reference one utterance at a time
(tests/make_golden_gmm_sample.py) and against its own B = 1 calls; the sampler against the numpy restatement of its
counter hash, its independence of B and of the padded T, forced components, its statistics over 2.5 M elements and its
CUDA-graph replays; the responsibilities against fp64 and their B = 1 calls; and mixture -> sample_mixture -> infer_batch
-> WaveGlow.infer -> Denoiser captured as one CUDA graph."""
import os

import numpy as np
import pytest
import torch

import gmm_sample_oracle as O
from conftest import GOLDEN, record_parity
from flowtron_b200 import synth

pytestmark = pytest.mark.gpu

CASES = ["gmm_sample_learned", "gmm_sample_fixed"]
HOP = 256


def _case(name):
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=2, n_components=int(g["K"]), fixed_gaussian=bool(g["fixed_gaussian"]),
               mean_scale=float(g["mean_scale"]))
    return g, cfg, synth.synth_gmm_params(cfg, int(g["seed"]))


def _model(cfg, params):
    from flowtron_b200.flowtron import Flowtron
    m = Flowtron(**cfg)
    m.load_state_dict(params, strict=True)
    return m.cuda()


def _rel(a, b):
    a, b = a.detach().double().cpu(), torch.as_tensor(b).double()
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-30)


def _ulps(a, b):
    """Largest distance between two fp32 tensors of one sign pattern in units in the last place."""
    ia, ib = a.float().contiguous().view(torch.int32).long(), b.float().contiguous().view(torch.int32).long()
    return int((ia - ib).abs().max().item())


@pytest.mark.parametrize("name", CASES)
def test_mixture_matches_the_reference_per_utterance(name):
    g, cfg, params = _case(name)
    model = _model(cfg, params).train()                         # eval semantics whatever the mode
    mel = torch.from_numpy(g["mel"]).cuda()
    lens = g["out_lens"].tolist()
    outs = {"host": model.mixture(mel, lens), "cuda": model.mixture(mel, torch.tensor(lens).cuda())}
    emb = {}
    h = model.mel_encoder.register_forward_hook(lambda m, i, o: emb.__setitem__("x", o.detach().clone()))
    errs = {}
    for kind, (mean, log_var, prob) in outs.items():
        for key, t in (("mean", mean), ("log_var", log_var), ("prob", prob)):
            ref = torch.from_numpy(g[key])
            assert t.shape == ref.shape, (kind, key)
            if ref.abs().max() > 0:
                errs[key] = _rel(t, ref)
                assert errs[key] < 1e-3, (kind, key, errs[key])
            else:
                assert t.abs().max().item() == 0.0, key
    for a, b in zip(outs["host"], outs["cuda"]):
        assert torch.equal(a, b)
    # row b against its own B = 1 call
    full = model.mixture(mel, lens)
    emb_full = emb["x"] * (torch.tensor(lens, dtype=torch.float32).max() / torch.tensor(lens, dtype=torch.float32))[:, None].cuda()
    worst_ulp, worst_rel = 0, 0.0
    for b, n in enumerate(lens):
        one = model.mixture(mel[b:b + 1, :, :n], [n])
        worst_ulp = max(worst_ulp, _ulps(emb_full[b], emb["x"][0]))
        for i, (x, y) in enumerate(zip(full, one)):
            row = x[b] if x.size(0) == len(lens) else x[0]
            worst_rel = max(worst_rel, _rel(row, y[0].cpu()))
    h.remove()
    record_parity(f"mixture {name}", dict(errs, b1_emb_ulps=worst_ulp, b1_rel=worst_rel))
    print(f"{name}: vs reference {errs}; vs B = 1: embedding {worst_ulp} ulps, mixture {worst_rel:.2e}")
    assert worst_ulp <= 4, worst_ulp
    assert worst_rel <= 1e-5, worst_rel
    assert model.training and model.mel_encoder.training


def _mix(B, K, per_row=True, seed=0, spread=3.0):
    g = torch.Generator().manual_seed(seed)
    Bm = B if per_row else 1
    mean = torch.randn(Bm, 80, K, generator=g) * spread
    log_var = torch.rand(Bm, 80, K, generator=g) * 4 - 3
    prob = torch.softmax(torch.randn(B, K, generator=g) * 2, dim=1)
    return mean, log_var, prob


def _rng(seed, counter=0):
    return torch.tensor([seed, counter], dtype=torch.int64, device="cuda")


@pytest.mark.parametrize("K,per_row", [(1, True), (8, True), (8, False), (32, True)])
def test_sampler_matches_the_numpy_restatement(K, per_row):
    from flowtron_b200 import style
    B, T, sigma, seed, ctr = 5, 130, 0.7, 0x5EED + K, 3 + K
    mean, log_var, prob = _mix(B, K, per_row, seed=K)
    n_frames = [130, 1, 64, 97, 33]
    comp = [-1, -1, K - 1, -1, 0]
    rng = _rng(seed, ctr)
    z = style.sample_mixture(mean.cuda(), log_var.cuda(), prob.cuda(), n_frames, T, sigma, comp, rng_state=rng)
    torch.cuda.synchronize()
    assert rng.tolist() == [seed, ctr + 1]
    ref, ks = O.sample(mean.numpy(), log_var.numpy(), prob.numpy(), n_frames, T, sigma, seed, ctr, comp)
    zc = z.double().cpu().numpy()
    valid = ks >= 0
    assert (zc[~valid] == 0).all()
    mb = np.broadcast_to(mean.numpy(), (B, 80, K)) if not per_row else mean.numpy()
    lb = np.broadcast_to(log_var.numpy(), (B, 80, K)) if not per_row else log_var.numpy()
    kk = np.where(valid, ks, 0)
    mu = np.take_along_axis(mb, kk, 2)
    scale = np.abs(mu) + np.abs(ref - mu)                   # |mean| + |sigma sd eps|: the size of the two terms
    err = np.abs(zc - ref)[valid] / np.maximum(scale[valid], 1e-30)
    record_parity(f"sampler K={K} per_row={per_row}", dict(max_err_in_ulps_of_terms=float(err.max() / 2 ** -24)))
    assert err.max() <= 8 * 2.0 ** -24, err.max() / 2 ** -24
    assert (ks[2][valid[2]] == K - 1).all() and (ks[4][valid[4]] == 0).all()


def test_rows_do_not_depend_on_the_batch_or_the_padded_length():
    from flowtron_b200 import style
    B, K, T = 8, 6, 240
    mean, log_var, prob = (t.cuda() for t in _mix(B, K, seed=7))
    n_frames = torch.randint(1, T + 1, (B,), generator=torch.Generator().manual_seed(1)).cuda()
    z8 = style.sample_mixture(mean, log_var, prob, n_frames, T, rng_state=_rng(99, 12))
    z1 = style.sample_mixture(mean[:1], log_var[:1], prob[:1], n_frames[:1], T, rng_state=_rng(99, 12))
    zl = style.sample_mixture(mean, log_var, prob, n_frames, T + 300, rng_state=_rng(99, 12))
    zs = style.sample_mixture(mean[:1], log_var[:1], prob[:1], n_frames[:1], T, component=torch.tensor([-1], device="cuda"),
                              rng_state=_rng(99, 12))
    torch.cuda.synchronize()
    assert torch.equal(z8[0], z1[0]) and torch.equal(z1, zs)
    assert torch.equal(zl[:, :, :T], z8) and (zl[:, :, T:] == 0).all()


def test_a_forced_component_uses_only_its_parameters():
    from flowtron_b200 import style
    B, K, T = 6, 5, 300
    mean = (torch.arange(K, dtype=torch.float32) * 100.0).expand(B, 80, K).contiguous()       # components 100 apart
    log_var = torch.full((B, 80, K), -2.0)
    prob = torch.full((B, K), 1.0 / K)
    comp = torch.tensor([0, 4, 2, -1, 1, 3])
    z = style.sample_mixture(mean.cuda(), log_var.cuda(), prob.cuda(), [T] * B, T, component=comp.cuda(),
                             rng_state=_rng(5)).cpu()
    nearest = (z[..., None] - mean[:, :, None, :]).abs().argmin(-1)                          # [B, 80, T]
    for b, k in enumerate(comp.tolist()):
        if k >= 0:
            assert (nearest[b] == k).all(), b
            assert (z[b] - 100.0 * k).abs().max() < 6 * np.exp(-1.0)
        else:
            assert len(nearest[b].unique()) == K
    # a one-hot prob row selects its component like a forced one
    one_hot = torch.zeros(B, K)
    one_hot[torch.arange(B), torch.tensor([3, 1, 0, 4, 2, 2])] = 1.0
    z = style.sample_mixture(mean.cuda(), log_var.cuda(), one_hot.cuda(), [T] * B, T, rng_state=_rng(6)).cpu()
    nearest = (z[..., None] - mean[:, :, None, :]).abs().argmin(-1)
    assert torch.equal(nearest, one_hot.argmax(1)[:, None, None].expand_as(nearest))


def test_frequencies_means_and_variances_over_2_5m_elements():
    from flowtron_b200 import style
    B, T, K, sigma = 32, 1000, 4, 0.8
    g = torch.Generator().manual_seed(17)
    centres = torch.tensor([-30.0, -10.0, 10.0, 30.0])
    mean = centres.expand(1, 80, K).contiguous()
    log_var = torch.tensor([0.0, -1.0, 0.5, -0.3]).expand(1, 80, K).contiguous()
    prob = torch.softmax(torch.randn(B, K, generator=g), dim=1)
    n_frames = torch.randint(900, T + 1, (B,), generator=g)
    z = style.sample_mixture(mean.cuda(), log_var.cuda(), prob.cuda(), n_frames.cuda(), T, sigma, rng_state=_rng(2024))
    z = z.double().cpu()
    valid = (torch.arange(T)[None, None, :] < n_frames[:, None, None]).expand(B, 80, T)
    assert int(valid.sum()) > 2.5e6 * 0.9
    k = (z[..., None] - centres.double()).abs().argmin(-1)      # components 20 apart, sd <= 1.03: no misassignment at 9 sd
    n_el = (n_frames * 80).double()
    worst = {}
    for c in range(K):
        sel = valid & (k == c)
        n = int(sel.sum())
        p = prob[:, c].double()
        expect = float((n_el * p).sum())
        sd_count = float((n_el * p * (1 - p)).sum()) ** 0.5
        assert abs(n - expect) <= 5 * sd_count, (c, n, expect, sd_count)
        x = z[sel] - float(centres[c])
        sd = sigma * float(np.exp(0.5 * float(log_var[0, 0, c])))
        m, v = float(x.mean()), float(x.var())
        # 5 standard errors of the sample mean and of the sample variance (normal: var(s^2) = 2 sd^4 / (n - 1))
        assert abs(m) <= 5 * sd / n ** 0.5, (c, m)
        assert abs(v / sd ** 2 - 1) <= 5 * (2 / (n - 1)) ** 0.5, (c, v, sd ** 2)
        worst[c] = dict(count_sd=(n - expect) / sd_count, mean_se=m / (sd / n ** 0.5), var_rel=v / sd ** 2 - 1)
    record_parity("sampler statistics", {f"c{c}_{k2}": v for c, d in worst.items() for k2, v in d.items()})
    print(worst)


def test_graph_replays_draw_new_values_equal_to_eager_calls():
    from flowtron_b200 import style
    B, K, T = 4, 8, 200
    mean, log_var, prob = (t.cuda() for t in _mix(B, K, seed=3))
    n_frames = torch.tensor([200, 150, 37, 1], device="cuda")
    rng = _rng(777, 40)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        style.sample_mixture(mean, log_var, prob, n_frames, T, rng_state=rng)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        z = style.sample_mixture(mean, log_var, prob, n_frames, T, rng_state=rng)
    torch.cuda.synchronize()
    c0 = int(rng[1].item())
    graph.replay()
    torch.cuda.synchronize()
    z1 = z.clone()
    graph.replay()
    torch.cuda.synchronize()
    z2 = z.clone()
    assert int(rng[1].item()) == c0 + 2
    assert not torch.equal(z1, z2)
    e1 = style.sample_mixture(mean, log_var, prob, n_frames, T, rng_state=_rng(777, c0))
    e2 = style.sample_mixture(mean, log_var, prob, n_frames, T, rng_state=_rng(777, c0 + 1))
    torch.cuda.synchronize()
    assert torch.equal(z1, e1) and torch.equal(z2, e2)


@pytest.mark.parametrize("K,per_row", [(2, True), (8, False), (32, True)])
def test_responsibilities_match_fp64_and_their_b1_calls(K, per_row):
    from flowtron_b200 import style
    B, T = 6, 170
    mean, log_var, prob = _mix(B, K, per_row, seed=40 + K)
    g = torch.Generator().manual_seed(K)
    z = torch.randn(B, 80, T, generator=g) * 3
    lens = [170, 1, 31, 32, 33, 99]
    z[3, :, 40:] = float("nan")                                 # past row 3's length: never read
    r = style.gmm_responsibilities(z.cuda(), lens, mean.cuda(), log_var.cuda(), prob.cuda())
    rc = style.gmm_responsibilities(z.cuda(), torch.tensor(lens).cuda(), mean.cuda(), log_var.cuda(), prob.cuda())
    ref, _ = O.responsibilities(torch.nan_to_num(z).numpy(), lens, mean.numpy(), log_var.numpy(), prob.numpy())
    err = float((r.double().cpu() - torch.from_numpy(ref)).abs().max())
    record_parity(f"responsibilities K={K} per_row={per_row}", dict(max_abs=err))
    assert err <= 1e-5, err
    assert torch.equal(r, rc)
    assert torch.allclose(r.sum(1).cpu(), torch.ones(B), atol=1e-5)
    for b, n in enumerate(lens):
        sl = slice(b, b + 1) if per_row else slice(0, 1)
        one = style.gmm_responsibilities(z[b:b + 1, :, :n].cuda(), [n], mean[sl].cuda(), log_var[sl].cuda(), prob[b:b + 1].cuda())
        assert torch.equal(one[0], r[b]), b
    # encode's storage order ([T, B, 80] viewed as [B, 80, T]) gives the same bits
    zt = z.cuda().permute(2, 0, 1).contiguous().permute(1, 2, 0)
    assert torch.equal(style.gmm_responsibilities(zt, lens, mean.cuda(), log_var.cuda(), prob.cuda()), r)


def _gm_flowtron(seed):
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=2, n_speakers=1, use_gate_layer=True, n_components=4,
               fixed_gaussian=False, mean_scale=0.0)
    p = synth.synth_gmm_params(cfg, seed)
    kb = [k for k in p if k.endswith("gate_layer.linear_layer.bias")][0]
    p[kb] = torch.full_like(p[kb], -0.3)
    return _model(cfg, p).eval()


def test_mixture_to_audio_replays_from_one_cuda_graph():
    """mixture -> sample_mixture -> infer_batch -> WaveGlow.infer -> Denoiser with CUDA lengths, captured once and replayed
    with new reference mels, lengths, texts and budgets; every replay equals an eager run from the same counter."""
    from flowtron_b200 import _lib, style
    from flowtron_b200.denoiser import Denoiser
    from flowtron_b200.waveglow import WaveGlow
    wcfg = synth.DEFAULT_WAVEGLOW_CONFIG
    wg = WaveGlow(**wcfg)
    wg.load_state_dict(synth.synth_waveglow_params(wcfg, 21), strict=True)
    wg = wg.cuda().eval()
    den = Denoiser(wg)
    m = _gm_flowtron(61)
    B, Tr, T, L, sigma, strength = 4, 180, 200, 40, 0.6, 0.1
    ref = torch.zeros(B, 80, Tr, device="cuda")
    ref_lens = torch.zeros(B, dtype=torch.long, device="cuda")
    text = torch.zeros(B, L, dtype=torch.long, device="cuda")
    spk = torch.zeros(B, dtype=torch.long, device="cuda")
    in_lens = torch.zeros(B, dtype=torch.long, device="cuda")
    n_frames = torch.zeros(B, dtype=torch.long, device="cuda")
    noise = torch.zeros(B, 8, 32 * T, device="cuda")
    rng = _rng(4242)

    def request(seed):
        g = torch.Generator().manual_seed(seed)
        rl = torch.randint(20, Tr + 1, (B,), generator=g)
        return (synth.synth_batch(B, Tr, 4, m_cfg, seed, out_lens=rl.tolist(), logmel_stats=True)["mel"].cuda(), rl,
                torch.randint(1, 100, (B, L), generator=g).cuda(), torch.randint(8, L + 1, (B,), generator=g),
                torch.randint(20, T + 1, (B,), generator=g), torch.randn(B, 8, 32 * T, generator=g).cuda())

    m_cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=2, n_speakers=1)

    def load(req):
        for dst, src in zip((ref, ref_lens, text, in_lens, n_frames, noise), req):
            dst.copy_(src)

    def chain():
        mean, log_var, prob = m.mixture(ref, ref_lens)
        z = style.sample_mixture(mean, log_var, prob, n_frames, T, 0.8, rng_state=rng)
        mel, mel_lens, _ = m.infer_batch(z, spk, text, in_lens, max_frames=n_frames)
        audio = wg.infer(mel, sigma=sigma, noise=noise, lengths=mel_lens)
        return z, mel, mel_lens, audio, den(audio, strength, lengths=HOP * mel_lens)

    with torch.no_grad():
        load(request(100))
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            chain()
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            outs = chain()
        torch.cuda.synchronize()
        for seed in (101, 102):
            req = request(seed)
            load(req)
            c0 = int(rng[1].item())
            graph.replay()
            torch.cuda.synchronize()
            got = [t.clone() for t in outs]
            rng[1] = c0
            want = chain()
            torch.cuda.synchronize()
            z, mel, mel_lens, audio, clean = got
            assert torch.isfinite(audio).all() and torch.isfinite(clean).all()
            assert (mel_lens.cpu() <= req[4]).all() and (mel_lens > 0).all()
            for name, a, b in zip(("z", "mel", "mel_lens", "audio", "clean"), got, want):
                assert torch.equal(a, b), (seed, name)
            print(f"replay {seed}: n_frames {req[4].tolist()} mel_lens {mel_lens.tolist()}")
    assert _lib.device_status() == 0
