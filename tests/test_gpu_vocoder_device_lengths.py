"""GPU: WaveGlow.infer and the Denoiser with per-row lengths in device memory.  CUDA lengths give rows bit-identical to host
lengths, make no host synchronisation, and let infer_batch -> WaveGlow.infer -> Denoiser be captured once as a CUDA graph
and replayed with new texts, text lengths, frame budgets and noise."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from flowtron_b200 import synth

pytestmark = pytest.mark.gpu

WCFG = synth.DEFAULT_WAVEGLOW_CONFIG
HOP = 256


def _waveglow(seed):
    from flowtron_b200.waveglow import WaveGlow
    m = WaveGlow(**WCFG)
    m.load_state_dict(synth.synth_waveglow_params(WCFG, seed), strict=True)
    return m.cuda().eval()


def _flowtron(seed, gate_bias=-0.3, gate_scale=40.0):
    from flowtron_b200.flowtron import Flowtron
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=2, n_speakers=1, use_gate_layer=True)
    p = synth.synth_params(cfg, seed)
    kb = [k for k in p if k.endswith("gate_layer.linear_layer.bias")][0]
    kw = [k for k in p if k.endswith("gate_layer.linear_layer.weight")][0]
    p[kb] = torch.full_like(p[kb], gate_bias)
    p[kw] = p[kw] * gate_scale
    m = Flowtron(**cfg)
    m.load_state_dict(p, strict=True)
    return m.cuda().eval()


def _wg_case(case):
    if case == "golden":
        g = dict(np.load(os.path.join(GOLDEN, "waveglow_ragged.npz")))
        seed, B, Fr = int(g["seed"]), int(g["B"]), int(g["F"])
        return seed, synth.synth_waveglow_mel(B, Fr, seed), synth.synth_waveglow_noise(B, Fr, seed), float(g["sigma"]), \
            g["lengths"].tolist()
    gen = torch.Generator().manual_seed(31)
    lengths = torch.randint(150, 861, (16,), generator=gen).tolist()
    Fr = max(lengths)
    return 31, synth.synth_waveglow_mel(16, Fr, 31), synth.synth_waveglow_noise(16, Fr, 31), 0.6, lengths


@pytest.mark.parametrize("case", ["golden", "b16_u150_860"])
def test_waveglow_device_lengths_equal_host_lengths(case):
    from flowtron_b200 import _lib
    seed, mel, noise, sigma, lengths = _wg_case(case)
    m = _waveglow(seed)
    mel, noise = mel.cuda(), noise.cuda()
    with torch.no_grad():
        host = m.infer(mel, sigma=sigma, noise=noise, lengths=lengths)
        for dtype in (torch.int32, torch.int64):
            dev = m.infer(mel, sigma=sigma, noise=noise, lengths=torch.tensor(lengths, dtype=dtype, device="cuda"))
            assert torch.equal(dev, host), dtype
    for b, n in enumerate(lengths):
        assert (host[b, 256 * n:] == 0).all(), b
    torch.cuda.synchronize()
    assert _lib.device_status() == 0


def test_waveglow_device_lengths_argument_checks():
    m = _waveglow(3)
    mel = synth.synth_waveglow_mel(2, 8, 3).cuda()
    for bad in (torch.tensor([8, 8, 8], device="cuda"), torch.tensor([[8, 8]], device="cuda"),
                torch.tensor([8.0, 8.0], device="cuda"), torch.tensor([8, 8], dtype=torch.int16, device="cuda")):
        with pytest.raises(ValueError):
            m.infer(mel, sigma=0.5, lengths=bad)
    with pytest.raises(ValueError):                            # host lengths are still range-checked
        m.infer(mel, sigma=0.5, lengths=[8, 9])


def _denoiser(wg):
    from flowtron_b200.denoiser import Denoiser
    return Denoiser(wg)


def test_denoiser_device_lengths_equal_host_lengths():
    from flowtron_b200 import _lib
    den = _denoiser(_waveglow(14))
    lengths = [256 * 40, 256 * 23, 256 * 31 + 77, 256 * 3]
    N = 256 * 41 + 13
    audio = synth.synth_istft_audio(len(lengths) + 1, N, 70).cuda()
    host = den(audio[:4], 0.3, lengths=lengths)
    for short in (512, 300):
        with pytest.raises(ValueError):                        # a host row at or below n_fft / 2 is refused ...
            den(audio, 0.3, lengths=lengths + [short])
        with pytest.raises(ValueError):                        # ... as is a B = 1 call on it
            den(audio[4:, :short], 0.3)
        for dtype in (torch.int32, torch.int64):
            dev = den(audio, 0.3, lengths=torch.tensor(lengths + [short], dtype=dtype, device="cuda"))
            assert tuple(dev.shape) == (5, 1, (N // 256) * 256)
            assert torch.equal(dev[:4], host), (short, dtype)
            assert (dev[4] == 0).all(), (short, dtype)         # ... and on the device comes out all zero
    torch.cuda.synchronize()
    assert _lib.device_status() == 0


def test_no_host_synchronisation_with_cuda_lengths():
    from flowtron_b200 import _lib
    wg = _waveglow(14)
    den = _denoiser(wg)
    m = _flowtron(61)
    B, T, L = 4, 36, 18
    g = torch.Generator().manual_seed(13)
    res = (torch.randn(B, 80, T, generator=g) * 0.5).cuda()
    text = torch.randint(0, 185, (B, L), generator=g).cuda()
    spk = torch.zeros(B, dtype=torch.long, device="cuda")
    in_lens = torch.tensor([18, 6, 12, 15], device="cuda")
    max_frames = torch.tensor([36, 20, 28, 2], device="cuda")
    noise = synth.synth_waveglow_noise(B, T, 15).cuda()
    mel = synth.synth_waveglow_mel(B, T, 15).cuda()
    frames = torch.tensor([36, 9, 20, 3], dtype=torch.int32, device="cuda")
    audio = synth.synth_istft_audio(B, 256 * T, 16).cuda()

    def chain():
        mel_b, mel_lens, _ = m.infer_batch(res, spk, text, in_lens, max_frames=max_frames)
        a = wg.infer(mel_b, sigma=0.6, noise=noise, lengths=mel_lens)
        return den(a, 0.1, lengths=HOP * mel_lens)

    with torch.no_grad():
        wg.infer(mel, sigma=0.6, noise=noise, lengths=frames)  # warm-up: packed weights and scratch exist
        den(audio, 0.1, lengths=frames * HOP)
        chain()
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            wg.infer(mel, sigma=0.6, noise=noise, lengths=frames)
            wg.infer(mel, sigma=0.6, noise=noise, lengths=frames.long())
            den(audio, 0.1, lengths=frames * HOP)
            den(audio, 0.1, lengths=(frames * HOP).long())
            chain()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert _lib.device_status() == 0


def test_launch_counts_with_cuda_lengths():
    from flowtron_b200 import _lib
    wg = _waveglow(13)
    den = _denoiser(wg)
    mel, z = synth.synth_waveglow_mel(2, 12, 13).cuda(), synth.synth_waveglow_noise(2, 12, 13).cuda()
    frames = torch.tensor([12, 7], dtype=torch.int32, device="cuda")
    with torch.no_grad():
        wg.infer(mel, sigma=0.6, noise=z, lengths=frames)
        _lib.reset_launch_count()
        host = wg.infer(mel, sigma=0.6, noise=z, lengths=[12, 7])
        n_host = _lib.launch_count()
        _lib.reset_launch_count()
        audio = wg.infer(mel, sigma=0.6, noise=z, lengths=frames)
        n_wg = _lib.launch_count()
        _lib.reset_launch_count()
        den(audio, 0.1, lengths=frames * HOP)
        n_den = _lib.launch_count()
    print(f"launches with CUDA lengths: WaveGlow.infer {n_wg}, Denoiser {n_den}")
    assert torch.equal(audio, host)
    assert n_wg == n_host == WCFG["n_flows"] * (2 * WCFG["WN_config"]["n_layers"] + 1) + 4, (n_wg, n_host)
    assert n_den == 3                                          # pack rows, transform, inverse


def test_one_graph_serves_many_requests():
    """infer_batch -> WaveGlow.infer -> Denoiser captured once at B = 16, T = 1000, L = 160 on static buffers, replayed with
    new texts, in_lens, max_frames and noise; every replay equals eager runs of the same inputs with host lengths."""
    from flowtron_b200 import _lib
    wg = _waveglow(21)
    den = _denoiser(wg)
    m = _flowtron(61)
    B, T, L, sigma, strength = 16, 1000, 160, 0.6, 0.1
    res = torch.zeros(B, 80, T, device="cuda")
    text = torch.zeros(B, L, dtype=torch.long, device="cuda")
    spk = torch.zeros(B, dtype=torch.long, device="cuda")
    in_lens = torch.zeros(B, dtype=torch.long, device="cuda")
    max_frames = torch.zeros(B, dtype=torch.long, device="cuda")
    noise = torch.zeros(B, 8, 32 * T, device="cuda")

    def request(seed):
        g = torch.Generator().manual_seed(seed)
        il = torch.randint(40, L + 1, (B,), generator=g)
        mf = torch.randint(150, T + 1, (B,), generator=g)
        mf[seed % B] = 2                                       # a row whose budget is 2 frames: denoised to silence
        return ((torch.randn(B, 80, T, generator=g) * 0.5).cuda(), torch.randint(0, 185, (B, L), generator=g).cuda(),
                il, mf, torch.randn(B, 8, 32 * T, generator=g).cuda())

    def load(req):
        r, t, il, mf, z = req
        res.copy_(r); text.copy_(t); in_lens.copy_(il); max_frames.copy_(mf); noise.copy_(z)

    def chain():
        mel, mel_lens, _ = m.infer_batch(res, spk, text, in_lens, max_frames=max_frames)
        audio = wg.infer(mel, sigma=sigma, noise=noise, lengths=mel_lens)
        return mel, mel_lens, audio, den(audio, strength, lengths=HOP * mel_lens)

    with torch.no_grad():
        load(request(100))
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            chain()                                            # warm-up: packed weights and scratch exist before capture
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            outs = chain()
        for seed in (101, 102, 103):
            req = request(seed)
            load(req)
            graph.replay()
            torch.cuda.synchronize()
            mel_g, lens_g, audio_g, clean_g = (t.clone() for t in outs)
            r, t, il, mf, z = req
            mel_e, lens_e, _ = m.infer_batch(r, spk, t, il.tolist(), max_frames=mf.tolist())
            lens = lens_e.tolist()
            audio_e = wg.infer(mel_e, sigma=sigma, noise=z, lengths=lens)
            assert torch.equal(lens_g, lens_e), seed
            assert torch.equal(mel_g, mel_e), seed
            assert torch.equal(audio_g, audio_e), seed
            assert min(lens) <= 2, (seed, lens)
            long_rows = [b for b, n in enumerate(lens) if HOP * n > 512]
            if long_rows:                                      # host lengths refuse the short rows: compare the others
                clean_e = den(audio_e[long_rows], strength, lengths=[HOP * lens[b] for b in long_rows])
                assert torch.equal(clean_g[long_rows], clean_e), seed
            print(f"replay {seed}: mel_lens {lens}")
            for b, n in enumerate(lens):
                assert (audio_g[b, HOP * n:] == 0).all() and (clean_g[b, 0, HOP * n:] == 0).all(), (seed, b)
                if HOP * n <= 512:
                    assert (clean_g[b] == 0).all(), (seed, b)
    torch.cuda.synchronize()
    assert _lib.device_status() == 0
