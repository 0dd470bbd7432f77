#!/usr/bin/env python
"""Time synthesis from the Gaussian-mixture prior, every arm as CUDA-graph replays.

Arms, alternated within each round:
  sample_cuda   style.sample_mixture at B = 16, T = 1000, K = 8 (learned Gaussians, ragged n_frames U{150..1000})
  sample_torch  the same draw in plain torch: multinomial + randn + gathers + the mask past n_frames
  mixture       Flowtron.mixture on 32 reference mels of U{150..860} frames (K = 8, learned Gaussians)
  chain         mixture -> sample_mixture -> infer_batch -> WaveGlow.infer -> Denoiser, B = 16, reference mels
                U{150..860}, budgets U{150..860} frames, texts U{40..160} tokens, CUDA lengths
Each time is CUDA events around --reps replays after a warm-up replay.  One JSON line per arm and round, with the card
name and power limit read in the same run.  Synthetic weights (2 flows with gate).  Needs a GPU.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from flowtron_b200 import _lib, style, synth  # noqa: E402
from flowtron_b200.denoiser import Denoiser  # noqa: E402
from flowtron_b200.flowtron import Flowtron  # noqa: E402
from flowtron_b200.waveglow import WaveGlow  # noqa: E402

ARMS = ("sample_cuda", "sample_torch", "mixture", "chain")


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        name, plim = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
        return name, float(plim)
    except Exception:                                            # noqa: BLE001 -- reported as unknown, never guessed
        return torch.cuda.get_device_name(0), None


def capture(fn):
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fn()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=side):
        out = fn()
    torch.cuda.synchronize()
    return graph, out


def timed(graph, reps):
    graph.replay()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        graph.replay()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / reps


def torch_sample(mean, log_var, prob, n_frames, T, sigma):
    """The sampler's draw in plain torch: a component per element, then mean + sigma sd eps, zero past n_frames."""
    B, M, K = mean.shape
    k = torch.multinomial(prob, M * T, replacement=True).view(B, M, T)
    eps = torch.randn(B, M, T, device=mean.device)
    z = torch.gather(mean, 2, k) + sigma * torch.gather(torch.exp(0.5 * log_var), 2, k) * eps
    return z.masked_fill(torch.arange(T, device=mean.device)[None, None, :] >= n_frames[:, None, None], 0.0)


def ref_mels(B, seed, cfg):
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(150, 861, (B,), generator=g)
    mel = synth.synth_batch(B, int(lens.max()), 8, cfg, seed, out_lens=lens.tolist(), logmel_stats=True)["mel"]
    return mel.cuda(), lens.cuda()


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--arms", default=",".join(ARMS))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_gmm_sample needs a GPU")
    arms = args.arms.split(",")
    assert all(a in ARMS for a in arms), arms
    name, plim = card()
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=2, n_speakers=1, use_gate_layer=True, n_components=8,
               fixed_gaussian=False, mean_scale=0.0)
    model = Flowtron(**cfg)
    model.load_state_dict(synth.synth_gmm_params(cfg, 1234), strict=True)
    model = model.cuda().eval()
    rng = torch.tensor([1234, 0], dtype=torch.int64, device="cuda")
    graphs = {}
    with torch.no_grad():
        # sampler, B = 16, T = 1000, K = 8
        B, T = 16, 1000
        g = torch.Generator().manual_seed(7)
        mean = (torch.randn(B, 80, 8, generator=g) * 2).cuda()
        log_var = (torch.rand(B, 80, 8, generator=g) * 2 - 1).cuda()
        prob = torch.softmax(torch.randn(B, 8, generator=g), 1).cuda()
        n_frames = torch.randint(150, T + 1, (B,), generator=g).cuda()
        graphs["sample_cuda"] = capture(lambda: style.sample_mixture(mean, log_var, prob, n_frames, T, 0.8, rng_state=rng))
        graphs["sample_torch"] = capture(lambda: torch_sample(mean, log_var, prob, n_frames, T, 0.8))
        # mixture on 32 reference mels
        mel32, lens32 = ref_mels(32, 11, cfg)
        graphs["mixture"] = capture(lambda: model.mixture(mel32, lens32))
        # the whole chain at B = 16
        wcfg = synth.DEFAULT_WAVEGLOW_CONFIG
        wg = WaveGlow(**wcfg)
        wg.load_state_dict(synth.synth_waveglow_params(wcfg, 21), strict=True)
        wg = wg.cuda().eval()
        den = Denoiser(wg)
        mel16, lens16 = ref_mels(16, 12, cfg)
        g = torch.Generator().manual_seed(13)
        budgets = torch.randint(150, 861, (16,), generator=g).cuda()
        in_lens = torch.randint(40, 161, (16,), generator=g).cuda()
        text = torch.randint(1, 185, (16, 160), generator=g).cuda()
        spk = torch.zeros(16, dtype=torch.long, device="cuda")
        Tc = 860
        noise = torch.randn(16, 8, 32 * Tc, generator=g).cuda()

        def chain():
            mu, lv, pr = model.mixture(mel16, lens16)
            z = style.sample_mixture(mu, lv, pr, budgets, Tc, 0.8, rng_state=rng)
            mel, mel_lens, _ = model.infer_batch(z, spk, text, in_lens, max_frames=budgets)
            audio = wg.infer(mel, sigma=0.6, noise=noise, lengths=mel_lens)
            return den(audio, 0.01, lengths=256 * mel_lens), mel_lens
        graphs["chain"] = capture(chain)
        frames = int(graphs["chain"][1][1].sum())
        for r in range(args.rounds):
            for arm in (arms if r % 2 == 0 else arms[::-1]):
                ms = timed(graphs[arm][0], args.reps)
                rec = {"arm": arm, "round": r, "ms_per_call": round(ms, 4)}
                if arm.startswith("sample"):
                    rec.update(B=B, T=T, K=8, elements=B * 80 * T)
                elif arm == "mixture":
                    rec.update(B=32, frames=int(lens32.sum()))
                else:
                    rec.update(B=16, mel_frames_out=frames, audio_s=round(frames * 256 / 22050, 2))
                assert _lib.device_status() == 0
                print(json.dumps({**rec, "gpu": name, "power_limit_w": plim}), flush=True)


if __name__ == "__main__":
    main()
