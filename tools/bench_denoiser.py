#!/usr/bin/env python
"""Time the WaveGlow Denoiser and Griffin-Lim (csrc/istft.cu + the fused STFT transform) on the GPU; one JSON line per
workload, in the style of tools/bench_waveglow.py.

Workloads (--workloads, default all):
  b16      Denoiser.forward on B=16 x 400 frames of audio (102,400 samples per row), strength 0.1
  ragged   Denoiser.forward on 16 utterances of U{150..860} frames, with lengths
  gl       griffin_lim, 30 iterations, B=1 x 400 frames, explicit angles (graph replay)
  e2e      WaveGlow.infer (B=1, 400 frames) then the Denoiser, each timed on its own in the same run

Reported: ms per call from CUDA-graph replay (not for ragged, whose offsets are copied from the host) and eager, x real time (22050 Hz), kernel launches per call, the algorithmic
HBM bytes (waveform read and written once, magnitude and phase written and read once) and the achieved fraction of the
3.35 TB/s HBM3 H100 SXM data-sheet figure (a data-sheet number, not a measured peak), plus the card name and power limit
read in the same run.  e2e reports the Denoiser's time as a share of WaveGlow.infer's.  Needs a GPU; there is no CPU path.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_waveglow import card, time_eager, time_graph  # noqa: E402
from flowtron_b200 import _lib, synth  # noqa: E402
from flowtron_b200.audio_processing import griffin_lim  # noqa: E402
from flowtron_b200.denoiser import Denoiser  # noqa: E402
from flowtron_b200.waveglow import WaveGlow  # noqa: E402

HBM_DATASHEET = 3.35e12
SR, HOP = 22050, 256


def stft_bytes(samples, frames):
    """One transform + one inverse: waveform read and written, magnitude + phase ([513] floats each per frame) written
    by the transform and read by the inverse."""
    return 4 * 2 * samples + 4 * 2 * 2 * 513 * frames


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="b16,ragged,gl,e2e")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_denoiser.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    name, plim = card()
    cfg = synth.DEFAULT_WAVEGLOW_CONFIG
    wg = WaveGlow(**cfg)
    wg.load_state_dict(synth.synth_waveglow_params(cfg, 1234), strict=True)
    wg = wg.to(dev).eval()
    den = Denoiser(wg)

    for wl in args.workloads.split(","):
        extra = {}
        if wl in ("b16", "ragged"):
            if wl == "b16":
                frames, lengths = [400] * 16, None
            else:
                g = torch.Generator().manual_seed(4321)
                frames = torch.randint(150, 861, (16,), generator=g).tolist()
                lengths = [HOP * f for f in frames]
            audio = synth.synth_istft_audio(len(frames), HOP * max(frames), 1234).to(dev)

            def fn():
                return den(audio, 0.1, lengths=lengths)
            samples = HOP * sum(frames)
            nbytes = stft_bytes(samples, sum(f + 1 for f in frames))
        elif wl == "gl":
            stft = den.stft
            mag, _ = stft.transform(synth.synth_istft_audio(1, HOP * 400, 1234).to(dev))
            angles = (torch.rand(mag.shape, generator=torch.Generator().manual_seed(1234)) * 6.283185307179586 - 3.141592653589793).to(dev)

            def fn():
                return griffin_lim(mag, stft, 30, angles=angles)
            frames, samples = [400], HOP * 400
            nbytes = 61 * stft_bytes(samples, 401) // 2           # 31 inverses + 30 transforms
        elif wl == "e2e":
            mel = synth.synth_waveglow_mel(1, 400, 1234).to(dev)
            noise = synth.synth_waveglow_noise(1, 400, 1234).to(dev)
            audio = wg.infer(mel, sigma=0.6, noise=noise)

            def wg_fn():
                return wg.infer(mel, sigma=0.6, noise=noise)

            def fn():
                return den(wg_fn(), 0.1)
            frames, samples = [400], HOP * 400
            nbytes = stft_bytes(samples, 401)
            wg_ms = time_graph(wg_fn, args.warmup, args.iters)
            den_ms = time_graph(lambda: den(audio, 0.1), args.warmup, args.iters)
            extra = dict(waveglow_graph_ms=round(wg_ms, 3), denoiser_graph_ms=round(den_ms, 4),
                         denoiser_share_of_waveglow=round(den_ms / wg_ms, 5))
        else:
            raise SystemExit(f"unknown workload {wl}")

        _lib.reset_launch_count()
        fn()
        torch.cuda.synchronize()
        launches = _lib.launch_count()
        eager_ms = time_eager(fn, args.warmup, args.iters)
        graph_ms = None
        if wl != "ragged":                                       # lengths are host prefix sums copied on every call
            graph_ms = time_graph(fn, args.warmup, args.iters)
        assert _lib.device_status() == 0
        best = graph_ms if graph_ms is not None else eager_ms
        rec_bytes_ms = extra["denoiser_graph_ms"] if wl == "e2e" else best
        rec = dict(workload=f"denoiser_{wl}" if wl != "gl" else "griffin_lim_30", B=len(frames), frames=sum(frames),
                   graph_ms=None if graph_ms is None else round(graph_ms, 4), eager_ms=round(eager_ms, 4),
                   x_real_time=round(samples / SR / (best / 1e3), 1), launches_per_call=launches,
                   hbm_bytes=int(nbytes), hbm_tb_per_s=round(nbytes / (rec_bytes_ms / 1e3) / 1e12, 3),
                   frac_of_datasheet_hbm=round(nbytes / (rec_bytes_ms / 1e3) / HBM_DATASHEET, 4),
                   gpu=name, power_limit_w=plim, **extra)
        if wl == "e2e":
            rec["note"] = "graph/eager ms are WaveGlow.infer + Denoiser; HBM figures are for the Denoiser alone"
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
