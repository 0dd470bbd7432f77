#!/usr/bin/env python
"""Time WaveGlow.infer (csrc/waveglow.cu) on the GPU; one JSON line per workload, in the style of bench.py.

Workloads (--workloads, default all):
  b1       B=1, 400 frames (inference.py's default n_frames)
  b16      B=16, 400 frames
  ragged   16 utterances of U{150..860} frames
  e2e      Flowtron.infer (2 flows, B=1, 400 frames, gate disabled as in bench.py --workload infer) then WaveGlow.infer

Reported: ms per call from CUDA-graph replay and eager, audio samples/s and x real time (22050 Hz), kernel launches per
call, achieved TFLOP/s of the WaveGlow model FLOPs (waveglow_flops) and its fraction of the 989 TFLOP/s dense-fp16
H100 SXM data-sheet figure (a data-sheet number, not a measured peak), plus the card name and power limit read in the
same run.  The b1 output is checked against the CPU fp32 oracle (tests/waveglow_oracle.py) at the timed size.
Needs a GPU; there is no CPU path.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from flowtron_b200 import _lib, synth  # noqa: E402
from flowtron_b200.waveglow import WaveGlow, waveglow_flops  # noqa: E402

PEAK_FP16_DENSE = 989e12
SR = 22050


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        name, plim = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
        return name, float(plim)
    except Exception:                                            # noqa: BLE001 -- reported as unknown, never guessed
        return torch.cuda.get_device_name(0), None


def time_eager(fn, warmup, iters):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def time_graph(fn, warmup, iters):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    for _ in range(warmup):
        g.replay()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        g.replay()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="b1,b16,ragged,e2e")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-check", action="store_true", help="skip the oracle check of the b1 output")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_waveglow.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    name, plim = card()
    cfg = synth.DEFAULT_WAVEGLOW_CONFIG
    sd = synth.synth_waveglow_params(cfg, 1234)
    wg = WaveGlow(**cfg)
    wg.load_state_dict(sd, strict=True)
    wg = wg.to(dev).eval()
    sigma = 0.6

    for wl in args.workloads.split(","):
        extra = {}
        if wl in ("b1", "b16", "e2e"):
            B, Fr = (16, 400) if wl == "b16" else (1, 400)
            lengths = None
            frames = [Fr] * B
        elif wl == "ragged":
            g = torch.Generator().manual_seed(4321)
            frames = torch.randint(150, 861, (16,), generator=g).tolist()
            B, Fr, lengths = 16, max(frames), frames
        else:
            raise SystemExit(f"unknown workload {wl}")
        mel = synth.synth_waveglow_mel(B, Fr, 1234).to(dev)
        noise = synth.synth_waveglow_noise(B, Fr, 1234).to(dev)
        if wl == "e2e":
            from flowtron_b200.flowtron import Flowtron
            fcfg = dict(synth.DEFAULT_MODEL_CONFIG)
            params = synth.synth_params(fcfg, 1234)
            key = [k for k in params if k.endswith("gate_layer.linear_layer.bias")][0]
            params[key] = torch.full_like(params[key], -10.0)       # the gate never fires: all 400 frames are produced
            ft = Flowtron(**fcfg)
            ft.load_state_dict(params, strict=True)
            ft = ft.to(dev).eval()
            gen = torch.Generator().manual_seed(1234)
            res = (torch.randn(1, 80, Fr, generator=gen) * 0.5).to(dev)
            text = torch.randint(0, fcfg["n_text"], (1, 100), generator=gen).to(dev)
            spk = torch.zeros(1, dtype=torch.long, device=dev)

            def fn():
                with torch.no_grad():
                    m, _ = ft.infer(res, spk, text, temperature=1.0, gate_threshold=0.5)
                return wg.infer(m, sigma=sigma, noise=noise)
        else:
            def fn():
                return wg.infer(mel, sigma=sigma, noise=noise, lengths=lengths)

        _lib.reset_launch_count()
        fn()
        torch.cuda.synchronize()
        launches = _lib.launch_count()
        eager_ms = time_eager(fn, args.warmup, args.iters)
        graph_ms = None
        if wl != "e2e":                                          # Flowtron.infer reads its gate result on the host
            graph_ms = time_graph(fn, args.warmup, args.iters)
        assert _lib.device_status() == 0
        samples = 256 * sum(frames)
        best = graph_ms if graph_ms is not None else eager_ms
        flops = waveglow_flops(sum(frames), cfg)
        if wl == "b1" and not args.no_check:
            import waveglow_oracle as WO
            out = fn().cpu()
            t0 = time.time()
            ref = WO.waveglow_infer(sd, mel.cpu(), noise.cpu(), sigma, cfg)
            extra["oracle_max_rel_err"] = (out - ref).abs().max().item() / ref.abs().max().item()
            extra["oracle_cpu_s"] = round(time.time() - t0, 2)
        rec = dict(workload=f"waveglow_{wl}", B=B, frames=sum(frames), max_frames=Fr, sigma=sigma,
                   graph_ms=None if graph_ms is None else round(graph_ms, 3), eager_ms=round(eager_ms, 3),
                   audio_samples_per_s=round(samples / (best / 1e3)), x_real_time=round(samples / SR / (best / 1e3), 1),
                   launches_per_call=launches, waveglow_gflop=round(flops / 1e9, 1),
                   achieved_tflops=round(flops / (best / 1e3) / 1e12, 1),
                   frac_of_datasheet_fp16_dense=round(flops / (best / 1e3) / PEAK_FP16_DENSE, 3),
                   gpu=name, power_limit_w=plim, **extra)
        if wl == "e2e":
            rec["note"] = "time includes Flowtron.infer (2 flows); TFLOP/s counts WaveGlow FLOPs only"
        print(json.dumps(rec), flush=True)
        if "oracle_max_rel_err" in extra and not extra["oracle_max_rel_err"] <= 1e-3:
            raise SystemExit(f"waveglow_{wl}: output differs from the oracle by {extra['oracle_max_rel_err']:.3e} (> 1e-3)")


if __name__ == "__main__":
    main()
