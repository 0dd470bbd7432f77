#!/usr/bin/env python
"""Time one WaveGlow training step (WaveGlow.forward + WaveGlowLoss + backward + torch.optim.Adam) on the GPU at the
reference training shape (tacotron2/waveglow/config.json: batch 12 x 16000-sample segments, shipped model config).

Reported, one JSON line per variant: ms per step (warm-up, then `--runs` timed windows of `--steps` steps each, CUDA
events), audio samples/s, and model FLOP/s over step time with the FLOP count computed below from the shapes (forward
tensor work x 3 for forward + backward).  Variants:
  kernels_graph   this library, the whole step replayed from one CUDA graph
  kernels_eager   this library, eager
  torch_fp32      the fp32 oracle module (tests/waveglow_oracle.py) in plain torch on the same GPU
  torch_autocast  the same under torch.autocast(float16)
The card name and power limit are read in the same run.  Needs a GPU; there is no CPU path.
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

from flowtron_b200 import synth  # noqa: E402
from flowtron_b200.waveglow import WaveGlow, WaveGlowLoss  # noqa: E402
import waveglow_oracle as O  # noqa: E402


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        name, plim = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
        return name, float(plim)
    except Exception:                                            # noqa: BLE001 -- reported as unknown, never guessed
        return torch.cuda.get_device_name(0), None


def train_flops(cfg, B, N):
    """Forward tensor FLOPs of WaveGlow.forward on B x N samples, times 3 (backward = 2x forward)."""
    C, L = cfg["WN_config"]["n_channels"], cfg["WN_config"]["n_layers"]
    rows = B * N // cfg["n_group"]
    fwd = 0.0
    for c, nh in synth.waveglow_channels(cfg):
        per_row = 2 * (3 * C + 640) * 2 * C * L + 2 * C * 2 * C * (L - 1) + 2 * C * C + 2 * nh * C + 2 * C * 2 * nh + 2 * c * c
        fwd += rows * per_row
    fwd += 2 * (B * N) * 80 * 80 * 4                             # upsample: each sample sums 4 frames x 80 channels per channel
    return 3 * fwd, fwd


def timed(step, warmup, steps, runs):
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    out = []
    for _ in range(runs):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(steps):
            step()
        b.record()
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b) / steps)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=12)
    ap.add_argument("--samples", type=int, default=16000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--skip-torch", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_waveglow_train needs a GPU")
    cfg = synth.DEFAULT_WAVEGLOW_CONFIG
    B, N = args.batch, args.samples
    Fr = 1 + N // 256
    spect = synth.synth_waveglow_mel(B, Fr, 1).cuda()
    audio = (0.3 * torch.randn(B, N, generator=torch.Generator().manual_seed(2))).clamp(-1, 1).cuda()
    name, plim = card()
    flops, fwd_flops = train_flops(cfg, B, N)
    crit = WaveGlowLoss(1.0)

    def report(variant, ms, extra=None):
        best = min(ms)
        rec = dict(variant=variant, batch=B, samples=N, ms_per_step=[round(x, 3) for x in ms],
                   samples_per_s=round(B * N / (best / 1e3)), model_tflops_per_s=round(flops / (best / 1e3) / 1e12, 1),
                   model_tflop_per_step=round(flops / 1e12, 3), forward_tflop=round(fwd_flops / 1e12, 3),
                   card=name, power_limit_w=plim)
        rec.update(extra or {})
        print(json.dumps(rec), flush=True)

    model = WaveGlow(**cfg)
    model.load_state_dict(synth.synth_waveglow_params(cfg, 1))
    model = model.cuda().train()
    opt = torch.optim.Adam(model.parameters(), lr=1e-4, capturable=True)

    def step():
        opt.zero_grad(set_to_none=False)
        loss = crit(model((spect, audio)))
        loss.backward()
        opt.step()
        return loss

    eager = timed(step, args.warmup, args.steps, args.runs)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        step()
    report("kernels_graph", timed(graph.replay, args.warmup, args.steps, args.runs),
           dict(peak_mem_gb=round(torch.cuda.max_memory_allocated() / 2**30, 2)))
    report("kernels_eager", eager)
    del graph, opt, model
    torch.cuda.empty_cache()
    if args.skip_torch:
        return
    sd = {k: v.cuda().requires_grad_(True) for k, v in synth.synth_waveglow_params(cfg, 1).items()}
    ropt = torch.optim.Adam(list(sd.values()), lr=1e-4)

    def ref_step(autocast):
        ropt.zero_grad()
        with torch.autocast("cuda", dtype=torch.float16, enabled=autocast):
            out = O.waveglow_forward(sd, spect, audio)
        loss = O.waveglow_loss((out[0].float(), [t.float() for t in out[1]], [t.float() for t in out[2]]), 1.0)
        loss.backward()
        ropt.step()

    for variant, ac in (("torch_fp32", False), ("torch_autocast", True)):
        torch.cuda.reset_peak_memory_stats()
        ms = timed(lambda: ref_step(ac), args.warmup, args.steps, args.runs)
        report(variant, ms, dict(peak_mem_gb=round(torch.cuda.max_memory_allocated() / 2**30, 2)))


if __name__ == "__main__":
    main()
