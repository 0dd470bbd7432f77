#!/usr/bin/env python
"""Time style transfer by posterior sampling on the GPU; one JSON line per workload and repetition, then one summary line
per workload.

Workloads (fixed seed; 2-flow model at the shipped sizes; gate bias -10 so the gate never fires and the work is fixed):
  encode     Flowtron.encode of 32 reference utterances of U{150..860} frames (texts of round(len / 6.5) tokens, at least
             20): one padded-batch call against 32 B = 1 calls on the unpadded inputs (the reference notebook's loop).
             The batched call is timed with host lengths (rows under 320 frames run as a second launch) and with CUDA
             length tensors (one launch).  Reported: ms per set, valid mel frames per second, the speed-up, and the
             largest difference of a batched row from its B = 1 run relative to max |z|.
  posterior  style.posterior_mean of that z, 'batch' at 400 frames and 'time_and_batch': mean of --iters-fast calls, eager
             (host-bound: argument checks and the ctypes call) and replayed from a CUDA graph (the kernel and its launch).
  chain      posterior_mean ('batch', 400 frames) + sigma * noise -> Flowtron.infer (B = 1, 400 frames) -> WaveGlow.infer
             (sigma 0.75) -> Denoiser (strength 0.01).

Times come from CUDA events around work that ends in a device synchronise, after warming up every shape; each workload is
repeated --reps times.  The card name and power limit are read in the same run.  Needs a GPU; there is no CPU path.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_waveglow import card, time_eager, time_graph  # noqa: E402
from flowtron_b200 import _lib, synth  # noqa: E402
from flowtron_b200.denoiser import Denoiser  # noqa: E402
from flowtron_b200.flowtron import Flowtron  # noqa: E402
from flowtron_b200.style import posterior_mean  # noqa: E402
from flowtron_b200.waveglow import WaveGlow  # noqa: E402

K, N_FRAMES, SIGMA = 32, 400, 0.5


def reference_set(dev, seed=2027):
    g = torch.Generator().manual_seed(seed)
    out_lens = torch.randint(150, 861, (K,), generator=g)
    in_lens = torch.clamp(torch.round(out_lens.double() / 6.5).long(), 20, 160)
    T, L = int(out_lens.max()), int(in_lens.max())
    mel = (torch.randn(K, 80, T, generator=g) * 2.0 - 5.5).clamp_(-11.5, 2.0).to(dev)
    text = torch.randint(0, 185, (K, L), generator=g).to(dev)
    spk = torch.zeros(K, dtype=torch.long, device=dev)
    return mel, spk, text, in_lens.tolist(), out_lens.tolist()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--iters-fast", type=int, default=200)
    ap.add_argument("--workloads", default="encode,posterior,chain")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_style_transfer.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    name, plim = card()
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=2)
    p = synth.synth_params(cfg, 1234)
    key = [k for k in p if k.endswith("gate_layer.linear_layer.bias")][0]
    p[key] = torch.full_like(p[key], -10.0)
    model = Flowtron(**cfg)
    model.load_state_dict(p, strict=True)
    model = model.to(dev).eval()
    torch.set_grad_enabled(False)
    mel, spk, text, in_lens, out_lens = reference_set(dev)
    in_d, out_d = torch.tensor(in_lens, device=dev), torch.tensor(out_lens, device=dev)
    frames = sum(out_lens)

    def batched():
        return model.encode(mel, spk, text, in_lens, out_lens)

    def batched_dev():
        return model.encode(mel, spk, text, in_d, out_d)

    def sequential():
        return [model.encode(mel[b:b + 1, :, :n], spk[b:b + 1], text[b:b + 1, :nl], [nl], [n])
                for b, (nl, n) in enumerate(zip(in_lens, out_lens))]

    # outputs at the timed sizes: every batched row against its B = 1 run
    z = batched()
    z_dev = batched_dev()
    singles = sequential()
    zmax = max(s.abs().max().item() for s in singles)
    row_diff = max((z[b, :, :n] - s[0]).abs().max().item() for b, (n, s) in enumerate(zip(out_lens, singles))) / zmax
    row_diff_dev = max((z_dev[b, :, :n] - s[0]).abs().max().item() for b, (n, s) in enumerate(zip(out_lens, singles))) / zmax
    assert _lib.device_status() == 0
    base = dict(K=K, T=mel.shape[-1], L=text.shape[1], valid_frames=frames, n_frames=N_FRAMES, gpu=name, power_limit_w=plim)

    wg = den = None
    if "chain" in args.workloads:
        wcfg = synth.DEFAULT_WAVEGLOW_CONFIG
        wg = WaveGlow(**wcfg)
        wg.load_state_dict(synth.synth_waveglow_params(wcfg, 1234), strict=True)
        wg = wg.to(dev).eval()
        den = Denoiser(wg)
    g = torch.Generator().manual_seed(7)
    noise = torch.randn(1, 80, N_FRAMES, generator=g).to(dev)
    new_text = torch.randint(0, 185, (1, 60), generator=g).to(dev)

    def chain():
        mu = posterior_mean(z, out_d, N_FRAMES)
        m1, _ = model.infer(mu + SIGMA * noise, spk[:1], new_text)
        return den(wg.infer(m1.contiguous(), sigma=0.75), 0.01)

    for wl in args.workloads.split(","):
        runs = []
        for rep in range(args.reps):
            if wl == "encode":
                bat = time_eager(batched, 1, args.iters)
                bat_dev = time_eager(batched_dev, 1, args.iters)
                seq = time_eager(sequential, 1, 1)
                rec = dict(workload="encode", rep=rep, batched_ms=round(bat, 2), batched_cuda_lens_ms=round(bat_dev, 2),
                           sequential_b1_ms=round(seq, 2), frames_per_s_batched=round(frames / (bat / 1e3)),
                           frames_per_s_sequential=round(frames / (seq / 1e3)), speedup=round(seq / bat, 2),
                           max_row_rel_diff=row_diff, max_row_rel_diff_cuda_lens=row_diff_dev)
            elif wl == "posterior":
                fb = lambda: posterior_mean(z, out_d, N_FRAMES)                                  # noqa: E731
                ft = lambda: posterior_mean(z, out_d, N_FRAMES, aggregation="time_and_batch")    # noqa: E731
                rec = dict(workload="posterior", rep=rep,
                           batch_eager_us=round(time_eager(fb, 10, args.iters_fast) * 1e3, 1),
                           batch_graph_us=round(time_graph(fb, 10, args.iters_fast) * 1e3, 1),
                           time_and_batch_eager_us=round(time_eager(ft, 10, args.iters_fast) * 1e3, 1),
                           time_and_batch_graph_us=round(time_graph(ft, 10, args.iters_fast) * 1e3, 1))
            elif wl == "chain":
                ms = time_eager(chain, 1, args.iters)
                rec = dict(workload="chain", rep=rep, chain_ms=round(ms, 2))
            else:
                raise SystemExit(f"unknown workload {wl}")
            assert _lib.device_status() == 0
            runs.append(rec)
            print(json.dumps({**rec, "gpu": name, "power_limit_w": plim}), flush=True)
        med = {k: statistics.median(r[k] for r in runs) for k in runs[0] if k not in ("workload", "rep")}
        print(json.dumps({"workload": runs[0]["workload"], "summary": "median of reps", "reps": args.reps, **med, **base}),
              flush=True)


if __name__ == "__main__":
    main()
