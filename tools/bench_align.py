#!/usr/bin/env python
"""Time hard alignment (align.mas, Flowtron.align) and duration-controlled synthesis (Flowtron.infer_durations) against
what users run without them; one JSON line per repetition, then one summary line per workload.

Workloads (fixed seeds):
  M1  mas on 32 rows with T ~ U{150..1000} frames and L ~ U{40..160} tokens (attention-like log-probabilities, CUDA
      lengths), eager and replayed from a CUDA graph, against the float32 numpy restatement (oracle/align_oracle.py) run on
      the host one row at a time -- the per-utterance CPU search users run today, here without a numba JIT.
  M2  the same on 8 rows of T = 3000 and L = 1024.
  A1  Flowtron.align (2 flows, shipped sizes) on 16 utterances of U{150..860} frames with in_lens = round(frames / 6.5),
      host and CUDA lengths, against 16 B = 1 align calls.
  D1  Flowtron.infer_durations with A1's durations against Flowtron.infer_batch on the same batch (gate threshold 1: both
      generate every frame).
Every GPU result is checked first (M: identical to the oracle; A: every row equal to its B = 1 call).  Times come from
CUDA events around work that ends in a device synchronise (host clock for the oracle), after a warm-up of every shape;
each workload is repeated --reps times.  The card name and power limit are read in the same run.  Needs a GPU.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_waveglow import card, time_eager, time_graph  # noqa: E402
from flowtron_b200 import _lib, align, synth  # noqa: E402
from flowtron_b200.flowtron import Flowtron  # noqa: E402
from oracle import align_oracle  # noqa: E402


def mas_rows(B, t_range, l_range, seed):
    g = torch.Generator().manual_seed(seed)
    in_lens = torch.randint(l_range[0], l_range[1] + 1, (B,), generator=g)
    out_lens = torch.stack([torch.randint(max(t_range[0], int(n)), t_range[1] + 1, (1,), generator=g)[0] for n in in_lens])
    T, L = int(out_lens.max()), int(in_lens.max())
    lp = torch.log_softmax(3.0 * torch.randn(B, T, L, generator=g), -1)
    return lp, in_lens.tolist(), out_lens.tolist()


def mas_workload(lp_host, in_lens, out_lens, dev, iters):
    lp = lp_host.to(dev)
    il, ol = torch.tensor(in_lens, device=dev), torch.tensor(out_lens, device=dev)
    d, tok = align.mas(lp, il, ol)
    ref_d, ref_t = align_oracle.mas(lp_host.numpy(), in_lens, out_lens)
    differing = int(sum(not (np.array_equal(d[b].cpu().numpy(), ref_d[b]) and np.array_equal(tok[b].cpu().numpy(), ref_t[b]))
                        for b in range(len(in_lens))))
    assert differing == 0, differing
    eager = time_eager(lambda: align.mas(lp, il, ol), 2, iters)
    graph = time_graph(lambda: align.mas(lp, il, ol), 2, iters)
    lp_np = lp_host.numpy()
    t0 = time.perf_counter()
    for b, (nl, nt) in enumerate(zip(in_lens, out_lens)):
        align_oracle.mas(lp_np[b:b + 1, :nt, :nl], [nl], [nt])
    cpu = (time.perf_counter() - t0) * 1e3
    return dict(mas_eager_ms=round(eager, 4), mas_graph_ms=round(graph, 4), oracle_cpu_ms=round(cpu, 1),
                speedup_graph_vs_cpu=round(cpu / graph, 1), rows_differing=differing)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--workloads", default="M1,M2,A1,D1")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_align.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    name, plim = card()
    torch.set_grad_enabled(False)

    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=2, n_speakers=2)
    p = synth.synth_params(cfg, 1234)
    key = [k for k in p if k.endswith("gate_layer.linear_layer.bias")][0]
    p[key] = torch.full_like(p[key], -10.0)
    model = Flowtron(**cfg)
    model.load_state_dict(p, strict=True)
    model = model.to(dev).eval()
    g = torch.Generator().manual_seed(2026)
    B = 16
    out_lens = torch.randint(150, 861, (B,), generator=g)
    in_lens = torch.round(out_lens.double() / 6.5).long()
    T, L = int(out_lens.max()), int(in_lens.max())
    mel = (torch.randn(B, 80, T, generator=g) * 2.0 - 5.5).clamp_(-11.5, 2.0).to(dev)
    text = torch.randint(0, 185, (B, L), generator=g).to(dev)
    spk = torch.randint(0, 2, (B,), generator=g).to(dev)
    residual = (torch.randn(B, 80, T, generator=g) * 0.5).to(dev)
    in_lens, out_lens = in_lens.tolist(), out_lens.tolist()
    in_d, out_d = torch.tensor(in_lens, device=dev), torch.tensor(out_lens, device=dev)

    def align_host():
        return model.align(mel, spk, text, in_lens, out_lens)

    def align_cuda():
        return model.align(mel, spk, text, in_d, out_d)

    def align_loop():
        return [model.align(mel[b:b + 1, :, :n], spk[b:b + 1], text[b:b + 1, :nl], [nl], [n])
                for b, (nl, n) in enumerate(zip(in_lens, out_lens))]

    durations, _ = align_host()
    for b, (d1, _) in enumerate(align_loop()):
        assert torch.equal(d1[0], durations[b, :in_lens[b]]), b
    assert durations.sum(1).tolist() == out_lens

    def by_durations():
        return model.infer_durations(residual, spk, text, in_d, durations)

    def by_scores():
        return model.infer_batch(residual, spk, text, in_d, gate_threshold=1.0, max_frames=out_d)

    assert by_durations()[1].tolist() == out_lens
    assert _lib.device_status() == 0
    m1 = mas_rows(32, (150, 1000), (40, 160), 11)
    m2 = mas_rows(8, (3000, 3000), (1024, 1024), 12)

    for wl in args.workloads.split(","):
        runs = []
        for rep in range(args.reps):
            if wl in ("M1", "M2"):
                lp, il, ol = m1 if wl == "M1" else m2
                rec = dict(workload=f"{wl}_mas", rep=rep, **mas_workload(lp, il, ol, dev, args.iters))
                base = dict(B=len(il), frames=sum(ol), T=lp.shape[1], L=lp.shape[2])
            elif wl == "A1":
                host = time_eager(align_host, 1, 3)
                cuda = time_eager(align_cuda, 1, 3)
                loop = time_eager(align_loop, 1, 1)
                rec = dict(workload="A1_flowtron_align", rep=rep, align_host_lens_ms=round(host, 2),
                           align_cuda_lens_ms=round(cuda, 2), loop_b1_ms=round(loop, 2), speedup_host_lens=round(loop / host, 2))
                base = dict(B=B, frames=sum(out_lens), T=T, L=L)
            elif wl == "D1":
                dur = time_eager(by_durations, 1, 3)
                sc = time_eager(by_scores, 1, 3)
                rec = dict(workload="D1_infer_durations_vs_infer_batch", rep=rep, infer_durations_ms=round(dur, 2),
                           infer_batch_ms=round(sc, 2), ratio=round(sc / dur, 3))
                base = dict(B=B, frames=sum(out_lens), T=T, L=L)
            else:
                raise SystemExit(f"unknown workload {wl}")
            assert _lib.device_status() == 0
            runs.append(rec)
            print(json.dumps({**rec, "gpu": name, "power_limit_w": plim}), flush=True)
        med = {k: statistics.median(r[k] for r in runs) for k in runs[0] if k not in ("workload", "rep")}
        print(json.dumps({"workload": runs[0]["workload"], "summary": "median of reps", "reps": args.reps, **med, **base,
                          "gpu": name, "power_limit_w": plim}), flush=True)


if __name__ == "__main__":
    main()
