#!/usr/bin/env python
"""Time Flowtron.infer_batch (ragged-batch inference) against sequential B = 1 Flowtron.infer calls on the GPU; one JSON
line per workload and repetition, then one summary line per workload.

Workloads (fixed seed; 2-flow model at the shipped sizes; gate bias -10 so the gate never fires and the work is fixed):
  W1  16 texts with in_lens drawn from U{40..160}, frame budgets round(6.5 in_len) clipped to [150, 1000].
      infer_batch eager and CUDA-graph replayed, against 16 sequential B = 1 infer calls on the unpadded rows.
      Reported: ms per batch, valid mel frames per second, the speed-up, and the largest per-row difference from the B = 1
      runs (checked against the 2e-3 bound of the tests).
  W2  W1's batch, then WaveGlow.infer(lengths=) and the Denoiser (strength 0.1), against 16 sequential B = 1 chains.
      Reported: ms per batch and seconds of 22050 Hz audio per wall-clock second.
  W2G W2 as a serving loop: infer_batch -> WaveGlow.infer(lengths=mel_lens) -> Denoiser(lengths=256 mel_lens) captured
      ONCE as one CUDA graph on static buffers (B = 16, T = 1000, L = 160, CUDA lengths), then replayed on fresh
      residuals, texts, noise and length sets (in_lens U{40..160}, budgets as W1's), each copied into the buffers from
      device memory before its replay.  The first request is checked bit for bit against eager calls with host lengths.
      Reported beside eager W2 (which reads mel_lens on the host): ms per request and audio seconds per second.

Times come from CUDA events around work that ends in a device synchronise, after warming up every shape; each workload
is repeated --reps times, alternating batched and sequential.  The card name and power limit are read in the same run.
Needs a GPU; there is no CPU path.
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
from flowtron_b200.waveglow import WaveGlow  # noqa: E402

SR, HOP = 22050, 256


def w1_batch(dev, B=16, seed=2026):
    g = torch.Generator().manual_seed(seed)
    in_lens = torch.randint(40, 161, (B,), generator=g)
    budgets = torch.clamp(torch.round(6.5 * in_lens.double()).long(), 150, 1000)
    T, L = int(budgets.max()), int(in_lens.max())
    res = (torch.randn(B, 80, T, generator=g) * 0.5).to(dev)
    text = torch.randint(0, 185, (B, L), generator=g).to(dev)
    spk = torch.zeros(B, dtype=torch.long, device=dev)
    return res, spk, text, in_lens.tolist(), budgets.tolist()


def serving_graph(model, wg, den, dev, B, T=1000, L=160, n_requests=4, seed=77):
    """Captures the text-to-audio chain once on static buffers with CUDA lengths; returns run(iters) -> (ms per request,
    mean audio seconds per request), which replays it over the requests round-robin."""
    g = torch.Generator().manual_seed(seed)
    reqs = []
    for _ in range(n_requests):
        in_lens = torch.randint(40, L + 1, (B,), generator=g)
        budgets = torch.clamp(torch.round(6.5 * in_lens.double()).long(), 150, T)
        reqs.append(dict(res=(torch.randn(B, 80, T, generator=g) * 0.5).to(dev), text=torch.randint(0, 185, (B, L), generator=g).to(dev),
                         in_lens=in_lens.to(dev), budgets=budgets.to(dev), noise=torch.randn(B, 8, 32 * T, generator=g).to(dev),
                         frames=int(budgets.sum())))
    buf = {k: torch.empty_like(v) for k, v in reqs[0].items() if torch.is_tensor(v)}
    spk = torch.zeros(B, dtype=torch.long, device=dev)

    def load(r):
        for k, v in buf.items():
            v.copy_(r[k])

    def chain():
        mel, mel_lens, _ = model.infer_batch(buf["res"], spk, buf["text"], buf["in_lens"], max_frames=buf["budgets"])
        audio = wg.infer(mel, sigma=0.6, noise=buf["noise"], lengths=mel_lens)
        return mel_lens, audio, den(audio, 0.1, lengths=HOP * mel_lens)

    load(reqs[0])
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            chain()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        outs = chain()
    # the first request against eager calls with host lengths, bit for bit
    load(reqs[1])
    graph.replay()
    torch.cuda.synchronize()
    r = reqs[1]
    mel_e, lens_e, _ = model.infer_batch(r["res"], spk, r["text"], r["in_lens"].tolist(), max_frames=r["budgets"].tolist())
    n = lens_e.tolist()
    audio_e = wg.infer(mel_e, sigma=0.6, noise=r["noise"], lengths=n)
    clean_e = den(audio_e, 0.1, lengths=[HOP * f for f in n])
    assert torch.equal(outs[0], lens_e) and torch.equal(outs[1], audio_e) and torch.equal(outs[2], clean_e)
    assert _lib.device_status() == 0

    def run(iters):
        for r in reqs:                                            # warm-up over every request
            load(r)
            graph.replay()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for i in range(iters):
            load(reqs[i % n_requests])
            graph.replay()
        b.record()
        torch.cuda.synchronize()
        frames = sum(reqs[i % n_requests]["frames"] for i in range(iters)) / iters
        return a.elapsed_time(b) / iters, HOP * frames / SR

    run.static = (spk, s, outs)                                   # the graph reads and writes these: keep them alive
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--workloads", default="W1,W2,W2G")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_infer_batch.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    name, plim = card()
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=2)
    p = synth.synth_params(cfg, 1234)
    key = [k for k in p if k.endswith("gate_layer.linear_layer.bias")][0]
    p[key] = torch.full_like(p[key], -10.0)
    model = Flowtron(**cfg)
    model.load_state_dict(p, strict=True)
    model = model.to(dev).eval()
    res, spk, text, in_lens, budgets = w1_batch(dev)
    B = len(in_lens)
    in_lens_d = torch.tensor(in_lens, device=dev)
    budgets_d = torch.tensor(budgets, device=dev)

    def batched():
        return model.infer_batch(res, spk, text, in_lens_d, max_frames=budgets_d)

    def sequential():
        return [model.infer(res[b:b + 1, :, :budgets[b]], spk[b:b + 1], text[b:b + 1, :in_lens[b]])[0] for b in range(B)]

    torch.set_grad_enabled(False)
    # outputs: every row against its B = 1 run, at the timed sizes
    mel, mel_lens, _ = batched()
    singles = sequential()
    lens = mel_lens.tolist()
    assert lens == [s.shape[-1] for s in singles] == budgets, (lens, budgets)
    row_err = max((mel[b, :, :n] - s[0]).abs().max().item() / s.abs().max().item() for b, (n, s) in enumerate(zip(lens, singles)))
    assert row_err <= 2e-3, row_err
    assert _lib.device_status() == 0
    frames = sum(budgets)
    base = dict(B=B, in_lens=in_lens, max_frames=budgets, T=res.shape[-1], L=text.shape[1], valid_frames=frames, gpu=name,
                power_limit_w=plim)

    wg = den = None
    if "W2" in args.workloads:                               # W2 and W2G
        wcfg = synth.DEFAULT_WAVEGLOW_CONFIG
        wg = WaveGlow(**wcfg)
        wg.load_state_dict(synth.synth_waveglow_params(wcfg, 1234), strict=True)
        wg = wg.to(dev).eval()
        den = Denoiser(wg)

    def chain_batched():
        m, ml, _ = batched()
        n = ml.tolist()
        audio = wg.infer(m.contiguous(), sigma=0.6, lengths=n)
        return den(audio, 0.1, lengths=[HOP * f for f in n])

    def chain_sequential():
        out = []
        for b in range(B):
            m1, _ = model.infer(res[b:b + 1, :, :budgets[b]], spk[b:b + 1], text[b:b + 1, :in_lens[b]])
            out.append(den(wg.infer(m1.contiguous(), sigma=0.6), 0.1))
        return out

    serve = serving_graph(model, wg, den, dev, B) if "W2G" in args.workloads.split(",") else None

    for wl in args.workloads.split(","):
        runs = []
        for rep in range(args.reps):
            if wl == "W1":
                eager = time_eager(batched, 1, args.iters)
                graph = time_graph(batched, 1, args.iters)
                seq = time_eager(sequential, 1, 1)
                rec = dict(workload="W1_infer_batch", rep=rep, batched_eager_ms=round(eager, 2), batched_graph_ms=round(graph, 2),
                           sequential_b1_ms=round(seq, 2), frames_per_s_eager=round(frames / (eager / 1e3)),
                           frames_per_s_graph=round(frames / (graph / 1e3)), frames_per_s_sequential=round(frames / (seq / 1e3)),
                           speedup_eager=round(seq / eager, 2), speedup_graph=round(seq / graph, 2), max_row_rel_err=row_err)
            elif wl == "W2":
                bat = time_eager(chain_batched, 1, args.iters)
                seq = time_eager(chain_sequential, 1, 1)
                audio_s = HOP * frames / SR
                rec = dict(workload="W2_text_to_audio", rep=rep, batched_ms=round(bat, 2), sequential_b1_ms=round(seq, 2),
                           audio_s=round(audio_s, 2), audio_s_per_s_batched=round(audio_s / (bat / 1e3), 1),
                           audio_s_per_s_sequential=round(audio_s / (seq / 1e3), 1), speedup=round(seq / bat, 2))
            elif wl == "W2G":
                bat = time_eager(chain_batched, 1, args.iters)
                graph_ms, audio_s = serve(args.iters)
                rec = dict(workload="W2G_text_to_audio_graph", rep=rep, graph_ms_per_request=round(graph_ms, 2),
                           eager_w2_ms=round(bat, 2), audio_s_per_request=round(audio_s, 2),
                           audio_s_per_s_graph=round(audio_s / (graph_ms / 1e3), 1),
                           audio_s_per_s_eager_w2=round(HOP * frames / SR / (bat / 1e3), 1))
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
