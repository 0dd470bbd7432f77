#!/usr/bin/env python
"""Time batched voice conversion (Flowtron.convert) against the per-utterance loop it replaces, and forced-alignment
inference (Flowtron.infer_aligned) against Flowtron.infer_batch on the same batch; one JSON line per repetition, then one
summary line per workload.

Workload (fixed seed; 2-flow, 2-speaker model at the shipped sizes; gate bias -10 so the gate never fires): 16 recorded
utterances of U{150..860} frames with in_lens = round(frames / 6.5), every row converted to the other speaker.
  C1  convert with host length lists (rows under and from 320 frames run as two encode launches, every row bit-equal to its
      B = 1 encode) and with CUDA length tensors (one launch, no host synchronisation), against 16 x
      (B = 1 forward + B = 1 infer(attns=)).  Reported: ms per batch, valid mel frames per second, the speed-up and the
      largest per-row difference from the loop (checked against the 2e-3 bound of the tests).
  C2  infer_aligned against infer_batch (gate threshold 1: both generate every frame) on the z and alignments of C1: what
      skipping the query / score / softmax phase is worth.

Times come from CUDA events around work that ends in a device synchronise, after warming up every shape; each workload
is repeated --reps times, alternating the arms.  The card name and power limit are read in the same run.  Needs a GPU;
there is no CPU path.
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

from bench_waveglow import card, time_eager  # noqa: E402
from flowtron_b200 import _lib, synth  # noqa: E402
from flowtron_b200.flowtron import Flowtron  # noqa: E402


def batch(dev, B=16, seed=2026):
    g = torch.Generator().manual_seed(seed)
    out_lens = torch.randint(150, 861, (B,), generator=g)
    in_lens = torch.round(out_lens.double() / 6.5).long()
    T, L = int(out_lens.max()), int(in_lens.max())
    mel = (torch.randn(B, 80, T, generator=g) * 2.0 - 5.5).clamp_(-11.5, 2.0).to(dev)
    text = torch.randint(0, 185, (B, L), generator=g).to(dev)
    spk = torch.randint(0, 2, (B,), generator=g).to(dev)
    return mel, spk, 1 - spk, text, in_lens.tolist(), out_lens.tolist()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--workloads", default="C1,C2")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_convert.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    name, plim = card()
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=2, n_speakers=2)
    p = synth.synth_params(cfg, 1234)
    key = [k for k in p if k.endswith("gate_layer.linear_layer.bias")][0]
    p[key] = torch.full_like(p[key], -10.0)
    model = Flowtron(**cfg)
    model.load_state_dict(p, strict=True)
    model = model.to(dev).eval()
    mel, spk, tgt, text, in_lens, out_lens = batch(dev)
    B = len(in_lens)
    in_lens_d, out_lens_d = torch.tensor(in_lens, device=dev), torch.tensor(out_lens, device=dev)

    def convert_host():
        return model.convert(mel, spk, tgt, text, in_lens, out_lens)

    def convert_cuda():
        return model.convert(mel, spk, tgt, text, in_lens_d, out_lens_d)

    def loop():
        outs = []
        for b in range(B):
            nl, nt = in_lens[b], out_lens[b]
            txt = text[b:b + 1, :nl]
            o = model(mel[b:b + 1, :, :nt].contiguous(), spk[b:b + 1], txt, in_lens_d[b:b + 1], out_lens_d[b:b + 1])
            outs.append(model.infer(o[0].permute(1, 2, 0), tgt[b:b + 1], txt, gate_threshold=1.0, attns=[a[0] for a in o[3]])[0])
        return outs

    torch.set_grad_enabled(False)
    # outputs: every row against the loop, at the timed sizes
    singles = loop()
    assert [s.shape[-1] for s in singles] == out_lens
    errs = {}
    for tag, fn in (("host", convert_host), ("cuda", convert_cuda)):
        out = fn()
        errs[tag] = max((out[b, :, :n] - s[0]).abs().max().item() / s.abs().max().item()
                        for b, (n, s) in enumerate(zip(out_lens, singles)))
        assert errs[tag] <= 2e-3, errs
    z, attns = model.encode(mel, spk, text, in_lens, out_lens, return_attns=True)
    z = z.contiguous()
    assert _lib.device_status() == 0
    frames = sum(out_lens)
    base = dict(B=B, in_lens=in_lens, out_lens=out_lens, T=mel.shape[-1], L=text.shape[1], valid_frames=frames, gpu=name,
                power_limit_w=plim)

    def aligned():
        return model.infer_aligned(z, tgt, text, in_lens_d, attns, out_lens_d)

    def scored():
        return model.infer_batch(z, tgt, text, in_lens_d, gate_threshold=1.0, max_frames=out_lens_d)

    for wl in args.workloads.split(","):
        runs = []
        for rep in range(args.reps):
            if wl == "C1":
                host = time_eager(convert_host, 1, args.iters)
                cuda = time_eager(convert_cuda, 1, args.iters)
                seq = time_eager(loop, 1, 1)
                rec = dict(workload="C1_convert", rep=rep, convert_host_lens_ms=round(host, 2), convert_cuda_lens_ms=round(cuda, 2),
                           loop_b1_ms=round(seq, 2), frames_per_s_host_lens=round(frames / (host / 1e3)),
                           frames_per_s_cuda_lens=round(frames / (cuda / 1e3)), frames_per_s_loop=round(frames / (seq / 1e3)),
                           speedup_host_lens=round(seq / host, 2), speedup_cuda_lens=round(seq / cuda, 2),
                           max_row_rel_err_host_lens=errs["host"], max_row_rel_err_cuda_lens=errs["cuda"])
            elif wl == "C2":
                al = time_eager(aligned, 1, args.iters)
                sc = time_eager(scored, 1, args.iters)
                rec = dict(workload="C2_infer_aligned_vs_infer_batch", rep=rep, infer_aligned_ms=round(al, 2),
                           infer_batch_ms=round(sc, 2), ratio=round(sc / al, 3))
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
