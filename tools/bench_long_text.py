#!/usr/bin/env python
"""Time long texts on the GPU: a training step (Flowtron.forward + FlowtronLoss with the prior and CTC + backward) at
B = 8, T = 1000 and Flowtron.infer at B = 1 for 1000 frames (gate off), at L = 256, 512 and 1024 tokens.  Each shape is
warmed up, then timed three times with CUDA events; the card's name and power limit are recorded with the numbers.

    python tools/bench_long_text.py [--lens 256 512 1024] [--reps 3] [--out result.json]
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
from flowtron_b200 import _lib, synth  # noqa: E402
from flowtron_b200.flowtron import Flowtron, FlowtronLoss  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else torch.cuda.get_device_name()


def timed(fn, reps):
    fn()                                             # warm-up: module loads, workspace allocation
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lens", type=int, nargs="+", default=[256, 512, 1024])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_long_text needs a GPU")
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=2)
    model = Flowtron(**cfg)
    model.load_state_dict(synth.synth_params(cfg, 1), strict=True)
    model = model.cuda()
    crit = FlowtronLoss(sigma=1.0, gate_loss=True, use_ctc_loss=True, ctc_loss_weight=1.0)
    rec = {"card": card(), "train": {}, "infer": {}}
    B, T, Ti = 8, 1000, 1000
    for L in args.lens:
        batch = synth.synth_batch(B, T, L, cfg, 2, with_prior=True)
        cu = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in batch.items()}
        model.train()

        def step():
            model.zero_grad(set_to_none=True)
            out = model(cu["mel"], cu["speaker_ids"], cu["text"], cu["in_lens"], cu["out_lens"], cu["attn_prior"])
            nll, gl, ctc = crit(out, cu["gate_target"], cu["in_lens"], cu["out_lens"])
            (nll + gl + ctc).sum().backward()
        ms = timed(step, args.reps)
        rec["train"][L] = {"B": B, "T": T, "ms": ms, "frames_per_s": B * T / (min(ms) / 1e3)}
        model.eval()
        g = torch.Generator().manual_seed(L)
        res = (torch.randn(1, 80, Ti, generator=g) * 0.5).cuda()
        text = torch.randint(0, cfg["n_text"], (1, L), generator=g).cuda()
        spk = torch.zeros(1, dtype=torch.long, device="cuda")

        def infer():
            with torch.no_grad():
                model.infer(res, spk, text, gate_threshold=1.1)      # sigmoid <= 1: every frame is generated
        ms = timed(infer, args.reps)
        rec["infer"][L] = {"B": 1, "frames": Ti, "ms": ms, "frames_per_s": Ti / (min(ms) / 1e3)}
        assert _lib.device_status() == 0
        print(json.dumps({"L": L, "train_ms": rec["train"][L]["ms"], "infer_ms": rec["infer"][L]["ms"]}), flush=True)
    print(json.dumps(rec))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
