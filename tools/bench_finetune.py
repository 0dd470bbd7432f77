#!/usr/bin/env python
"""Time one Flowtron fine-tuning step per set of trainable parameters, at the configs[1] training shape of bench.py
(2 flows, batch 32, T <= 1000 with LJSpeech-like lengths from a fixed seed, attention prior and gate on).

A step is forward + FlowtronLoss + backward + clip_grad_norm + the fused capturable RAdam on the trainable parameters,
replayed from one CUDA graph.  Variants:
  full     every parameter (what bench.py times)
  speaker  speaker_embedding.weight only (few-shot speaker adaptation)
  gate     the last flow's gate layer only (retraining the gate)
  flow1    every parameter of flows.1
The flow-step backward runs only what the trainable parameters need (ft_ar_step_bwd_plan), so the frozen variants skip
recurrences and weight-gradient GEMMs.

One JSON line per variant and round: ms per step (CUDA events over --steps replays after --warmup), ft launches per step
(_lib.launch_count over one eager step: the counter counts at enqueue, so a replay adds nothing), the peak allocated
memory of that eager step above what was resident before it (model, optimizer state, inputs), and the card name and
power limit, read in the same run.  The variants alternate within each round.  Needs a GPU; there is no CPU path.
"""
from __future__ import annotations

import argparse
import gc
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from flowtron_b200 import _lib, synth  # noqa: E402
from flowtron_b200.flowtron import Flowtron, FlowtronLoss  # noqa: E402
from flowtron_b200.radam import RAdam  # noqa: E402

VARIANTS = ("full", "speaker", "gate", "flow1")


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        name, plim = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
        return name, float(plim)
    except Exception:                                            # noqa: BLE001 -- reported as unknown, never guessed
        return torch.cuda.get_device_name(0), None


def train_lengths(B, T, seed):
    """bench.py's configs[1] lengths: out_lens ~ U{T/2..T} with the max forced to T, in_lens = round(out / 6.5) in [40, 160]."""
    g = torch.Generator().manual_seed(seed)
    out_lens = torch.randint(T // 2, T + 1, (B,), generator=g)
    out_lens[0] = T
    in_lens = torch.clamp((out_lens.float() / 6.5).round().long(), 40, 160)
    return out_lens, in_lens


def trainable(names, variant):
    if variant == "full":
        return set(names)
    if variant == "speaker":
        return {"speaker_embedding.weight"}
    if variant == "gate":
        return {n for n in names if "gate_layer" in n}
    return {n for n in names if n.startswith("flows.1.")}


def run_variant(variant, model, state, static, crit, args):
    model.load_state_dict(state, strict=True)
    names = [n for n, _ in model.named_parameters()]
    train = trainable(names, variant)
    for n, p in model.named_parameters():
        p.requires_grad_(n in train)
        p.grad = None
    opt = RAdam([p for p in model.parameters() if p.requires_grad], lr=1e-3, weight_decay=1e-6, capturable=True)

    def step():
        opt.zero_grad()
        out = model(static["mel"], static["speaker_ids"], static["text"], static["in_lens"], static["out_lens"],
                    static["attn_prior"])
        nll, gl, _ = crit(out, static["gate_target"], static["in_lens"], static["out_lens"])
        (nll + gl).sum().backward()
        opt.clip_grad_norm_(1.0)
        opt.step()

    for _ in range(2):
        step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    resident = torch.cuda.memory_allocated()
    _lib.reset_launch_count()
    step()
    torch.cuda.synchronize()
    launches = _lib.launch_count()
    peak = torch.cuda.max_memory_allocated() - resident
    graph = torch.cuda.CUDAGraph()
    opt.zero_grad()
    torch.cuda.synchronize()
    with torch.cuda.graph(graph):
        step()
    torch.cuda.synchronize()
    for _ in range(args.warmup):
        graph.replay()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(args.steps):
        graph.replay()
    t1.record()
    torch.cuda.synchronize()
    assert _lib.device_status() == 0, "device watchdog tripped"
    ms = t0.elapsed_time(t1) / args.steps
    n_train = sum(p.numel() for p in model.parameters() if p.requires_grad)
    del graph, opt
    gc.collect()
    torch.cuda.empty_cache()
    return {"variant": variant, "ms_per_step": round(ms, 3), "ft_launches_per_step": int(launches),
            "step_peak_allocated_gib": round(peak / 2**30, 3), "trainable_params": int(n_train)}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--variants", default=",".join(VARIANTS))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_finetune needs a GPU")
    variants = args.variants.split(",")
    assert all(v in VARIANTS for v in variants), variants
    name, plim = card()
    dev = torch.device("cuda", 0)
    cfg = dict(synth.DEFAULT_MODEL_CONFIG)
    B, T = 32, 1000
    state = synth.synth_params(cfg, 1234)
    model = Flowtron(**cfg)
    model.load_state_dict(state, strict=True)
    model = model.to(dev).train()
    crit = FlowtronLoss(sigma=1.0, gate_loss=True, use_ctc_loss=False)
    out_lens, in_lens = train_lengths(B, T, 1234)
    L = int(in_lens.max())
    batch = synth.synth_batch(B, T, L, cfg, 1234, out_lens=out_lens.tolist(), in_lens=in_lens.tolist(), with_prior=True,
                              logmel_stats=True)
    static = {k: batch[k].to(dev) for k in ("mel", "speaker_ids", "text", "in_lens", "out_lens", "gate_target", "attn_prior")}
    for r in range(args.rounds):
        order = variants if r % 2 == 0 else variants[::-1]
        for v in order:
            rec = run_variant(v, model, state, static, crit, args)
            print(json.dumps({**rec, "round": r, "batch": B, "max_frames": T, "max_text": L, "gpu": name,
                              "power_limit_w": plim}), flush=True)


if __name__ == "__main__":
    main()
