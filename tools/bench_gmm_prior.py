#!/usr/bin/env python
"""Step-time cost of the Gaussian-mixture prior on the bench.py --config 2 shape: 2 flows, B = 32, T <= 1000 (LJS-like lengths),
attention prior + CTC, flowtron_b200.RAdam + clip_grad_norm_(1.0), for n_components 0, 8 fixed and 8 learned, eager and
replayed from one CUDA graph.  Also times the mel encoder's forward and backward alone (CUDA events) and reports how much of
them the side stream hides: hidden = 1 - (step(K) - step(0)) / (mel-encoder fwd + bwd).

    python tools/bench_gmm_prior.py [--steps 10] [--warmup 3] [--out results/bench_gmm_prior.json]
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


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
        return r.stdout.strip()
    except OSError:
        return torch.cuda.get_device_name()


def median(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2]


def run_case(K, fixed, args):
    from flowtron_b200 import synth
    from flowtron_b200.flowtron import Flowtron, FlowtronLoss
    from flowtron_b200.radam import RAdam
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=2, n_components=K, fixed_gaussian=fixed, mean_scale=3.0 if fixed else 0.0)
    params = synth.synth_gmm_params(cfg, 1234) if K > 1 else synth.synth_params(cfg, 1234)
    model = Flowtron(**cfg)
    model.load_state_dict(params, strict=True)
    model = model.cuda().train()
    out_lens, in_lens = synth.ljs_like_lengths(32, 1000, 1234)
    b = synth.synth_batch(32, 1000, int(in_lens.max()), cfg, 1234, out_lens=out_lens.tolist(), in_lens=in_lens.tolist(),
                          with_prior=True, logmel_stats=True)
    d = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in b.items()}
    crit = FlowtronLoss(sigma=1.0, gm_loss=K > 1, gate_loss=True, use_ctc_loss=True, ctc_loss_weight=1.0)
    opt = RAdam(model.parameters(), lr=1e-4, weight_decay=1e-6, capturable=True)

    def body():
        opt.zero_grad()
        out = model(d["mel"], d["speaker_ids"], d["text"], d["in_lens"], d["out_lens"], d["attn_prior"])
        nll, gl, ctc = crit(out, d["gate_target"], d["in_lens"], d["out_lens"])
        (nll + gl + ctc).sum().backward()
        opt.clip_grad_norm_(1.0)
        opt.step()

    def timed(fn, n):
        ts = []
        for _ in range(n):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        return ts

    for _ in range(args.warmup):
        body()
    torch.cuda.synchronize()
    eager = timed(body, args.steps)
    graph = torch.cuda.CUDAGraph()
    opt.zero_grad()
    torch.cuda.synchronize()
    with torch.cuda.graph(graph):
        body()
    graph.replay()
    torch.cuda.synchronize()
    replay = timed(graph.replay, args.steps)
    rec = dict(n_components=K, fixed_gaussian=fixed if K > 1 else None, eager_ms=median(eager), graph_ms=median(replay),
               eager_all=eager, graph_all=replay)
    if K > 1:
        enc = model.mel_encoder
        mel, lens = d["mel"], d["out_lens"]

        def fwd():
            return enc(mel, lens)
        for _ in range(2):
            fwd().sum().backward()
        torch.cuda.synchronize()
        rec["mel_encoder_fwd_ms"] = median(timed(fwd, args.steps))
        embs = [fwd() for _ in range(args.steps)]
        torch.cuda.synchronize()
        it = iter(embs)
        rec["mel_encoder_bwd_ms"] = median(timed(lambda: next(it).sum().backward(), args.steps))
    del graph, opt, model
    torch.cuda.empty_cache()
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark needs a GPU"
    res = dict(gpu=gpu_info(), shape="bench.py --config 2: 2 flows, B=32, T<=1000, prior + CTC, RAdam + clip", cases=[])
    for K, fixed in ((0, True), (8, True), (8, False)):
        res["cases"].append(run_case(K, fixed, args))
    base = res["cases"][0]
    for c in res["cases"][1:]:
        enc = c["mel_encoder_fwd_ms"] + c["mel_encoder_bwd_ms"]
        for mode in ("eager", "graph"):
            extra = c[f"{mode}_ms"] - base[f"{mode}_ms"]
            c[f"{mode}_extra_ms"] = extra
            c[f"{mode}_hidden_fraction"] = 1.0 - extra / enc
    for c in res["cases"]:
        print({k: (round(v, 3) if isinstance(v, float) else v) for k, v in c.items() if not k.endswith("_all")})
    print(json.dumps(dict(gpu=res["gpu"])))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
