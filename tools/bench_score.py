#!/usr/bin/env python
"""Time Flowtron.score, the per-utterance NLL / gate / attention-CTC losses of a padded batch, against the loop it replaces:
one B = 1 ``forward`` + ``FlowtronLoss`` (gate and CTC on) + ``.item()`` per utterance, on this library's kernels.

Workload: 2 flows with gate, attention prior and CTC, B utterances (default 32 and 128) of U{150..860} frames and
U{40..160} tokens from a fixed seed, synthetic weights.  Arms, alternated within each round:
  score_host   score() with host lengths (rows split around the attention-overlap threshold, as B = 1 calls run them)
  score_cuda   score() with CUDA length tensors, eager (one launch group, no host synchronisation)
  score_graph  the score_cuda call captured once as a CUDA graph and replayed
  loop_b1      the B = 1 loop (host synchronisation per utterance)
Each arm's time is the wall clock around --reps calls ending in a device synchronise, after one warm-up call.  The loop's
rows are compared with score_host's (largest relative difference of nll, gate and the mean CTC cost over the flows).
One JSON line per arm, batch size and round, with the card name and power limit read in the same run.  Needs a GPU.
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

from flowtron_b200 import _lib, synth  # noqa: E402
from flowtron_b200.flowtron import Flowtron, FlowtronLoss  # noqa: E402

ARMS = ("score_host", "score_cuda", "score_graph", "loop_b1")


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        name, plim = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
        return name, float(plim)
    except Exception:                                            # noqa: BLE001 -- reported as unknown, never guessed
        return torch.cuda.get_device_name(0), None


def make_batch(B, seed):
    g = torch.Generator().manual_seed(seed)
    out_lens = torch.randint(150, 861, (B,), generator=g)
    in_lens = torch.randint(40, 161, (B,), generator=g)
    T, L = int(out_lens.max()), int(in_lens.max())
    b = synth.synth_batch(B, T, L, synth.DEFAULT_MODEL_CONFIG, seed, out_lens=out_lens, in_lens=in_lens, with_prior=True,
                          logmel_stats=True)
    return {k: v.cuda() for k, v in b.items()}


def loop_b1(model, crit, b):
    """The per-utterance loop score replaces: rows of (nll, gate_loss, loss_ctc) as Python floats."""
    rows = []
    with torch.no_grad():
        for i, (nl, n) in enumerate(zip(b["in_lens"].tolist(), b["out_lens"].tolist())):
            il, ol = b["in_lens"][i:i + 1], b["out_lens"][i:i + 1]
            out = model(b["mel"][i:i + 1, :, :n], b["speaker_ids"][i:i + 1], b["text"][i:i + 1, :nl], il, ol,
                        b["attn_prior"][i:i + 1, :n, :nl])
            nll, gl, ctc = crit(out, b["gate_target"][i:i + 1, :n], il, ol)
            rows.append((nll.item(), gl.item(), ctc.item()))
    return rows


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / reps


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--batches", default="32,128")
    ap.add_argument("--reps", type=int, default=5, help="timed calls per score arm")
    ap.add_argument("--loop-reps", type=int, default=1, help="timed passes of the B = 1 loop")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--arms", default=",".join(ARMS))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_score needs a GPU")
    arms = args.arms.split(",")
    assert all(a in ARMS for a in arms), arms
    name, plim = card()
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=2)
    model = Flowtron(**cfg)
    model.load_state_dict(synth.synth_params(cfg, 1234), strict=True)
    model = model.cuda().eval()
    crit = FlowtronLoss(sigma=1.0, gate_loss=True, use_ctc_loss=True, ctc_loss_weight=1.0)
    for B in (int(x) for x in args.batches.split(",")):
        b = make_batch(B, 5000 + B)
        il_host, ol_host = b["in_lens"].tolist(), b["out_lens"].tolist()
        args_cuda = (b["mel"], b["speaker_ids"], b["text"], b["in_lens"], b["out_lens"], b["attn_prior"])
        call_host = lambda: model.score(b["mel"], b["speaker_ids"], b["text"], il_host, ol_host, b["attn_prior"])
        call_cuda = lambda: model.score(*args_cuda)
        graph = None
        if "score_graph" in arms:
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                call_cuda()
            torch.cuda.current_stream().wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                captured = call_cuda()
        ref = call_host()
        eager = call_cuda()
        if graph is not None:
            graph.replay()
            torch.cuda.synchronize()
            assert all(torch.equal(captured[k], eager[k]) for k in ("nll", "gate", "ctc")), "graph replay differs"
        for r in range(args.rounds):
            for arm in (arms if r % 2 == 0 else arms[::-1]):
                rec = {"arm": arm, "batch": B, "round": r}
                if arm == "score_host":
                    rec["ms_per_call"] = round(timed(call_host, args.reps), 2)
                elif arm == "score_cuda":
                    rec["ms_per_call"] = round(timed(call_cuda, args.reps), 2)
                elif arm == "score_graph":
                    rec["ms_per_call"] = round(timed(graph.replay, args.reps), 2)
                else:
                    rows = []
                    rec["ms_per_call"] = round(timed(lambda: rows.append(loop_b1(model, crit, b)), args.loop_reps), 2)
                    got = torch.tensor(rows[-1], dtype=torch.float64)
                    want = torch.stack([ref["nll"].double().cpu(), ref["gate"].double().cpu(),
                                        ref["ctc"].double().mean(0).cpu()], 1)
                    rec["max_rel_diff_vs_score"] = float(((got - want).abs() / want.abs().clamp_min(1e-12)).max())
                rec["utterances_per_s"] = round(B / rec["ms_per_call"] * 1e3, 1)
                assert _lib.device_status() == 0
                print(json.dumps({**rec, "frames": int(sum(ol_host)), "max_frames": max(ol_host),
                                  "max_text": max(il_host), "gpu": name, "power_limit_w": plim}), flush=True)
        del graph


if __name__ == "__main__":
    main()
