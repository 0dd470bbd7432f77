#!/usr/bin/env python
"""Does the layer pipeline's BPTT overlap?  One eager configs[1] training step (2 flows, B = 32, T <= 1000) under
torch.profiler (CUDA activities only), then, for each flow's backward, the start and end of every LSTM BPTT chunk
kernel on the two pipeline streams and the share of layer 0's chunk time that overlaps layer 1's chunks.

Also prints how many 4-CTA clusters of the BPTT cluster kernel fit on the device at its launch configuration, the
card and its power limit, and the kernels that start in the 300 us before each flow's first BPTT chunk (to see whether
the side-stream weight-gradient GEMMs delay it).

    python tools/bptt_overlap.py [--out DIR]       # DIR (default: a new temporary directory) receives the chrome trace
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from torch.profiler import profile, ProfilerActivity
from flowtron_b200 import _lib, synth
from flowtron_b200.flowtron import Flowtron, FlowtronLoss


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip() or r.stderr.strip()


def union_overlap(iv, others):
    """Length of interval iv covered by the union of `others`."""
    s, e = iv
    cov, cur = 0.0, s
    for a, b in sorted(others):
        a, b = max(a, cur), min(b, e)
        if b > a:
            cov += b - a
            cur = b
    return cov


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if args.out is None:
        args.out = tempfile.mkdtemp(prefix="bptt_overlap_")
    os.makedirs(args.out, exist_ok=True)
    print("card:", card())
    L = _lib.lib()
    if hasattr(L, "ft_debug_lstm_bwd_max_clusters"):
        L.ft_debug_lstm_bwd_max_clusters.argtypes = [ctypes.c_int]
        print("lstm_bwd4_kernel: max active 4-CTA clusters at B=32:", L.ft_debug_lstm_bwd_max_clusters(32),
              "(two pipelined chunks need 32)")
    print("SMs:", torch.cuda.get_device_properties(0).multi_processor_count)

    cfg = dict(synth.DEFAULT_MODEL_CONFIG)
    model = Flowtron(**cfg)
    model.load_state_dict(synth.synth_params(cfg, 1234), strict=True)
    model = model.cuda().train()
    crit = FlowtronLoss()
    ol, il = synth.ljs_like_lengths(32, 1000, 1234)
    batch = synth.synth_batch(32, 1000, int(il.max()), cfg, 1234, out_lens=ol.tolist(), in_lens=il.tolist(),
                              with_prior=True, logmel_stats=True)
    d = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in batch.items()}
    print("T =", int(ol.max()))

    def step():
        model.zero_grad(set_to_none=True)
        out = model(d["mel"], d["speaker_ids"], d["text"], d["in_lens"], d["out_lens"], d["attn_prior"])
        nll, gl, _ = crit(out, d["gate_target"], d["in_lens"], d["out_lens"])
        (nll + gl).sum().backward()

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    assert _lib.device_status() == 0
    path = os.path.join(args.out, "bptt_overlap_trace.json")
    prof.export_chrome_trace(path)
    print("trace:", path)
    with open(path) as f:
        tr = json.load(f)
    ks = [e for e in tr["traceEvents"] if e.get("cat") == "kernel" and "dur" in e]
    ks.sort(key=lambda e: e["ts"])
    bw = [e for e in ks if "ft::lstm_bwd" in e["name"]]
    by_stream = {}
    for e in bw:
        by_stream.setdefault(e["args"]["stream"], []).append(e)
    print("BPTT kernels per stream:", {s: (len(v), sorted({e['name'].split('(')[0] for e in v})) for s, v in by_stream.items()})
    # the attention LSTM's BPTT is one launch per flow; the pipeline streams carry the chunks
    pipe = {s: v for s, v in by_stream.items() if len(v) > 2}
    if len(pipe) != 2:
        print("could not find the two pipeline streams")
        return
    s1, s0 = sorted(pipe, key=lambda s: pipe[s][0]["ts"])     # layer 1's first chunk starts first
    c1, c0 = pipe[s1], pipe[s0]
    n_flows = 2
    per = len(c1) // n_flows
    t_origin = ks[0]["ts"]
    for f in range(n_flows):
        a = c1[f * per:(f + 1) * per]
        b = c0[f * per:(f + 1) * per]
        print(f"\nbackward {f}: layer 1 on stream {s1}, layer 0 on stream {s0} (us from the first kernel of the step)")
        print("  chunk  layer1 start    end   dur   | layer0 start    end   dur   overlap")
        iv1 = [(e["ts"], e["ts"] + e["dur"]) for e in a]
        tot0 = ov0 = 0.0
        for i, (x, y) in enumerate(zip(a, b)):
            s, e = y["ts"], y["ts"] + y["dur"]
            ov = union_overlap((s, e), iv1)
            tot0 += e - s
            ov0 += ov
            print(f"  {i:5d}  {x['ts'] - t_origin:10.0f} {x['ts'] + x['dur'] - t_origin:8.0f} {x['dur']:6.0f} | "
                  f"{s - t_origin:10.0f} {e - t_origin:8.0f} {e - s:6.0f}  {ov / (e - s):6.1%}")
        span = b[-1]["ts"] + b[-1]["dur"] - a[0]["ts"]
        busy1 = sum(e["dur"] for e in a)
        print(f"  layer-0 chunk time overlapping layer 1: {ov0 / tot0:.1%}; pipeline span {span / 1e3:.2f} ms, "
              f"layer 1 {busy1 / 1e3:.2f} ms + layer 0 {tot0 / 1e3:.2f} ms of chunk time")
        first = a[0]["ts"]
        pre = [e for e in ks if first - 300 <= e["ts"] < first or (e["ts"] < first < e["ts"] + e["dur"])]
        print("  kernels running or starting in the 300 us before the first chunk (start, end relative to it, stream):")
        for e in pre[-12:]:
            print(f"    {e['ts'] - first:8.0f} {e['ts'] + e['dur'] - first:8.0f}  s{e['args']['stream']}  {e['name'][:70]}")
    att = [v for s, v in by_stream.items() if s not in pipe]
    for v in att:
        for e in v:
            print(f"attention-LSTM BPTT (stream {e['args']['stream']}): {e['dur'] / 1e3:.2f} ms, {e['name'][:40]}")
    if hasattr(L, "ft_debug_lstm_bwd_chunk"):
        isolated_step_time(L)


def isolated_step_time(L):
    """Per-step time of each BPTT kernel running alone: T = 1000, B = 32, ten 100-step chunks back to back."""
    L.ft_debug_lstm_bwd_chunk.argtypes = [ctypes.c_int] * 4 + [ctypes.c_void_p, ctypes.c_longlong] + [ctypes.c_void_p] * 9
    T, B, H, CH = 1000, 32, 1024, 100
    g = torch.Generator(device="cuda").manual_seed(0)
    dh = torch.randn(T, B, H, device="cuda", generator=g)
    whhT = (torch.randn(H, 4 * H, device="cuda", generator=g) * 0.02).half()
    gates = torch.rand(T, B, 4 * H, device="cuda", generator=g).half()
    cst = torch.randn(T, B, H, device="cuda", generator=g)
    lens = torch.full((B,), T, device="cuda", dtype=torch.int32)
    dG = torch.empty(T, B, 4 * H, device="cuda", dtype=torch.float16)
    carry = torch.zeros(B, H, device="cuda")
    flags = torch.empty(CH * 128, device="cuda", dtype=torch.int32)
    xchg = torch.empty(2 * 16 * 4 * B * 64, device="cuda")
    st = torch.cuda.current_stream().cuda_stream

    def seq(x):
        for c in range(T // CH - 1, -1, -1):
            assert L.ft_debug_lstm_bwd_chunk(T, B, c * CH, (c + 1) * CH, dh.data_ptr(), H, whhT.data_ptr(), gates.data_ptr(),
                                             cst.data_ptr(), lens.data_ptr(), dG.data_ptr(), carry.data_ptr(), flags.data_ptr(),
                                             x, st) == 0

    for name, x in (("cluster (lstm_bwd4_kernel)", None), ("flat (lstm_bwd_flat_kernel)", xchg.data_ptr())):
        seq(x)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(5):
            seq(x)
        b.record()
        torch.cuda.synchronize()
        print(f"isolated BPTT, T={T} B={B} in {CH}-step chunks, {name}: {a.elapsed_time(b) / 5 / T * 1e3:.2f} us/step")
    assert _lib.device_status() == 0


if __name__ == "__main__":
    main()
