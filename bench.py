#!/usr/bin/env python
"""Benchmarks of the H100-native Flowtron hot path (one JSON line per run).

    python bench.py [--gpus N] [--steps K] [--warmup W]                 # headline: training, BASELINE.json configs[1]
    python bench.py --workload train --config 3 ...                     # configs[2]: LibriTTS-like, 123 speakers, B=64/GPU
    python bench.py --workload infer --batch {1,16} [--frames 400]      # configs[3]: Flowtron.infer, frames/s + RTF
    python bench.py --workload mel [--utterances 10000]                 # configs[4]: TacotronSTFT sweep, GB/s vs HBM
    python bench.py --impl reference [--workload ...]                   # the UNMODIFIED reference on the host CPU cores
    python bench.py ... --dump-outputs DIR                              # also write the last timed step's outputs as DIR/<name>.npy

train: a step = Flowtron.forward -> FlowtronLoss -> backward -> bucketed NCCL gradient all-reduce (N>1) -> grad-norm clip
-> RAdam step (train.py:281-331).  `value` = valid mel frames (sum of out_lens over all ranks) per second with inputs
resident in HBM; `e2e` = the same through the public module API from pinned host inputs: mel / text / lengths / gate
target are copied every step on a copy stream into double buffers, the attention prior is built on the device from the
lengths (flowtron_b200.data.attn_prior_batch: it is the reference's CPU data-loader work, data.py:31-41), and every
step's loss is read back to the host (pinned, one step late so the launch queue is not drained).
FT_GRAPH=1 (default where it captures): forward + backward + all-reduce + clip + optimizer are replayed from ONE CUDA
graph (CUDA streams and graphs instead of a tracing compiler); FT_GRAPH=0 issues the ~1500 launches eagerly.
Precision: fp16 tensor-core operands (backward on device-side loss-scaled gradients), fp32 accumulation/state (DESIGN.md).
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import threading
import time

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

FLOP_PER_FRAME_FWD = lambda L: 53_677_312 + 1_280 * L        # SURVEY.md §8d, per flow, tensor ops only
WEIGHT_PARAMS_PER_FLOW = 4096 * 80 + 4 * 4096 * 1024 + 4096 * 1664 + 640 * 1024 + 2 * 1024 * 1024 + 160 * 1024   # matvec weights read per frame
MEL_BYTES_PER_FRAME = {"f32": 1344, "s16": 832}              # SURVEY.md §8d: 256 new samples + 80 f32 mel values


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--workload", default="train", choices=["train", "infer", "mel"])
    ap.add_argument("--config", type=int, default=2, choices=[2, 3], help="train: BASELINE.json configs index (2 = LJS B=32, 3 = LibriTTS B=64)")
    ap.add_argument("--batch", type=int, default=None)
    ap.add_argument("--frames", type=int, default=None)
    ap.add_argument("--utterances", type=int, default=10000, help="mel: utterances in the sweep")
    ap.add_argument("--wav-int16", action="store_true", help="mel: int16 PCM input (832 B/frame) instead of f32 (1344 B/frame)")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--streams", type=int, default=1, help="train: 2 = two half-batch pipelines on two CUDA streams")
    ap.add_argument("--profile", action="store_true", help="short run for a profiler: no e2e leg, no CPU baseline, no graph, warm-up as given")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write what the timed path computed in its last step as DIR/<name>.npy (float32)")
    return ap.parse_args()


DUMP_LIMIT = 2 << 20          # elements per dumped array; larger outputs are dumped as a fixed, seeded sample (64 MB cap in all)


def snapshot(arrays):
    """Host float32 copies of the named device tensors, each at most DUMP_LIMIT elements (a seeded sample of larger ones,
    the same indices on every run) -- taken right after the timed window, before anything else runs."""
    out = {}
    for name, t in arrays.items():
        if not torch.is_tensor(t):
            continue
        a = t.detach().float()
        if a.numel() > DUMP_LIMIT:
            idx = torch.randint(0, a.numel(), (DUMP_LIMIT,), generator=torch.Generator().manual_seed(0)).sort().values
            a = a.reshape(-1)[idx.to(a.device)]
            name += "_sample"
        out[name] = a.cpu().numpy()
    assert sum(a.nbytes for a in out.values()) <= 64 << 20, "dumped outputs exceed 64 MB"
    return out


def write_dump(directory, arrays):
    import numpy as np
    os.makedirs(directory, exist_ok=True)
    for name, a in arrays.items():
        np.save(os.path.join(directory, name + ".npy"), a)


# ------------------------------------------------------------------------------------------------ clocks
class ClockSampler(threading.Thread):
    Q = "clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown," \
        "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"

    def __init__(self, index: int):
        super().__init__(daemon=True)
        self.index, self.samples, self._stop_ev = index, [], threading.Event()

    def run(self):
        while not self._stop_ev.is_set():
            try:
                r = subprocess.run(["nvidia-smi", f"--id={self.index}", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits"],
                                   capture_output=True, text=True, timeout=5)
                f = [x.strip() for x in r.stdout.strip().split(",")]
                if len(f) >= 7:
                    self.samples.append(f)
            except Exception:
                pass
            self._stop_ev.wait(0.2)

    def stop(self):
        self._stop_ev.set()
        self.join(timeout=3)
        if not self.samples:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["no_samples"]}
        sm = sorted(int(float(s[0])) for s in self.samples)
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        reasons = [n for i, n in enumerate(names) if any(s[3 + i].lower().startswith("active") for s in self.samples)]
        return {"sm_mhz": sm[len(sm) // 2], "sm_max_mhz": int(float(self.samples[0][1])), "reasons": reasons,
                "power_w_max": max(float(s[2]) for s in self.samples), "samples": len(sm)}


def peaks():
    """(bf16 TFLOP/s, sustained bf16 TFLOP/s, HBM GB/s, source): MEASURED_PEAKS.json where the machine provides one, else
    NVIDIA's H100 SXM data sheet (dense bf16 at 700 W; no sustained figure is published, so the same value stands in)."""
    path = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(path):
        p = json.load(open(path))
        return p.get("bf16_tflops", 989.0), p.get("bf16_tflops_sustained", 989.0), p.get("hbm_gbs", 3350.0), "measured"
    return 989.0, 989.0, 3350.0, "fallback (H100 SXM data sheet)"


def dist_env():
    return int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0"))


def make_timed(world, dev):
    import torch.distributed as dist

    def timed(fn, k):
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(k):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms = torch.tensor([e0.elapsed_time(e1)], device=dev, dtype=torch.float64)
        if world > 1:
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
            dist.barrier()
        return float(ms.item())
    return timed


def kernel_tables(trep, steps):
    by_name = {}
    for name, m, n, k, cnt, tms in trep:
        a = by_name.setdefault(name, {"count": 0, "ms": 0.0, "flop": 0.0})
        a["count"] += cnt
        a["ms"] += tms
        if name.startswith("gemm"):
            a["flop"] += 2.0 * m * n * k * cnt
        elif name.startswith("lstm"):
            a["flop"] += 2.0 * n * 1024 * 4096 * max(m - 1, 0) * cnt       # (T-1) recurrent [B,1024]x[1024,4096] products
        elif name.startswith("attn_fwd") or name.startswith("attn_bwd"):
            a["flop"] += (2.0 if name == "attn_fwd" else 6.0) * n * m * k * 640 * cnt
    table = {k: {"ms_per_step": v["ms"] / steps, "launches_per_step": v["count"] / steps,
                 "tflops": (v["flop"] / (v["ms"] / 1e3) / 1e12) if v["ms"] > 0 and v["flop"] > 0 else None} for k, v in by_name.items()}
    top_shapes = sorted(trep, key=lambda r: -r[5])[:14]
    shapes = [{"kernel": n_, "m": m_, "n": nn_, "k": k_, "launches_per_step": c_ / steps, "ms_per_launch": t_ / c_,
               "tflops": (2.0 * m_ * nn_ * k_ / (t_ / c_ / 1e3) / 1e12) if n_.startswith("gemm") else None}
              for n_, m_, nn_, k_, c_, t_ in top_shapes]
    return by_name, table, shapes


def cpu_baseline_leg(workload, world):
    """The UNMODIFIED reference on this box's host cores, bounded sample (rank 0 only; test infrastructure from oracle/)."""
    from oracle import ref_runner, ref_shims
    if not ref_shims.runnable():
        return {"value": None, "unit": None, "cores": 0, "kind": "reference", "sample": "oracle/_ref not staged (run build() where /root/reference exists)"}
    if workload == "train":
        return ref_runner.time_train(steps=1 if world > 1 else 2, warmup=0, B=2, T=500)
    if workload == "infer":
        return ref_runner.time_infer(steps=1, warmup=1, T=200)
    return ref_runner.time_mel(n_utt=48)


# ------------------------------------------------------------------------------------------------ reference arm
def run_reference_arm(args):
    world, rank, _ = dist_env()
    if rank != 0:
        return
    from oracle import ref_runner, ref_shims
    t0 = time.perf_counter()
    if not ref_shims.runnable():
        print(json.dumps({"impl": "reference", "unavailable": "oracle/_ref (byte-compiled reference modules) not staged on this box"}))
        return
    steps, warm = max(1, args.steps), min(max(0, args.warmup), 1)      # bounded: the CPU reference runs ~150 frames/s
    if args.workload == "train":
        cb = ref_runner.time_train(steps=steps, warmup=warm, B=2, T=args.frames or 1000)
        metric, unit = "training mel-frames/sec", "valid mel-frames/s"
        wl = "configs[1] sequence shape (2-flow, T<=1000, LJS-like text lengths, prior on) at the batch the CPU finishes in seconds (B=2)"
    elif args.workload == "infer":
        cb = ref_runner.time_infer(steps=steps, warmup=warm, T=args.frames or 400)
        metric, unit = "inference mel-frames/sec", "mel-frames/s"
        wl = "configs[3]: Flowtron.infer, 2-flow, sigma=0.5, B=1 (the reference raises for B>1 with a gate layer)"
    else:
        cb = ref_runner.time_mel(n_utt=min(args.utterances, 64 * steps))
        metric, unit = "mel front-end mel-frames/sec", "mel-frames/s"
        wl = "configs[4]: TacotronSTFT.mel_spectrogram, 22.05 kHz, hop 256, 80 mel, one utterance at a time (data.py:149-155)"
    out = {"impl": "reference", "metric": metric, "value": cb["value"], "unit": unit, "n_gpus": args.gpus, "steps": steps,
           "warmup": warm, "ms_per_step": cb.get("s_per_step", 0.0) * 1e3 if cb.get("s_per_step") else None, "higher_is_better": True,
           "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
           "config": {"workload": wl, "sample": cb["sample"], "cpu_model": cb.get("cpu_model"), "physical_cores": cb.get("physical_cores"),
                      "thread_sweep_s": cb.get("thread_sweep_s")},
           "cpu_baseline": cb, "e2e": {"value": cb["value"], "unit": unit, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
           "gpu_launches": 0, "wall_s": time.perf_counter() - t0}
    print(json.dumps(out))


# ------------------------------------------------------------------------------------------------ train
def train_lengths(config, B, T, seed):
    from flowtron_b200 import synth
    if config == 3:        # SURVEY §8d cfg 3: LibriTTS (<10 s): out_lens ~ U{150..860}, max forced
        g = torch.Generator().manual_seed(seed)
        out_lens = torch.randint(150, T + 1, (B,), generator=g)
        out_lens[0] = T
        in_lens = torch.clamp((out_lens.float() / 6.5).round().long(), 20, 160)
        return out_lens, in_lens
    return synth.ljs_like_lengths(B, T, seed)


def run_train(args):
    import torch.distributed as dist
    from flowtron_b200 import _lib, synth
    from flowtron_b200 import data as ftdata
    from flowtron_b200 import distributed as ftd
    from flowtron_b200.flowtron import Flowtron, FlowtronLoss

    world, rank, local = dist_env()
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        ftd.init_distributed(rank, world, "nccl")
    timed = make_timed(world, dev)

    cfg = dict(synth.DEFAULT_MODEL_CONFIG)                    # config.json model_config: 2 flows
    if args.config == 3:
        cfg["n_speakers"] = 123                               # unique speaker ids in the LibriTTS filelist (SURVEY §8d)
    B = args.batch or (64 if args.config == 3 else 32)
    T = args.frames or (860 if args.config == 3 else 1000)
    model = Flowtron(**cfg)
    model.load_state_dict(synth.synth_params(cfg, 1234), strict=True)
    model = model.to(dev).train()
    model.n_streams = args.streams
    crit = FlowtronLoss(sigma=1.0, gate_loss=True, use_ctc_loss=False)
    use_graph = os.environ.get("FT_GRAPH", "1") != "0" and not args.profile and args.streams == 1
    # flowtron_b200.RAdam (fused clip + update, reference radam.py semantics, capturable) is the default since r2: 60.3 -> 58.4
    # ms/step vs torch.optim.RAdam(foreach, capturable); FT_FUSED_OPT=0 selects torch's
    fused_opt = os.environ.get("FT_FUSED_OPT", "1") != "0"
    # train.py:231-252 order: optimizer first, then the all-reduce wrapper
    if fused_opt:
        from flowtron_b200.radam import RAdam
        opt = RAdam(model.parameters(), lr=1e-3, weight_decay=1e-6, capturable=use_graph)
    else:
        opt = torch.optim.RAdam(model.parameters(), lr=1e-3, weight_decay=1e-6, capturable=use_graph, foreach=True)
    if world > 1:
        ftd.apply_gradient_allreduce(model)

    out_lens, in_lens = train_lengths(args.config, B, T, 1234 + rank)        # every rank gets its own utterances (weak scaling)
    L = int(in_lens.max())
    batch = synth.synth_batch(B, T, L, cfg, 1234 + rank, out_lens=out_lens.tolist(), in_lens=in_lens.tolist(), with_prior=True,
                              logmel_stats=True)
    keys_h2d = ["mel", "speaker_ids", "text", "in_lens", "out_lens", "gate_target"]      # the prior is built on the device
    host = {k: batch[k].pin_memory() for k in keys_h2d}
    static = {k: batch[k].to(dev) for k in keys_h2d + ["attn_prior"]}       # resident inputs (`value`); also the graph's inputs
    frames_rank = int(batch["out_lens"].sum())
    frames_t = torch.tensor([frames_rank], device=dev, dtype=torch.float64)
    if world > 1:
        dist.all_reduce(frames_t)
    frames_all = float(frames_t.item())
    h2d_bytes = sum(host[k].numel() * host[k].element_size() for k in keys_h2d)

    def zero_grads():
        if world > 1:
            model.zero_grad_buckets()
        elif fused_opt:
            opt.zero_grad()                                   # one memset of the flat gradient buffer
        else:
            opt.zero_grad(set_to_none=True)

    loss_static = torch.zeros((), device=dev)

    last = {}

    def step_body(d):
        zero_grads()
        out = model(d["mel"], d["speaker_ids"], d["text"], d["in_lens"], d["out_lens"], d["attn_prior"])
        nll, gl, _ = crit(out, d["gate_target"], d["in_lens"], d["out_lens"])
        # detached views only: a reference into the autograd graph would keep it alive across steps and break graph capture
        last.update(z=out[0].detach(), log_s=[t.detach() for t in out[1]], gate=out[2].detach(),
                    attns=[t.detach() for t in out[3] if torch.is_tensor(t)], nll=nll.detach(), gate_loss=gl.detach())
        loss = (nll + gl).sum()
        loss.backward()
        if fused_opt:
            opt.clip_grad_norm_(1.0)                          # norm + coefficient stay on the device, applied inside step()
        else:
            torch.nn.utils.clip_grad_norm_(model.parameters(), 1.0, foreach=True)
        opt.step()
        loss_static.copy_(loss.detach())

    n_warm = args.warmup if args.profile else max(3, args.warmup)
    _lib.reset_launch_count()
    for _ in range(n_warm):
        step_body(static)
    torch.cuda.synchronize()
    assert _lib.device_status() == 0, "device watchdog tripped"
    launches_per_step = _lib.launch_count() / max(1, n_warm)

    graph, graph_note = None, None
    if use_graph:
        try:
            g = torch.cuda.CUDAGraph()
            zero_grads()
            torch.cuda.synchronize()
            with torch.cuda.graph(g):
                step_body(static)
            torch.cuda.synchronize()
            g.replay()
            torch.cuda.synchronize()
            assert _lib.device_status() == 0
            graph = g
        except Exception as e:                                # capture is an optimisation: fall back to eager launches, say so
            graph_note = f"capture failed: {type(e).__name__}: {str(e)[:160]}"
            try:
                torch.cuda.synchronize()
            except Exception:
                pass

    def step_value():
        if graph is not None:
            graph.replay()
        else:
            step_body(static)

    # ---- e2e: pinned host -> (copy stream) -> staging double buffers -> static inputs; prior on the device; loss read back
    copy_stream = torch.cuda.Stream(device=dev)
    staging = [{k: torch.empty_like(static[k]) for k in keys_h2d} for _ in range(2)]
    ready = [torch.cuda.Event() for _ in range(2)]
    consumed = [torch.cuda.Event() for _ in range(2)]
    loss_host = torch.zeros((), dtype=torch.float32).pin_memory()
    loss_ev = torch.cuda.Event()
    e2e_state = {"i": 0, "losses": [], "pending": False}

    def prefetch(slot):
        with torch.cuda.stream(copy_stream):
            copy_stream.wait_event(consumed[slot])            # the step that last read this slot has copied it out
            for k in keys_h2d:
                staging[slot][k].copy_(host[k], non_blocking=True)
            ready[slot].record(copy_stream)

    def step_e2e():
        i = e2e_state["i"]
        slot = i & 1
        cur = torch.cuda.current_stream(dev)
        cur.wait_event(ready[slot])
        for k in keys_h2d:
            static[k].copy_(staging[slot][k], non_blocking=True)
        consumed[slot].record(cur)
        prefetch(slot)                                        # the copy for step i+2 runs under steps i and i+1
        ftdata.attn_prior_batch(static["in_lens"], static["out_lens"], T, L, out=static["attn_prior"])
        if e2e_state["pending"]:                              # read the PREVIOUS step's loss (already on the host or about to be)
            loss_ev.synchronize()
            e2e_state["losses"].append(float(loss_host))
        step_value()
        loss_host.copy_(loss_static, non_blocking=True)
        loss_ev.record(cur)
        e2e_state["pending"] = True
        e2e_state["i"] = i + 1

    sampler = ClockSampler(local)
    sampler.start()
    ms = timed(step_value, args.steps)
    dump = None
    if args.dump_outputs:
        arrays = {"z": last["z"], "gate": last["gate"], "nll": last["nll"], "gate_loss": last["gate_loss"], "loss": loss_static,
                  "params_after_step": torch.cat([q.detach().reshape(-1) for q in model.parameters()])}
        arrays.update({f"log_s{i}": t for i, t in enumerate(last["log_s"])})
        arrays.update({f"attn{i}": t for i, t in enumerate(last["attns"])})
        dump = snapshot(arrays)
    ms_e2e = ms
    if not args.profile:
        for s in range(2):
            consumed[s].record(torch.cuda.current_stream(dev))
            prefetch(s)
        step_e2e()                                            # untimed: fills the pipeline
        torch.cuda.synchronize()

        def e2e_k():
            step_e2e()
        ms_e2e = timed(e2e_k, args.steps)
        loss_ev.synchronize()
        e2e_state["losses"].append(float(loss_host))
    clocks = sampler.stop()

    # ---- per-kernel device times (CUDA events around every launch of the library, eager pass of the same step)
    _lib.timing(True)
    for _ in range(args.steps):
        step_body(static)
    trep = _lib.timing_report()
    _lib.timing(False)
    assert _lib.device_status() == 0, "device watchdog tripped"

    if rank != 0:
        return
    value = frames_all * args.steps / (ms / 1e3)
    e2e = frames_all * args.steps / (ms_e2e / 1e3)
    burst, sustained, hbm, src = peaks()
    by_name, kernel_table, shape_table = kernel_tables(trep, args.steps)
    lstm = {k: v for k, v in by_name.items() if k.startswith("lstm")}
    top = max(lstm.items(), key=lambda kv: kv[1]["ms"]) if lstm else (max(by_name.items(), key=lambda kv: kv[1]["ms"]) if by_name else (None, None))
    roof = None
    if top[0]:
        t = top[1]
        ach = t["flop"] / (t["ms"] / 1e3) / 1e12
        steps_per_launch = (T - 1)
        roof = {"kernel": top[0], "bound": "tensor", "achieved": ach, "peak": sustained, "unit": "TFLOP/s", "frac": ach / sustained,
                "traffic": None, "peak_source": f"{src} bf16 sustained (kernel timed inside a long step)",
                "launches": t["count"], "avg_ms": t["ms"] / t["count"], "share_of_step": t["ms"] / (ms if graph is None else ms),
                "us_per_recurrent_step": (t["ms"] / t["count"]) * 1e3 / steps_per_launch,
                "note": "latency-bound T-step dependency chain (DESIGN.md): algorithmic FLOPs = 2*B*1024*4096*(T-1) per launch; "
                        "kernel times from an eager instrumented pass of the same step"}
    flop_step = 3.0 * 2 * FLOP_PER_FRAME_FWD(L) * B * T * world       # fwd+bwd, 2 flows, padded frames
    wl = ("configs[1]: LJS single-speaker 2-flow Flowtron train step, n_mel=80, per-GPU batch 32, T<=1000" if args.config == 2 else
          "configs[2]: LibriTTS multi-speaker (123 speakers) 2-flow Flowtron train step, per-GPU batch 64, T<=860")
    out = {
        "metric": "training mel-frames/sec", "value": value, "unit": "valid mel-frames/s", "n_gpus": world,
        "steps": args.steps, "warmup": n_warm, "ms_per_step": ms / args.steps, "higher_is_better": True,
        "scaling": "weak", "vs_baseline": None, "dtype": "f16 tensor-core operands (loss-scaled in backward), f32 accumulate+state",
        "data": "synthetic",
        "config": {"workload": wl, "per_gpu_batch": B, "global_batch": B * world, "max_frames": T, "max_text": L, "attn_prior": True,
                   "optimizer": ("flowtron_b200.RAdam (fused)" if fused_opt else "torch.optim.RAdam" + (" capturable" if use_graph else "")) + " lr=1e-3 wd=1e-6 + clip_grad_norm 1.0",
                   "parallelism": f"dp{world}", "streams_per_rank": args.streams, "cuda_graph": graph is not None, "cuda_graph_note": graph_note,
                   "encoder_overlap": bool(model.overlap_encoder), "padded_frames_per_s": B * T * world * args.steps / (ms / 1e3),
                   "pipe_fwd": os.environ.get("FT_PIPE_FWD", "default"), "pipe_bwd": os.environ.get("FT_PIPE_BWD", "default"),
                   "att_overlap": os.environ.get("FT_ATT_OVERLAP", "default"), "fuse_bwd": os.environ.get("FT_FUSE_BWD", "default"),
                   "l2": "working set per step (>3 GB of activations) exceeds the 50 MB L2; no explicit flush"},
        "e2e": {"value": e2e, "unit": "valid mel-frames/s", "h2d_bytes_per_step": h2d_bytes, "d2h_bytes_per_step": 4,
                "ms_per_step": ms_e2e / args.steps, "prior": "built on the device from the lengths (ft_attn_prior)",
                "losses_read": len(e2e_state["losses"]), "last_loss": e2e_state["losses"][-1] if e2e_state["losses"] else None},
        "gpu_launches": int(round(launches_per_step * args.steps)), "clocks": clocks, "roofline": roof, "kernels": kernel_table,
        "top_launch_shapes": shape_table,
        "model_tflops": flop_step * args.steps / (ms / 1e3) / 1e12,
        "model_tensor_frac": flop_step * args.steps / (ms / 1e3) / 1e12 / (sustained * world),
    }
    if args.profile:
        out["invalid"] = "profiling run (timings under a profiler are never reported)"
    elif not args.no_cpu_baseline:
        out["cpu_baseline"] = cpu_baseline_leg("train", world)
    if dump is not None:
        write_dump(args.dump_outputs, dump)
        out["dumped_outputs"] = sorted(dump)
    print(json.dumps(out))


# ------------------------------------------------------------------------------------------------ infer
def run_infer(args):
    from flowtron_b200 import _lib, synth
    from flowtron_b200.flowtron import Flowtron
    world, rank, local = dist_env()
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        from flowtron_b200 import distributed as ftd
        ftd.init_distributed(rank, world, "nccl")              # replicas only: the group exists for the barrier / max-over-ranks
    timed = make_timed(world, dev)
    cfg = dict(synth.DEFAULT_MODEL_CONFIG)
    B, T, L = args.batch or 1, args.frames or 400, 100        # inference.py:104-108 defaults; SURVEY §8d cfg 4
    params = synth.synth_params(cfg, 1234)
    key = [k for k in params if k.endswith("gate_layer.linear_layer.bias")][0]
    params[key] = torch.full_like(params[key], -10.0)          # the gate never fires: all T frames are produced (fixed work)
    model = Flowtron(**cfg)
    model.load_state_dict(params, strict=True)
    model = model.to(dev).eval()
    g = torch.Generator().manual_seed(1234 + rank)
    res_h = (torch.randn(B, 80, T, generator=g) * 0.5).pin_memory()
    text_h = torch.randint(0, cfg["n_text"], (B, L), generator=g).pin_memory()
    spk_h = torch.zeros(B, dtype=torch.long).pin_memory()
    res, text, spk = res_h.to(dev), text_h.to(dev), spk_h.to(dev)
    out_h = torch.empty(B, 80, T).pin_memory()

    def step():
        with torch.no_grad():
            mel, _ = model.infer(res, spk, text, temperature=1.0, gate_threshold=0.5)
        return mel

    def step_e2e():
        with torch.no_grad():
            mel, _ = model.infer(res_h.to(dev, non_blocking=True), spk_h.to(dev, non_blocking=True), text_h.to(dev, non_blocking=True))
        out_h[:, :, :mel.size(2)].copy_(mel, non_blocking=True)
        torch.cuda.current_stream().synchronize()             # the request's result is on the host

    n_warm = args.warmup if args.profile else max(3, args.warmup)
    for _ in range(n_warm):
        mel = step()
    torch.cuda.synchronize()
    assert _lib.device_status() == 0 and mel.size(2) == T
    sampler = ClockSampler(local)
    sampler.start()
    _lib.reset_launch_count()
    _lib.timing(True)
    last = {}

    def step_timed():
        last["mel"] = step()

    ms = timed(step_timed, args.steps)
    launches = _lib.launch_count()
    trep = _lib.timing_report()
    _lib.timing(False)
    dump = snapshot({"mel": last["mel"]}) if args.dump_outputs else None
    ms_e2e = ms if args.profile else timed(step_e2e, args.steps)
    clocks = sampler.stop()
    if rank != 0:
        return
    burst, sustained, hbm, src = peaks()
    fps = B * T * args.steps * world / (ms / 1e3)
    fps_e2e = B * T * args.steps * world / (ms_e2e / 1e3)
    by_name, kernel_table, _ = kernel_tables(trep, args.steps)
    kms = by_name.get("infer", {"ms": 0.0, "count": 1})
    wbytes = WEIGHT_PARAMS_PER_FLOW * 2.0                      # fp16 weights streamed per frame per flow (L2-resident after the first frame)
    ach = wbytes * T / (kms["ms"] / max(1, kms["count"]) / 1e3) / 1e9 if kms["ms"] else None
    out = {
        "metric": "inference mel-frames/sec", "value": fps, "unit": "mel-frames/s", "n_gpus": world, "steps": args.steps, "warmup": n_warm,
        "ms_per_step": ms / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "f16 weights/operands, f32 accumulate+state", "data": "synthetic",
        "config": {"workload": f"configs[3]: Flowtron.infer, 2-flow, sigma=0.5, batch {B}, {T} frames, {L} text tokens, gate disabled (fixed work)",
                   "batch": B, "frames": T, "text": L, "parallelism": f"replicas x{world}",
                   "l2": "weights (107 MB fp16 for 2 flows) are re-read every frame; inputs/outputs are KBs -- no flush"},
        "rtf": {"frames_per_s_per_stream": T * args.steps / (ms / 1e3), "x_real_time_per_stream": T * args.steps / (ms / 1e3) / (22050.0 / 256.0),
                "us_per_frame_per_flow": ms * 1e3 / args.steps / T / 2},
        "e2e": {"value": fps_e2e, "unit": "mel-frames/s", "h2d_bytes_per_step": res_h.numel() * 4 + text_h.numel() * 8 + spk_h.numel() * 8,
                "d2h_bytes_per_step": out_h.numel() * 4, "ms_per_step": ms_e2e / args.steps},
        "gpu_launches": int(launches), "clocks": clocks,
        "roofline": {"kernel": "infer_kernel", "bound": "hbm", "achieved": ach, "peak": hbm, "unit": "GB/s", "frac": (ach / hbm) if ach else None,
                     "traffic": None, "peak_source": f"{src} HBM copy bandwidth", "launches": kms["count"],
                     "avg_ms": kms["ms"] / max(1, kms["count"]),
                     "note": f"algorithmic bytes = {wbytes / 1e6:.1f} MB of fp16 weights per frame per flow x {T} frames per launch (batch-independent)"},
        "kernels": kernel_table,
    }
    if args.profile:
        out["invalid"] = "profiling run"
    elif not args.no_cpu_baseline:
        out["cpu_baseline"] = cpu_baseline_leg("infer", world)
    if dump is not None:
        write_dump(args.dump_outputs, dump)
        out["dumped_outputs"] = sorted(dump)
    print(json.dumps(out))


# ------------------------------------------------------------------------------------------------ mel
def run_mel(args):
    from flowtron_b200 import _lib
    from flowtron_b200.audio_processing import TacotronSTFT
    world, rank, local = dist_env()
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        from flowtron_b200 import distributed as ftd
        ftd.init_distributed(rank, world, "nccl")              # replicas only (each rank sweeps its own shard)
    timed = make_timed(world, dev)
    stft = TacotronSTFT(1024, 256, 1024, 80, 22050, 0.0, 8000.0).to(dev)
    g = torch.Generator().manual_seed(7 + rank)
    n_utt = args.utterances
    lens = torch.randint(22050, 220501, (n_utt,), generator=g)           # U{1..10} s at 22.05 kHz (SURVEY §8d cfg 5)
    total = int(lens.sum())
    fmt = "s16" if args.wav_int16 else "f32"
    gd = torch.Generator(device=dev).manual_seed(7 + rank)
    if args.wav_int16:
        flat = torch.randint(-31130, 31131, (total,), generator=gd, device=dev, dtype=torch.int32).to(torch.int16)
    else:
        flat = torch.rand(total, generator=gd, device=dev) * 1.9 - 0.95
    frames = int((1 + lens // 256).sum())
    out = torch.empty(frames * 80, device=dev)
    lens_l = lens.tolist()

    def step():
        stft.mel_spectrogram_packed(flat, lens_l, out=out)

    n_warm = args.warmup if args.profile else max(3, args.warmup)
    for _ in range(n_warm):
        step()
    torch.cuda.synchronize()
    assert _lib.device_status() == 0
    sampler = ClockSampler(local)
    sampler.start()
    _lib.reset_launch_count()
    _lib.timing(True)
    ms = timed(step, args.steps)
    launches = _lib.launch_count()
    trep = _lib.timing_report()
    _lib.timing(False)
    dump = snapshot({"mel": out}) if args.dump_outputs else None
    ms_e2e = ms
    h2d = d2h = 0
    if not args.profile:
        flat_h = torch.empty(total, dtype=flat.dtype).pin_memory()
        flat_h.copy_(flat)
        out_h = torch.empty(frames * 80).pin_memory()
        h2d, d2h = flat_h.numel() * flat_h.element_size(), out_h.numel() * 4

        def step_e2e():
            stft.mel_spectrogram_packed(flat_h.to(dev, non_blocking=True), lens_l, out=out)
            out_h.copy_(out, non_blocking=True)
            torch.cuda.current_stream().synchronize()
        step_e2e()
        ms_e2e = timed(step_e2e, args.steps)
    clocks = sampler.stop()
    if rank != 0:
        return
    burst, sustained, hbm, src = peaks()
    fps = frames * args.steps * world / (ms / 1e3)
    by_name, kernel_table, _ = kernel_tables(trep, args.steps)
    k = by_name.get("mel_fused", {"ms": ms, "count": args.steps})
    bpf = MEL_BYTES_PER_FRAME[fmt]
    ach = frames * bpf / (k["ms"] / k["count"] / 1e3) / 1e9
    traffic = None
    res = {
        "metric": "mel front-end mel-frames/sec", "value": fps, "unit": "mel-frames/s", "n_gpus": world, "steps": args.steps, "warmup": n_warm,
        "ms_per_step": ms / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "f32" if fmt == "f32" else "int16 PCM in, f32 math", "data": "synthetic",
        "config": {"workload": f"configs[4]: TacotronSTFT mel front-end sweep, 22.05 kHz, hop 256, n_mel 80, {n_utt} utterances U{{1..10}} s, one launch",
                   "utterances": n_utt, "frames": frames, "samples": total, "wav_format": fmt, "parallelism": f"replicas x{world}",
                   "l2": f"input {total * (2 if fmt == 's16' else 4) / 1e9:.2f} GB + output {frames * 320 / 1e9:.2f} GB per step: far larger than the 50 MB L2"},
        "gbs_algorithmic": frames * bpf * args.steps / (ms / 1e3) / 1e9,
        "e2e": {"value": frames * args.steps * world / (ms_e2e / 1e3), "unit": "mel-frames/s", "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": d2h,
                "ms_per_step": ms_e2e / args.steps, "note": "PCIe-bound: the whole waveform goes in and the whole mel comes back every step"},
        "gpu_launches": int(launches), "clocks": clocks,
        "roofline": {"kernel": "mel_fused_kernel", "bound": "hbm", "achieved": ach, "peak": hbm, "unit": "GB/s", "frac": ach / hbm,
                     "traffic": traffic, "peak_source": f"{src} HBM copy bandwidth", "launches": k["count"], "avg_ms": k["ms"] / k["count"],
                     "note": f"algorithmic bytes = {bpf} B/frame x {frames} frames per launch"},
        "kernels": kernel_table,
    }
    if args.profile:
        res["invalid"] = "profiling run"
    elif not args.no_cpu_baseline:
        res["cpu_baseline"] = cpu_baseline_leg("mel", world)
    if dump is not None:
        write_dump(args.dump_outputs, dump)
        res["dumped_outputs"] = sorted(dump)
    print(json.dumps(res))


def main():
    args = parse()
    torch.manual_seed(1234)       # the encoder's dropout masks are seeded from torch's: identical arguments, identical run
    if args.impl == "reference":
        return run_reference_arm(args)
    if args.workload == "train":
        return run_train(args)
    if args.workload == "infer":
        return run_infer(args)
    return run_mel(args)


if __name__ == "__main__":
    main()
    try:
        import torch.distributed as dist
        if dist.is_initialized():
            dist.destroy_process_group()
    except Exception:
        pass
