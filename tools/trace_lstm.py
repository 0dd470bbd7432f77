#!/usr/bin/env python
"""Per-phase timing of the persistent LSTM forward kernel (clock64 stamps of CTA 0) -> where a step's time goes."""
import ctypes, sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from flowtron_b200 import _lib

def main():
    T, B, H = 400, int(sys.argv[1]) if len(sys.argv) > 1 else 32, 1024
    g = torch.Generator().manual_seed(0)
    xproj = (torch.randn(T, B, 4 * H, generator=g) * 0.8).cuda()
    whh = (torch.randn(4 * H, H, generator=g) * 0.02).cuda().half()
    hseq = torch.zeros(T, B, H, device="cuda", dtype=torch.float16)
    gates = torch.zeros(T, B, 4 * H, device="cuda", dtype=torch.float16)
    cst = torch.zeros(T, B, H, device="cuda")
    trace = torch.zeros(T, 16, dtype=torch.int64, device="cuda")
    L = _lib.lib()
    L.ft_debug_set_lstm_trace.argtypes = [ctypes.c_void_p]
    for it in range(3):
        if it == 2:
            L.ft_debug_set_lstm_trace(ctypes.c_void_p(trace.data_ptr()))
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        _lib.lstm_fwd(xproj, whh, None, hseq, gates, cst)
        e1.record()
        torch.cuda.synchronize()
        print(f"run {it}: {e0.elapsed_time(e1) * 1e3 / T:.2f} us/step")
    L.ft_debug_set_lstm_trace(None)
    report(trace, T, "forward", {0: "flags_seen", 1: "tma_issued", 2: "first_group_landed", 4: "accum_done(wgmma)",
                                 5: "last_group_landed", 6: "proxy_fence_done", 7: "release_issued",
                                 8: "acc_in_smem", 9: "cell_done_h_stored", 10: "epi_barrier_done"})
    if os.environ.get("FT_TRACE_FWD_ONLY"):
        return
    # ---- backward
    w = torch.randn(T, B, H, generator=g).cuda()
    dG = torch.zeros(T, B, 4 * H, device="cuda", dtype=torch.float16)
    whhT = whh.float().t().contiguous().half()
    trace.zero_()
    for it in range(3):
        if it == 2:
            L.ft_debug_set_lstm_trace(ctypes.c_void_p(trace.data_ptr()))
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        _lib.lstm_bwd(w, whhT, gates, cst, None, dG)
        e1.record()
        torch.cuda.synchronize()
        print(f"bwd run {it}: {e0.elapsed_time(e1) * 1e3 / T:.2f} us/step")
    L.ft_debug_set_lstm_trace(None)
    report(trace, T, "backward", {0: "flags_seen", 1: "partials_visible(cluster)", 2: "first_group_landed", 4: "accum_done(wgmma)",
                                  5: "dG_stored", 6: "own_partial_written", 7: "release_issued"}, reverse=True)


def report(trace, T, title, names, reverse=False):
    tr = trace.cpu().double()[50:350]
    if reverse:
        tr = torch.flip(tr, (0,))
    print(f"== {title}")
    period = (tr[1:, 0] - tr[:-1, 0]).mean().item()
    print(f"step period: {period:.0f} clk = {period / 1.98e3:.2f} us @1.98GHz")
    base = tr[:, 0:1]
    rel = (tr - base).mean(0)
    for slot, n in names.items():               # {trace slot: phase}; slots a kernel does not stamp are not listed
        v = rel[slot].item()
        print(f"  {n:24s} +{v:8.0f} clk ({v / 1980:.2f} us)")
    # time from own release (slot 7, step t) to flags_seen of step t+1
    gap = (tr[1:, 0] - tr[:-1, 7]).mean().item()
    print(f"  own release(t) -> flags_seen(t+1): {gap:.0f} clk ({gap / 1980:.2f} us)")

if __name__ == "__main__":
    main()
