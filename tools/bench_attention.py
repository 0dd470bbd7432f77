#!/usr/bin/env python
"""Time the standalone Attention module (ft_attention_fwd / ft_attention_bwd) on the GPU at the model shape (Dq 1024, E 640,
A 640, L 160, T 1000: the attention of one AR_Step), for B = 8 and 32, and the reference module's math in plain torch on the
same GPU at B = 8 (fp32 and under fp16 autocast), where its [B, T, L, A] tanh tensor fits.

Reported, one JSON line per variant and direction: ms per call (warm-up, then `--runs` timed windows of `--steps` calls each,
CUDA events), for the forward alone (under torch.no_grad) and forward + backward (all three outputs feed a weighted sum).  The
card name and power limit are read in the same run.  Needs a GPU; there is no CPU path.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from flowtron_b200.flowtron import Attention  # noqa: E402
from oracle import flowtron_oracle as O  # noqa: E402
from bench_waveglow_train import card, timed  # noqa: E402

DQ, E, A, L, T = 1024, 640, 640, 160, 1000


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--batches", type=int, nargs="+", default=[8, 32])
    ap.add_argument("--torch-batch", type=int, default=8)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_attention needs a GPU")
    name, plim = card()
    torch.manual_seed(0)
    m = Attention(n_mel_channels=DQ, n_speaker_dim=E - 512, n_text_channels=512, n_att_channels=A).cuda()
    W = dict(m.state_dict())

    def report(variant, direction, B, ms):
        print(json.dumps(dict(variant=variant, direction=direction, B=B, T=T, L=L, Dq=DQ, E=E, A=A,
                              ms_per_call=[round(x, 3) for x in ms], card=name, power_limit_w=plim)), flush=True)

    def inputs(B):
        g = torch.Generator(device="cuda").manual_seed(B)
        q = torch.randn(T, B, DQ, generator=g, device="cuda", requires_grad=True)
        k = torch.randn(L, B, E, generator=g, device="cuda", requires_grad=True)
        lens = torch.randint(L // 2, L + 1, (B,), generator=g, device="cuda")
        lens[0] = L
        mask = ~(torch.arange(L, device="cuda")[None, :] < lens[:, None])[..., None]
        gs = [torch.randn(s, generator=g, device="cuda") for s in ((B, A, T), (B, T, L), (B, T, L))]
        return q, k, lens.to(torch.int32), mask, gs

    for B in args.batches:
        q, k, lens, _, gs = inputs(B)

        def fwd():
            with torch.no_grad():
                m(q, k, k, in_lens=lens)

        def fwd_bwd():
            out = m(q, k, k, in_lens=lens)
            torch.autograd.backward(out, gs)

        report("kernels", "forward", B, timed(fwd, args.warmup, args.steps, args.runs))
        report("kernels", "forward+backward", B, timed(fwd_bwd, args.warmup, args.steps, args.runs))
        del q, k, gs
        torch.cuda.empty_cache()

    B = args.torch_batch
    q, k, _, mask, gs = inputs(B)
    Wt = {f"att.{n}": p.detach().requires_grad_() for n, p in W.items()}
    for autocast in (False, True):
        variant = "torch_autocast_fp16" if autocast else "torch_fp32"

        def ref_fwd():
            with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16, enabled=autocast):
                O.attention_forward(Wt, "att", q, k, mask, None)

        def ref_fwd_bwd():
            with torch.autocast("cuda", dtype=torch.float16, enabled=autocast):
                out = O.attention_forward(Wt, "att", q, k, mask, None)
            torch.autograd.backward([o.float() for o in out], gs)

        report(variant, "forward", B, timed(ref_fwd, args.warmup, args.steps, args.runs))
        report(variant, "forward+backward", B, timed(ref_fwd_bwd, args.warmup, args.steps, args.runs))


if __name__ == "__main__":
    main()
