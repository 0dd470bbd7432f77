#!/usr/bin/env python
"""Generate tests/golden/{train,infer}_long*.npz: texts longer than 256 tokens (up to the kernels' 1024), by running the
UNMODIFIED reference on CPU fp32 through oracle/ref_shims with flowtron_b200.synth.synth_params weights.  Writes these new
files only; the other fixtures are left as they are.

Run where the reference tree exists (FLOWTRON_REFERENCE, default /root/reference):
    python tests/make_golden_long_text.py
Cases (all 2 flows):
  * train_long400:  B = 2, T = 420, L = 400, in_lens [400, 290], prior + CTC weight 1.0.  T >= 320 runs the attention /
    attention-LSTM overlap of the training step, and every utterance has at least as many frames as tokens, so its CTC
    loss is finite (2L + 1 = 801 states: the several-states-per-thread CTC kernel).  To keep the file small, z, log_s,
    gate and one utterance's attention are stored at every 6th frame (`t_stride` in the file); losses and
    gradients are stored in full.
  * train_long1024: B = 2, T = 40, L = 1024, in_lens [1024, 700], prior + CTC weight 1.0: the global-memory attention
    variant (L > 672).  Fewer frames than tokens: the CTC losses are infinite and zeroed (zero_infinity), as in the
    reference.  Both utterances' attention and attention log-probabilities are stored, at every other frame.
The reference's FlowtronLoss rolls a back step's attn_logprob by -out_lens[b] in time, in place, when the CTC loss is on, and
restores only a flipped copy (flowtron.py:249-269); the files hold attn_logprob as the flows returned it (rolled back).
  * infer_long1024: B = 1, T = 48, L = 1024, gate off (bias -10).
  * infer_long600gate: B = 1, T = 48, L = 600, gate bias chosen so that the gate stops generation before T.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import ref_shims  # noqa: E402
import make_golden  # noqa: E402

def subsample_frames(tag, stride):
    """Keep every stride-th frame of the per-frame outputs of train_{tag}.npz (written by make_golden.train_case): z, gate,
    log_s_i, attn_i_b0 ([T, ...]) and attn_i, attn_logprob_i ([B, T, L]); undo FlowtronLoss's roll of the back steps'
    attn_logprob first."""
    path = os.path.join(make_golden.OUT, f"train_{tag}.npz")
    rec = dict(np.load(path))
    if float(rec["ctc_weight"]) > 0:
        for k in [k for k in rec if k.startswith("attn_logprob_") and int(k.rsplit("_", 1)[1]) % 2 == 1]:
            rec[k] = np.stack([np.roll(rec[k][b], int(n), axis=0) for b, n in enumerate(rec["out_lens"])])
    for k in list(rec):
        if k in ("z", "gate") or k.startswith("log_s_") or (k.startswith("attn_") and k.endswith("_b0")):
            rec[k] = np.ascontiguousarray(rec[k][::stride])
        elif k.startswith("attn_"):
            rec[k] = np.ascontiguousarray(rec[k][:, ::stride])
    rec["t_stride"] = np.int64(stride)
    np.savez_compressed(path, **rec)


def main():
    assert ref_shims.available(), "needs the reference tree"
    torch.manual_seed(0)
    torch.set_num_threads(8)
    which = sys.argv[1:] or ["train400", "train1024", "infer1024", "infer600"]
    if "train400" in which:
        make_golden.train_case("long400", n_flows=2, B=2, T=420, L=400, out_lens=[420, 330], in_lens=[400, 290],
                               with_prior=True, seed=4400, store_attn=False, ctc_weight=1.0)
        subsample_frames("long400", 6)
    if "train1024" in which:
        make_golden.train_case("long1024", n_flows=2, B=2, T=40, L=1024, out_lens=[40, 31], in_lens=[1024, 700],
                               with_prior=True, seed=4401, ctc_weight=1.0)
        subsample_frames("long1024", 2)
    if "infer1024" in which:
        make_golden.infer_case("long1024", n_flows=2, B=1, T=48, L=1024, seed=4402, gate_bias=-10.0)
    if "infer600" in which:
        make_golden.infer_case("long600gate", n_flows=2, B=1, T=48, L=600, seed=4403, gate_bias=0.25)


if __name__ == "__main__":
    main()
