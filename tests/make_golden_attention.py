#!/usr/bin/env python
"""Generate tests/golden/attention_<case>.npz by running the UNMODIFIED reference Attention module (flowtron.py:528-592) on the
CPU in fp32, through oracle/ref_shims, for every case of tests/attention_oracle.CASES.  Writes new files only.

Run where the reference tree exists (FLOWTRON_REFERENCE, default /root/reference):
    python tests/make_golden_attention.py
Each file holds the case's seed-derived input sums (sum/<tensor>) and the reference's output, attn and attn_logprob (absent
when attn is given)."""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import ref_shims  # noqa: E402
import attention_oracle as AO  # noqa: E402


def main():
    F = ref_shims.import_flowtron()
    for name, c in AO.CASES.items():
        Dq, E, A = AO.DIMS[c["dims"]]
        x = AO.case_inputs(c)
        m = F.Attention(n_mel_channels=Dq, n_speaker_dim=E - 512, n_text_channels=512, n_att_channels=A, temperature=c["temp"])
        m.load_state_dict(x["W"], strict=True)
        with torch.no_grad():
            out, attn, lp = m(x["queries"], x["keys"], x["values"], mask=x["mask"], attn=x["attn"], attn_prior=x["prior"])
        rec = dict(AO.input_sums(x), output=out.numpy(), attn=attn.numpy())
        if lp is not None:
            rec["attn_logprob"] = lp.numpy()
        np.savez_compressed(os.path.join(AO.GOLDEN, f"attention_{name}.npz"), **{k: np.asarray(v) for k, v in rec.items()})
        print(name, tuple(out.shape), float(out.abs().max()))


if __name__ == "__main__":
    main()
