#!/usr/bin/env python
"""Generate tests/golden/score_*.npz: per-utterance FlowtronLoss terms (what Flowtron.score returns) from the UNMODIFIED
reference on CPU fp32, in eval mode without autograd.  Writes these files only.

Run where the reference tree exists (its directory in the FLOWTRON_REFERENCE environment variable):
    python tests/make_golden_score.py

For row b the reference's FlowtronLoss is applied to that row alone: z, log_s, gate and attn_logprob cut to its own
out_lens[b] frames and 1-row lengths.  Its `loss` and `gate_loss` are the row's `nll` and `gate`; flow f's `ctc` is the
reference's AttentionCTCLoss on flow f's attn_logprob, put back in natural time first for a back step (FlowtronLoss's
in-place roll by -out_lens[b] and flip, which for one row cut to its length is the flip alone).

Cases (weights from flowtron_b200.synth; every flow's conv layer non-zero; gate, attention prior and CTC on):
  * score_f2 / score_f3: 2 and 3 flows, 7 ragged rows, each run as its own B = 1 forward on its unpadded inputs (the
    loop Flowtron.score replaces).
  * score_gmm_learned / score_gmm_fixed: n_components > 1 with learned / fixed Gaussians, 6 rows run as ONE padded batch:
    the MelEncoder averages over the padded length, so mixture rows are defined by the batch they come in.
  * score_l1024: one row of 1024 tokens and 1040 frames (2 flows).
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from flowtron_b200 import synth  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")

# name: (n_flows, out_lens, in_lens, L, K, fixed_gaussian, mean_scale, seed, per_utterance)
CASES = {
    "score_f2": (2, [96, 41, 70, 23, 88, 57, 64], [24, 9, 20, 30, 17, 12, 24], 30, 0, True, 0.0, 5101, True),
    "score_f3": (3, [60, 33, 52, 80, 19, 47, 71], [14, 20, 11, 22, 6, 17, 9], 22, 0, True, 0.0, 5102, True),
    "score_gmm_learned": (2, [44, 30, 51, 18, 37, 26], [12, 9, 14, 6, 10, 11], 14, 4, False, 0.0, 5103, False),
    "score_gmm_fixed": (3, [35, 48, 22, 40, 29, 31], [8, 13, 7, 12, 10, 9], 13, 8, True, 3.0, 5104, False),
    "score_l1024": (2, [1040], [1024], 1024, 0, True, 0.0, 5105, True),
}


def row_losses(F, out, b, in_lens, out_lens, gate_target, gm):
    """The reference's FlowtronLoss / AttentionCTCLoss on row b of a forward output, cut to its own length."""
    z, log_s_list, gate, attns, lps, mean, log_var, prob = out
    n = int(out_lens[b])
    il, ol = in_lens[b:b + 1], out_lens[b:b + 1]
    cut = lambda t: t[:n, b:b + 1]
    row = (cut(z), [cut(ls) for ls in log_s_list], cut(gate), [a[b:b + 1, :n] for a in attns], [lp[b:b + 1, :n] for lp in lps],
           None if mean is None else (mean if mean.size(0) == 1 else mean[b:b + 1]),
           None if log_var is None else (log_var if log_var.size(0) == 1 else log_var[b:b + 1]),
           None if prob is None else prob[b:b + 1])
    nll, gate_loss, _ = F.FlowtronLoss(sigma=1.0, gm_loss=gm, gate_loss=True)(row, gate_target[b:b + 1, :n], il, ol)
    ctc_fn = F.AttentionCTCLoss(blank_logprob=-1)
    ctc = []
    for f, lp in enumerate(row[4]):
        lp = torch.flip(lp, (1,)) if f % 2 else lp
        ctc.append(float(ctc_fn(row[3][f].unsqueeze(1), il, ol, attn_logprob=lp.unsqueeze(1))))
    return float(nll), float(gate_loss), ctc


def main():
    from oracle import ref_shims
    assert ref_shims.available(), "the reference tree is needed to generate fixtures"
    torch.set_num_threads(os.cpu_count() or 1)
    which = sys.argv[1:] or list(CASES)
    for name in which:
        n_flows, out_lens, in_lens, L, K, fixed, mean_scale, seed, per_utt = CASES[name]
        cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=n_flows)
        if K > 1:
            cfg.update(n_components=K, fixed_gaussian=fixed, mean_scale=mean_scale)
            params = synth.synth_gmm_params(cfg, seed)
        else:
            params = synth.synth_params(cfg, seed)
        F, model = ref_shims.reference_model(cfg, params)
        B, T = len(out_lens), max(out_lens)
        bt = synth.synth_batch(B, T, L, cfg, seed, out_lens=out_lens, in_lens=in_lens, with_prior=True, logmel_stats=True)
        il_all, ol_all = bt["in_lens"], bt["out_lens"]
        nll, gate, ctc = np.zeros(B, np.float32), np.zeros(B, np.float32), np.zeros((n_flows, B), np.float32)
        with torch.no_grad():
            if per_utt:
                for b in range(B):
                    n, nl = int(ol_all[b]), int(il_all[b])
                    out = model(bt["mel"][b:b + 1, :, :n].clone(), bt["speaker_ids"][b:b + 1], bt["text"][b:b + 1, :nl],
                                il_all[b:b + 1], ol_all[b:b + 1], bt["attn_prior"][b:b + 1, :n, :nl].clone())
                    nll[b], gate[b], ctc[:, b] = row_losses(F, out, 0, il_all[b:b + 1], ol_all[b:b + 1],
                                                            bt["gate_target"][b:b + 1], False)
            else:
                out = model(bt["mel"].clone(), bt["speaker_ids"], bt["text"], il_all, ol_all, bt["attn_prior"].clone())
                for b in range(B):
                    nll[b], gate[b], ctc[:, b] = row_losses(F, out, b, il_all, ol_all, bt["gate_target"], True)
        rec = dict(seed=seed, n_flows=n_flows, K=K, fixed_gaussian=int(fixed), mean_scale=np.float32(mean_scale),
                   mel=bt["mel"].numpy(), speaker_ids=bt["speaker_ids"].numpy(), text=bt["text"].numpy(),
                   in_lens=il_all.numpy(), out_lens=ol_all.numpy(), nll=nll, gate=gate, ctc=ctc)
        if bt["attn_prior"].numel() <= 1 << 20:     # larger priors are rebuilt by the test (synth.beta_binomial_prior)
            rec["attn_prior"] = bt["attn_prior"].numpy()
        path = os.path.join(OUT, name + ".npz")
        np.savez_compressed(path, **rec)
        print(f"{name}: B {B} T {T} L {L}; nll {nll.round(4).tolist()} gate {gate.round(4).tolist()} "
              f"ctc {ctc.round(3).tolist()}; {os.path.getsize(path) / 1e6:.2f} MB")


if __name__ == "__main__":
    main()
