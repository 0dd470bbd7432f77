#!/usr/bin/env python
"""Generate tests/golden/gmm_sample_*.npz by running the UNMODIFIED reference MelEncoder + GaussianMixture one utterance at a
time on CPU fp32 in eval mode, and the reference FlowtronLoss(gm_loss=True) on a drawn z under the resulting mixtures.
Writes these new files only.

Run where the reference tree exists (its directory in the FLOWTRON_REFERENCE environment variable):
    python tests/make_golden_gmm_sample.py

Weights come from flowtron_b200.synth.synth_gmm_params(cfg, SEED).  Each utterance is handed to the reference as
mel[b:b+1, :, :out_lens[b]] (a copy: the reference zeroes padded frames in place), which is what Flowtron.mixture's row b
must equal.  Stored per case: the padded mel (random values past each length) and its lengths, the per-utterance
embedding, mean / log_var / prob (the fixed buffers once for a fixed-Gaussian model), a z [B, 80, T] and the reference
loss of that z with every log_s zero and no gate or CTC term: -sum_valid logsumexp / (n_valid * 80).
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

# name: (K, fixed_gaussian, mean_scale, out_lens, seed)
CASES = {
    "gmm_sample_learned": (4, False, 0.0, [41, 17, 60, 8], 51),
    "gmm_sample_fixed": (8, True, 3.0, [23, 55, 9], 52),
}


def case_config(K, fixed, mean_scale):
    return dict(synth.DEFAULT_MODEL_CONFIG, n_flows=2, n_components=K, fixed_gaussian=fixed, mean_scale=mean_scale)


def main():
    from oracle import ref_shims
    assert ref_shims.available(), "the reference tree is needed to generate fixtures"
    torch.set_num_threads(os.cpu_count() or 1)
    F = ref_shims.import_flowtron()
    for name, (K, fixed, mean_scale, out_lens, seed) in CASES.items():
        cfg = case_config(K, fixed, mean_scale)
        params = synth.synth_gmm_params(cfg, seed)
        _, model = ref_shims.reference_model(cfg, params)
        B, T = len(out_lens), max(out_lens)
        b = synth.synth_batch(B, T, 8, cfg, seed, out_lens=out_lens, logmel_stats=True)
        out_lens = b["out_lens"].tolist()                     # the batch's own row order
        g = torch.Generator().manual_seed(seed + 1)
        pad = torch.arange(T)[None, None, :] >= b["out_lens"][:, None, None]
        mel = torch.where(pad, torch.randn(B, 80, T, generator=g), b["mel"])
        embs, means, log_vars, probs = [], [], [], []
        with torch.no_grad():
            for i, n in enumerate(out_lens):
                e = model.mel_encoder(mel[i:i + 1, :, :n].clone(), torch.tensor([n]))
                mean, log_var, prob = model.gaussian_mixture(e, 1)
                embs.append(e)
                means.append(mean)
                log_vars.append(log_var)
                probs.append(prob)
            emb, prob = torch.cat(embs), torch.cat(probs)
            mean, log_var = (means[0], log_vars[0]) if fixed else (torch.cat(means), torch.cat(log_vars))
            z = torch.randn(B, 80, T, generator=g) * 2.0
            zt = z.permute(2, 0, 1).contiguous()
            crit = F.FlowtronLoss(sigma=1.0, gm_loss=True, gate_loss=False)
            out = (zt, [torch.zeros_like(zt)], None, [], [], mean, log_var, prob)
            loss = crit(out, None, torch.ones(B, dtype=torch.long), b["out_lens"])[0]
        rec = dict(seed=seed, K=K, fixed_gaussian=int(fixed), mean_scale=np.float32(mean_scale), mel=mel.numpy(),
                   out_lens=b["out_lens"].numpy(), mel_embedding=emb.numpy(), mean=mean.numpy(), log_var=log_var.numpy(),
                   prob=prob.numpy(), z=z.numpy(), loss=np.float32(loss.item()))
        path = os.path.join(OUT, name + ".npz")
        np.savez_compressed(path, **rec)
        print(f"{name}: B {B} T {T} K {K} fixed {fixed}; loss {loss.item():.6f}; {os.path.getsize(path) / 1e6:.2f} MB")


if __name__ == "__main__":
    main()
