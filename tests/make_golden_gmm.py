#!/usr/bin/env python
"""Generate tests/golden/gmm_*.npz by running the UNMODIFIED reference Flowtron with the Gaussian-mixture prior
(n_components > 1) and FlowtronLoss(gm_loss=True) on CPU fp32 in eval mode (no dropout).  Writes these new files only.

Run where the reference tree exists (its directory in the FLOWTRON_REFERENCE environment variable):
    python tests/make_golden_gmm.py

The reference zeroes padded mel frames in place (flowtron.py:428), so it is handed a copy.  For B > 1 the same in-place
masked_fill_ also hits the first block's output before the second convolution; in eval mode F.dropout returns its input, so
that output is the relu result autograd saved and the reference's backward raises.  The reference module is therefore given
a functional namespace whose eval-mode dropout returns a copy (the same values); nothing else changes.  Weights come from
flowtron_b200.synth.synth_gmm_params(cfg, SEED).  Stored per case: the inputs, the mel embedding (MelEncoder output),
mean / log_var / prob, the three losses, and for every mel-encoder and mixture parameter, one flow weight and the text
embedding a seeded sample of at most N_SAMPLE gradient elements (flat indices `gidx_<key>`, values `grad_<key>`) plus the
gradient's full L2 norm (`gnorm_<key>`), which keeps each file under 1 MB.
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
N_SAMPLE = 1024
FLOW_KEY = "flows.0.dense_layer.layers.1.linear_layer.weight"

# name: (n_flows, K, fixed_gaussian, mean_scale, out_lens, L, with_prior, ctc, seed)
CASES = {
    "gmm_f2_fixed": (2, 8, True, 3.0, [37, 40, 22, 31, 16], 12, True, True, 41),
    "gmm_f3_learned": (3, 4, False, 0.0, [29, 40, 40, 18, 33], 10, False, False, 42),
    "gmm_b1_learned": (2, 8, False, 0.0, [36], 11, True, True, 43),
    "gmm_b1_fixed": (2, 4, True, 2.0, [33], 9, False, False, 44),
}


def case_config(n_flows, K, fixed, mean_scale):
    return dict(synth.DEFAULT_MODEL_CONFIG, n_flows=n_flows, n_components=K, fixed_gaussian=fixed, mean_scale=mean_scale)


def grad_keys(params):
    return [k for k in params if k.startswith(("mel_encoder.", "gaussian_mixture.")) and k not in
            ("gaussian_mixture.mean", "gaussian_mixture.log_var")] + [FLOW_KEY, "embedding.weight"]


def sample_index(key, numel, seed):
    g = torch.Generator().manual_seed(seed * 7919 + len(key))
    return torch.randperm(numel, generator=g)[:N_SAMPLE].sort().values


class _CopyingDropout:
    """torch.nn.functional with F.dropout(x, p, training=False) returning a copy of x instead of x itself."""

    def __getattr__(self, name):
        return getattr(torch.nn.functional, name)

    @staticmethod
    def dropout(x, p=0.5, training=True, inplace=False):
        assert not training
        return x.clone()


def main():
    from oracle import ref_shims
    assert ref_shims.available(), "the reference tree is needed to generate fixtures"
    torch.set_num_threads(os.cpu_count() or 1)
    F = ref_shims.import_flowtron()
    F.F = _CopyingDropout()
    for name, (n_flows, K, fixed, mean_scale, out_lens, L, with_prior, ctc, seed) in CASES.items():
        cfg = case_config(n_flows, K, fixed, mean_scale)
        params = synth.synth_gmm_params(cfg, seed)
        _, model = ref_shims.reference_model(cfg, params)           # strict load of the synthetic state dict
        B, T = len(out_lens), max(out_lens)
        b = synth.synth_batch(B, T, L, cfg, seed, out_lens=out_lens, with_prior=with_prior, logmel_stats=True)
        # padded frames hold random values: the port must ignore them like the reference's in-place zeroing does
        g = torch.Generator().manual_seed(seed + 1)
        pad = torch.arange(T)[None, None, :] >= b["out_lens"][:, None, None]
        mel = torch.where(pad, torch.randn(B, 80, T, generator=g), b["mel"])
        emb = {}
        model.mel_encoder.register_forward_hook(lambda m, i, o: emb.__setitem__("x", o.detach().clone()))
        crit = F.FlowtronLoss(sigma=1.0, gm_loss=True, gate_loss=True, use_ctc_loss=ctc, ctc_loss_weight=1.0 if ctc else 0.0)
        out = model(mel.clone(), b["speaker_ids"], b["text"], b["in_lens"], b["out_lens"], b["attn_prior"])
        loss, gate_loss, loss_ctc = crit(out, b["gate_target"], b["in_lens"], b["out_lens"])
        (loss + gate_loss + loss_ctc).sum().backward()
        named = dict(model.named_parameters())
        rec = dict(seed=seed, n_flows=n_flows, K=K, fixed_gaussian=int(fixed), mean_scale=np.float32(mean_scale),
                   with_prior=int(with_prior), ctc=int(ctc), mel=mel.numpy(), speaker_ids=b["speaker_ids"].numpy(),
                   text=b["text"].numpy(), in_lens=b["in_lens"].numpy(), out_lens=b["out_lens"].numpy(),
                   gate_target=b["gate_target"].numpy(), mel_embedding=emb["x"].numpy(),
                   mean=out[5].detach().numpy(), log_var=out[6].detach().numpy(), prob=out[7].detach().numpy(),
                   loss=np.float32(loss.item()), gate_loss=np.float32(gate_loss.item()), loss_ctc=np.float32(loss_ctc.item()),
                   state_keys=np.array(list(model.state_dict().keys())))
        if with_prior:
            rec["attn_prior"] = b["attn_prior"].numpy()
        if fixed:
            rec["fixed_mean"] = params["gaussian_mixture.mean"].numpy()
        for k in grad_keys(params):
            gr = named[k].grad.reshape(-1)
            idx = sample_index(k, gr.numel(), seed)
            rec[f"gidx_{k}"] = idx.numpy().astype(np.int32)
            rec[f"grad_{k}"] = gr[idx].numpy()
            rec[f"gnorm_{k}"] = np.float32(gr.norm().item())
        path = os.path.join(OUT, name + ".npz")
        np.savez_compressed(path, **rec)
        print(f"{name}: B {B} T {T} L {L} K {K} fixed {fixed}; loss {loss.item():.6f} gate {gate_loss.item():.6f} "
              f"ctc {loss_ctc.item():.6f}; {os.path.getsize(path) / 1e6:.2f} MB")


if __name__ == "__main__":
    main()
