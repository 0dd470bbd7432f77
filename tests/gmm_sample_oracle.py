"""fp64 restatement of the Gaussian-mixture synthesis path: Flowtron.mixture (the oracle's MelEncoder + GaussianMixture per
utterance), the mixture sampler of csrc/gmm_sample.cu (its counter hash, component choice and Box-Muller draw) and the
component responsibilities.  numpy / torch on the CPU only."""
from __future__ import annotations

import numpy as np
import torch

from oracle import flowtron_oracle as FO

_GOLDEN_GAMMA = np.uint64(0x9E3779B97F4A7C15)
_IDX_MUL = np.uint64(0xD1B54A32D192ED03)
_MIX1 = np.uint64(0xBF58476D1CE4E5B9)
_MIX2 = np.uint64(0x94D049BB133111EB)


def hash3(seed, ctr, idx):
    """The dropout masks' and the sampler's counter hash (splitmix64 finaliser over (seed, counter, element)) -> uint32."""
    with np.errstate(over="ignore"):
        z = np.uint64(seed) + _GOLDEN_GAMMA * (np.uint64(ctr) + np.uint64(1)) + np.asarray(idx, dtype=np.uint64) * _IDX_MUL
        z = (z ^ (z >> np.uint64(30))) * _MIX1
        z = (z ^ (z >> np.uint64(27))) * _MIX2
        return ((z ^ (z >> np.uint64(31))) >> np.uint64(32)).astype(np.uint32)


def sample(mean, log_var, prob, n_frames, T, sigma, seed, counter, component=None):
    """The sampler's draw for state {seed, counter} -> (z [B, M, T] float64, k [B, M, T] int64, -1 past n_frames).

    The component choice is restated exactly (the fp32 running sum of prob[b] in component order, the fp32 product
    u * total); the Gaussian draw in float64 from the same uniforms."""
    mean, log_var, prob = (np.asarray(t, dtype=np.float32) for t in (mean, log_var, prob))
    B, K = prob.shape
    M = mean.shape[1]
    z = np.zeros((B, M, T))
    ks = np.full((B, M, T), -1, dtype=np.int64)
    base = np.uint64(counter) * np.uint64(4)
    for b in range(B):
        n = min(int(n_frames[b]), T)
        if n <= 0:
            continue
        mb, lb = mean[b if mean.shape[0] > 1 else 0], log_var[b if log_var.shape[0] > 1 else 0]
        c, t = np.meshgrid(np.arange(M, dtype=np.uint64), np.arange(n, dtype=np.uint64), indexing="ij")
        idx = ((np.uint64(b * M) + c) << np.uint64(32)) | t
        forced = -1 if component is None else int(component[b])
        if 0 <= forced < K:
            k = np.full((M, n), forced, dtype=np.int64)
        else:
            cdf = np.cumsum(prob[b], dtype=np.float32)
            pos = np.nonzero(prob[b] > 0)[0]
            last = int(pos[-1]) if pos.size else 0
            x = (hash3(seed, base, idx) >> np.uint32(8)).astype(np.float32) * np.float32(2.0 ** -24) * cdf[-1]
            hit = x[..., None] < cdf                                   # [M, n, K]
            k = np.where(hit.any(-1), hit.argmax(-1), last)
        u1 = ((hash3(seed, base + np.uint64(1), idx) >> np.uint32(8)).astype(np.float64) + 1.0) * 2.0 ** -24
        u2 = (hash3(seed, base + np.uint64(2), idx) >> np.uint32(8)).astype(np.float64) * 2.0 ** -24
        eps = np.sqrt(-2.0 * np.log(u1)) * np.cos(2.0 * np.pi * u2)
        rows = np.arange(M)[:, None]
        mu = mb.astype(np.float64)[rows, k]
        sd = np.exp(0.5 * lb.astype(np.float64)[rows, k])
        z[b, :, :n] = mu + sigma * sd * eps
        ks[b, :, :n] = k
    return z, ks


def responsibilities(z, out_lens, mean, log_var, prob):
    """z [B, M, T] -> (r [B, K], lse [B]): r[b, k] = the mean over t < out_lens[b] and all channels of the posterior
    prob_k N_k / sum_j prob_j N_j; lse[b] = the sum over the same elements of the oracle's mixture log-density, the term
    whose negative FlowtronLoss(gm_loss=True) sums."""
    z, mean, log_var, prob = (torch.as_tensor(np.asarray(t, dtype=np.float64)) for t in (z, mean, log_var, prob))
    z = z.permute(2, 0, 1)                                                              # [T, B, M], the flows' layout
    valid = FO.get_mask_from_lengths(torch.as_tensor(np.asarray(out_lens)), z.shape[0]).t()[..., None]   # [T, B, 1]
    post = torch.softmax(FO.mixture_log_terms(z, mean, log_var, prob), dim=3)                  # [T, B, M, K]
    r = torch.where(valid[..., None], post, 0.0).sum((0, 2)) / (valid.sum((0, 2)) * z.shape[2])[:, None]
    lse = torch.where(valid, FO.mixture_log_density(z, mean, log_var, prob), 0.0).sum((0, 2))
    return r.numpy(), lse.numpy()


def mixture(params, mel, out_lens, n_components, fixed_gaussian):
    """Flowtron.mixture restated: row b is the oracle's MelEncoder on mel[b, :, :out_lens[b]] alone, then its
    GaussianMixture -> (emb [B, 512], mean, log_var, prob) float64; mean / log_var [B, 80, K], or the fixed [1, 80, K]
    buffers."""
    p = {k: v.double() for k, v in params.items() if k.startswith(("mel_encoder.", "gaussian_mixture."))}
    mel = torch.as_tensor(mel).double()
    with torch.no_grad():
        emb = torch.cat([FO.mel_encoder_forward(p, mel[b:b + 1, :, :int(n)], torch.tensor([int(n)]))
                         for b, n in enumerate(out_lens)])
        return (emb, *FO.gaussian_mixture(p, emb, n_components, fixed_gaussian))
