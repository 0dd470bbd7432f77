"""fp64 oracle of a padded Flowtron training batch, run one utterance at a time (TEST INFRASTRUCTURE).

With ``n_components = 0`` every output row of Flowtron.forward depends on its own utterance only, and FlowtronLoss (+ the
attention-CTC loss) is a sum of per-row terms under batch-wide normalisers.  So the batch's outputs, losses and parameter
gradients are exactly those of B separate ``O.flowtron_forward`` calls on each row's unpadded inputs, each row's loss term
scaled by the batch's normalisers, and the gradients summed over rows:

    nll  = sum_b (sum z_b^2 / (2 sigma^2) - sum_flows sum log_s_b) / (N M)        N = sum of out_lens over the batch
    gate = sum_b sum BCE(gate_b, gate_target_b) / N
    ctc  = w * sum_b sum_flows ctc_{f,b} / (B n_flows)

Run this way the oracle's attention holds a [1, T_b, L_b, A] fp64 tensor per flow instead of [B, T, L, A] (26 GB at
B = 32, T = 1000, L = 160, A = 640), so the fp64 oracle of a full-size training batch fits beside the product on one GPU.
Each row's graph is freed before the next row starts.  tests/test_train_step_oracle_host.py pins this against one batched
oracle call; tests/test_gpu_train_step_oracle.py compares the CUDA training step with it."""
from __future__ import annotations

import time
from typing import Dict, Iterable, Optional

import torch
import torch.nn.functional as F

from oracle import flowtron_oracle as O

Tensor = torch.Tensor


def _row(leaves: Dict[str, Tensor], batch: dict, b: int, dev):
    """Row b of the padded batch through ``O.flowtron_forward`` (B = 1, the explicit LSTM loop: it has an fp64 backward on
    every device) on its own valid region."""
    t_b, l_b = int(batch["out_lens"][b]), int(batch["in_lens"][b])
    f64 = lambda t: t.to(dev, torch.float64)
    prior = batch.get("attn_prior")
    prior = None if prior is None else f64(prior[b:b + 1, :t_b, :l_b])
    in_lens, out_lens = torch.tensor([l_b], device=dev), torch.tensor([t_b], device=dev)
    out = O.flowtron_forward(leaves, f64(batch["mel"][b:b + 1, :, :t_b]), batch["speaker_ids"][b:b + 1].to(dev),
                             batch["text"][b:b + 1, :l_b].to(dev), in_lens, out_lens, prior)
    return out, t_b, l_b


def train_step_oracle(params: Dict[str, Tensor], batch: dict, sigma: float = 1.0, gate_loss: bool = True,
                      ctc_weight: float = 0.0, rows: Optional[Iterable[int]] = None, row_frames: bool = False) -> dict:
    """The fp64 forward outputs, losses and parameter gradients of a padded ``synth_batch``-style batch.

    params: {state_dict key: tensor}, cast to fp64 on their own device (where the oracle runs).  batch: mel [B, M, T],
    speaker_ids [B], text [B, L], in_lens [B], out_lens [B], gate_target [B, T] and attn_prior [B, T, L] or None.
    ctc_weight > 0 adds ``ctc_weight`` times the attention-CTC loss of every flow; it is evaluated on a CPU copy of each
    row's attn_logprob (the oracle builds its CTC targets on the CPU) and autograd carries its gradient back.

    ``rows`` restricts the sum to some rows (the normalisers stay the whole batch's), which gives one row's contribution;
    ``row_frames`` normalises each row by its own frame count instead of the batch's.  Only tests that show the
    comparison can tell these apart use the last two.

    Returns {"rows": {b: {"z": [T_b, M], "log_s": [[T_b, M]] per flow, "gate": [T_b] or None, "attn": [[T_b, L_b]] per
    flow, "attn_logprob": [[T_b, L_b]] per flow}}, "nll", "gate", "ctc": floats, "grads": {key: fp64 gradient of
    nll + gate + ctc}, "seconds": wall time}.  Back-step flows' log_s, attn and attn_logprob (and the last flow's gate) are
    in the flow's flipped time, as Flowtron.forward returns them; z is in natural time."""
    t0 = time.perf_counter()
    leaves = {k: v.detach().to(torch.float64).requires_grad_(True) for k, v in params.items()}
    dev = next(iter(leaves.values())).device
    keys = list(leaves)
    grads = {k: torch.zeros_like(v) for k, v in leaves.items()}
    B = int(batch["out_lens"].shape[0])
    N = float(batch["out_lens"].sum())
    totals = {"nll": 0.0, "gate": 0.0, "ctc": 0.0}
    outs = {}
    for b in (range(B) if rows is None else rows):
        out, t_b, l_b = _row(leaves, batch, b, dev)
        z, log_s, gate, attns, lps = out[:5]
        n = float(t_b) if row_frames else N
        M = z.shape[2]
        terms = {"nll": ((z * z).sum() / (2 * sigma * sigma) - sum(ls.sum() for ls in log_s)) / (n * M)}
        if gate_loss and gate is not None:
            target = batch["gate_target"][b, :t_b].to(dev, torch.float64)
            terms["gate"] = F.binary_cross_entropy_with_logits(gate[:, 0, 0], target, reduction="sum") / n
        if ctc_weight:
            lens = (torch.tensor([l_b]), torch.tensor([t_b]))
            ctc = O.flowtron_ctc_loss((None,) * 4 + ([lp.cpu() for lp in lps],), *lens)       # sum_flows ctc_{f,b} / n_flows
            terms["ctc"] = ctc_weight * ctc.to(dev) / B
        loss = sum(terms.values())
        gs = torch.autograd.grad(loss, [leaves[k] for k in keys], allow_unused=True)
        with torch.no_grad():
            for k, g in zip(keys, gs):
                if g is not None:
                    grads[k] += g
        for k, v in terms.items():
            totals[k] += float(v.detach())
        outs[b] = {"z": z.detach()[:, 0], "log_s": [ls.detach()[:, 0] for ls in log_s],
                   "gate": None if gate is None else gate.detach()[:, 0, 0],
                   "attn": [a.detach()[0] for a in attns], "attn_logprob": [lp.detach()[0] for lp in lps]}
        del out, z, log_s, gate, attns, lps, terms, loss, gs
    if dev.type == "cuda":
        torch.cuda.synchronize(dev)
    return {"rows": outs, **totals, "grads": grads, "seconds": time.perf_counter() - t0}
