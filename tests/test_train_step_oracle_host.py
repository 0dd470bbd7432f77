"""CPU: the per-utterance training-step oracle (tests/train_step_oracle.py) equals one batched oracle call.

On a small ragged batch in fp64 (2 flows, prior, gate and attention-CTC losses), running each utterance alone as a B = 1
``O.flowtron_forward`` with its loss term under the batch's normalisers gives the batched ``O.flowtron_forward`` +
``O.flowtron_loss`` + ``O.flowtron_ctc_loss``: forward outputs on each row's valid positions, the three losses and every
parameter gradient, to 1e-10.  A B = 1 call takes the encoder's unmasked instance norm and the batched call its masked one,
so this also pins that the two agree on a row's valid keys, down to a one-token text.  The same comparison fails when a row is normalised by its own
frame count or when one row's contribution is left out, so tests/test_gpu_train_step_oracle.py can rely on it."""
import torch

from flowtron_b200 import synth
from oracle import flowtron_oracle as O
from train_step_oracle import train_step_oracle

CFG = dict(synth.DEFAULT_MODEL_CONFIG, n_speakers=3, n_text=20, n_hidden=16, n_attn_channels=8, n_mel_channels=4,
           n_text_dim=8, n_speaker_dim=4, n_flows=2)
B, T, L = 3, 24, 8
OUT_LENS, IN_LENS = [13, 24, 4], [8, 6, 1]      # the longest text is not the longest utterance; the last row is short
CTC_WEIGHT = 0.1
TOL = 1e-10


def _setup():
    params = synth.synth_params(CFG, 7, dtype=torch.float64)
    batch = synth.synth_batch(B, T, L, CFG, 7, out_lens=OUT_LENS, in_lens=IN_LENS, with_prior=True)
    batch["speaker_ids"] = torch.tensor([2, 0, 2])
    return params, batch


def _batched(params, batch):
    leaves = {k: v.clone().requires_grad_(True) for k, v in params.items()}
    prior = batch["attn_prior"].double()
    out = O.flowtron_forward(leaves, batch["mel"].double(), batch["speaker_ids"], batch["text"], batch["in_lens"],
                             batch["out_lens"], prior)
    nll, gate = O.flowtron_loss(out, batch["gate_target"].double(), batch["in_lens"], batch["out_lens"])
    ctc = CTC_WEIGHT * O.flowtron_ctc_loss(out, batch["in_lens"], batch["out_lens"])
    grads = torch.autograd.grad(nll + gate + ctc, list(leaves.values()))
    return out, {"nll": float(nll.detach()), "gate": float(gate.detach()), "ctc": float(ctc.detach())}, dict(zip(leaves, grads))


def _errors(ref, bat_out, bat_loss, bat_grads, batch):
    """Worst relative error of the per-utterance oracle `ref` against the batched call: outputs per row on its valid
    region (relative to the row's max |value|), each loss, each parameter gradient (relative L2, floor 1e-6 of the
    largest gradient norm: the conv biases that feed an instance norm have a gradient of rounding size)."""
    z, log_s, gate, attns, lps = bat_out[:5]
    err = {"outputs": 0.0}
    for b in range(B):
        t, l = int(batch["out_lens"][b]), int(batch["in_lens"][b])
        if b not in ref["rows"]:
            err["outputs"] = float("inf")
            continue
        r = ref["rows"][b]
        pairs = [(r["z"], z[:t, b]), (r["gate"], gate[:t, b, 0])]
        for f in range(CFG["n_flows"]):
            pairs += [(r["log_s"][f], log_s[f][:t, b]), (r["attn"][f], attns[f][b, :t, :l]),
                      (r["attn_logprob"][f], lps[f][b, :t, :l])]
        for u, v in pairs:
            assert u.dtype == torch.float64 and u.shape == v.shape
            err["outputs"] = max(err["outputs"], float((u - v).abs().max()) / max(float(v.abs().max()), 1e-300))
    for k, v in bat_loss.items():
        err[k] = abs(ref[k] - v) / abs(v)
    gmax = max(float(g.norm()) for g in bat_grads.values())
    err["grads"] = max(float((ref["grads"][k] - g).norm()) / (float(g.norm()) + 1e-6 * gmax) for k, g in bat_grads.items())
    return err


def test_per_utterance_oracle_equals_batched_oracle():
    params, batch = _setup()
    bat = _batched(params, batch)
    assert all(v > 0 for v in bat[1].values()), bat[1]          # every loss term takes part
    ref = train_step_oracle(params, batch, ctc_weight=CTC_WEIGHT)
    assert set(ref["grads"]) == set(params) and all(g.dtype == torch.float64 for g in ref["grads"].values())
    err = _errors(ref, *bat, batch)
    assert all(v <= TOL for v in err.values()), err


def test_comparison_sees_row_normalisers_and_dropped_rows():
    params, batch = _setup()
    bat = _batched(params, batch)
    own_n = _errors(train_step_oracle(params, batch, ctc_weight=CTC_WEIGHT, row_frames=True), *bat, batch)
    assert own_n["nll"] > 1e-3 and own_n["gate"] > 1e-3 and own_n["grads"] > 1e-3, own_n
    short = int(batch["out_lens"].argmin())
    dropped = _errors(train_step_oracle(params, batch, ctc_weight=CTC_WEIGHT, rows=[b for b in range(B) if b != short]),
                      *bat, batch)
    assert all(dropped[k] > 1e-3 for k in ("nll", "gate", "ctc", "grads")), dropped
    assert dropped["outputs"] == float("inf")
