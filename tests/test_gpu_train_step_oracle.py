"""GPU: the benchmarked training steps against the fp64 oracle at their own shapes, one utterance at a time.

bench.py times the configs[1] training step (B = 32, T <= 1000, LJS-like lengths, prior on, 2 flows) replayed from one CUDA
graph with the fused clip + RAdam, and the configs[2] step (B = 64, 123 speakers, T <= 860).  Here the product runs those
steps as bench.py sets them up (synth_params(cfg, 1234), synth_batch(..., with_prior=True, logmel_stats=True),
FlowtronLoss(sigma=1, gate_loss=True), train() with the encoder dropout at 0) and every forward output, loss and parameter
gradient is compared with tests/train_step_oracle.py: oracle/flowtron_oracle.py in fp64 on the GPU, one utterance at a
time under the batch's loss normalisers (pinned against one batched oracle call by tests/test_train_step_oracle_host.py).

Cases: `cfg1` is the headline step itself; `cfg2` adds two 32-row flow launches and repeated speaker ids; `edges` (B = 33,
T = 1001, CTC weight 0.1) runs the layer-0/1 pipeline over 10 chunks plus a 1-step tail and the attention LSTM over
3 x 256 + 233 steps, a 1-row launch, row ends on both sides of every 100- and 256-step boundary and of the 320-step
attention-overlap threshold, and one row whose text is longer than its frames (CTC infinite, zeroed).

Checks: each forward output of each row on its own valid region, relative to that row's max |value| (a short row cannot
hide behind a long one), against the north-star 1e-3; nll within 1e-4 relative, gate and CTC within 1e-3; every parameter
gradient's relative L2 and cosine against its own fp64 gradient, no floor, except tensors whose oracle norm is below 1e-6
of the largest (the conv biases that feed an instance norm, analytically ~0), which are held to 1e-4 of the largest norm
in absolute terms.  `cfg1` is also captured and replayed from one CUDA graph as bench.py times it.

Measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit; repeated runs give the same values to 3 digits.  Each
gradient bar is about 3x the worst value measured, and none is looser than the flow-step test's "all" path
(tests/test_gpu_ar_step_backward.py: 1e-2, 1 - 2.1e-5).  The worst tensor is an encoder instance-norm bias in every case.
The flow tensors stay at <= 8.2e-4, as at the flow-step test's small shapes.  "oracle" is the oracle's wall time and
"peak" the test's peak allocated memory, oracle included.

    case    forward worst (output, row out_len)   param rel L2 (bar)     1 - cosine (bar)      oracle   peak
    cfg1    8.33e-4 (log_s_0, 821)               2.41e-3 (7.2e-3)       2.9e-6 (8.7e-6)       84 s     6.2 GiB
    cfg2    7.70e-4 (log_s_1, 703)               1.67e-3 (5.0e-3)       1.4e-6 (4.2e-6)       113 s    9.3 GiB
    edges   8.45e-4 (log_s_0, 200)               2.48e-3 (7.4e-3)       3.1e-6 (9.2e-6)       47 s     7.7 GiB

cfg1 replay: the same gradient errors as the eager step; replay against eager at 0.34 of its bar (3x the spread of three
eager backwards); loss 2.2e-7 relative to the eager loss; clip_grad_norm_'s total norm 1.97e-5 from the oracle's (bar
6e-5).  Losses: nll <= 7.8e-6, gate <= 1.4e-5, CTC 1.6e-7.  The shortest cfg1 row (506 frames) carries about 2.1% of
every flow tensor group's gradient norm (13.6% of the text embedding's), so leaving it out would show as a relative L2 of
about 2e-2, 3x the gradient bar; the per-row forward checks see any row directly.
"""
import math

import pytest
import torch

from conftest import record_parity
from flowtron_b200 import synth
from train_step_oracle import train_step_oracle

pytestmark = pytest.mark.gpu

SEED = 1234
FWD_BAR = 1e-3
GATE_FLOOR = 1.0                # the gate is a logit: below |g| = 1 its check is absolute (see _check_forward)
LOSS_BARS = {"nll": 1e-4, "gate": 1e-3, "ctc": 1e-3}
SMALL = 1e-6                    # oracle norm below SMALL * largest: compared on the absolute scale ...
SMALL_BAR = 1e-4                # ... |g - r| <= SMALL_BAR * largest norm
BARS = {                        # param rel L2, 1 - cosine
    "cfg1": (7.2e-3, 8.7e-6),
    "cfg2": (5.0e-3, 4.2e-6),
    "edges": (7.4e-3, 9.2e-6),
}
NORM_BAR = 6e-5                 # clip_grad_norm_'s device-side total norm against the oracle's fp64 norm

# edges: row ends on both sides of the 100-step layer chunks, the 256-step attention-LSTM chunks and T = 320
EDGE_OUT = [1001, 1000, 901, 900, 800, 769, 768, 767, 700, 640, 600, 513, 512, 511, 400, 321, 320, 319, 300, 257, 256, 255,
            201, 200, 199, 161, 160, 101, 100, 99, 40, 2, 1]


def _edge_lengths():
    out_lens = torch.tensor(EDGE_OUT)
    in_lens = torch.clamp((out_lens.float() / 6.5).round().long(), 1, 160)
    in_lens[out_lens == 1001] = 160
    in_lens[out_lens == 40] = 60                # longer than its 40 frames: the CTC term is infinite and zeroed
    return out_lens, in_lens


def _case(name):
    """cfg, the padded CPU batch and the CTC weight of a case."""
    from bench import train_lengths
    cfg = dict(synth.DEFAULT_MODEL_CONFIG)
    if name == "cfg1":
        T, ctc = 1000, 0.0
        out_lens, in_lens = train_lengths(2, 32, T, SEED)
    elif name == "cfg2":
        T, ctc = 860, 0.0
        cfg["n_speakers"] = 123
        out_lens, in_lens = train_lengths(3, 64, T, SEED)
    else:
        T, ctc = 1001, 0.1
        out_lens, in_lens = _edge_lengths()
    B, L = len(out_lens), int(in_lens.max())
    batch = synth.synth_batch(B, T, L, cfg, SEED, out_lens=out_lens.tolist(), in_lens=in_lens.tolist(), with_prior=True,
                              logmel_stats=True)
    return cfg, batch, ctc


@pytest.fixture(scope="module")
def oracle():
    """The fp64 oracle of each case (cfg, batch, ctc weight, result), computed once for this module."""
    cache = {}

    def get(name):
        if name not in cache:
            cfg, batch, ctc = _case(name)
            params = {k: v.cuda() for k, v in synth.synth_params(cfg, SEED).items()}
            cache[name] = (cfg, batch, ctc, train_step_oracle(params, batch, ctc_weight=ctc))
            record_parity(f"train_oracle_{name}_wall", {"oracle_s": cache[name][3]["seconds"]})
        return cache[name]
    yield get
    cache.clear()
    torch.cuda.empty_cache()


def _model(cfg):
    from flowtron_b200.flowtron import Flowtron
    model = Flowtron(**cfg)
    model.load_state_dict(synth.synth_params(cfg, SEED), strict=True)
    model = model.cuda().train()
    model.encoder.p_dropout = 0.0
    return model


def _fwd_bwd(model, crit, cu, ctc_weight):
    """Forward -> FlowtronLoss -> backward as bench.py's step (plus the weighted CTC term when it is on)."""
    out = model(cu["mel"], cu["speaker_ids"], cu["text"], cu["in_lens"], cu["out_lens"], cu["attn_prior"])
    nll, gl, ctc = crit(out, cu["gate_target"], cu["in_lens"], cu["out_lens"])
    loss = nll + gl
    if ctc_weight:
        loss = loss + ctc_weight * ctc
    loss = loss.sum()
    loss.backward()
    return out, {"nll": nll.detach(), "gate": gl.detach(), "ctc": ctc_weight * ctc.detach()}, loss.detach()


def _crit(ctc_weight):
    from flowtron_b200.flowtron import FlowtronLoss
    return FlowtronLoss(sigma=1.0, gate_loss=True, use_ctc_loss=ctc_weight > 0, ctc_loss_weight=ctc_weight)


def _check_forward(tag, out, ref, batch):
    """Each output of each row against that row's oracle, relative to the row's own max |value| on its valid region.
    Like the other checks, records every error and returns the failures.

    The gate logits of a row are normalised by max(row max |g|, GATE_FLOOR).  They are an fp32 projection of [hA; ctx],
    whose fp16 tensor-core operands leave an absolute error of 2e-4 to 4e-4 logit units in every case (worst: 2.4e-4 cfg1,
    3.8e-4 cfg2, 2.2e-4 edges).  A row whose logits all stay near 0 (cfg2's 180-frame row: |g| <= 0.20) shows that as
    1.9e-3 of its own max, though its sigmoid moves by 1e-4 at most; a row whose gate a bug gets wrong is far above 1e-3
    logit units either way.  The raw per-row figure is recorded as gate_row_relative."""
    z, log_s, gate, attns, lps = out[:5]
    worst, gate_rel = {}, (0.0, -1)
    for b, r in ref["rows"].items():
        t, l = int(batch["out_lens"][b]), int(batch["in_lens"][b])
        pairs = [("z", z[:t, b], r["z"]), ("gate", gate[:t, b, 0], r["gate"])]
        for f in range(len(log_s)):
            pairs += [(f"log_s_{f}", log_s[f][:t, b], r["log_s"][f]), (f"attn_{f}", attns[f][b, :t, :l], r["attn"][f]),
                      (f"attn_logprob_{f}", lps[f][b, :t, :l], r["attn_logprob"][f])]
        for name, o, v in pairs:
            d, vmax = float((o.detach().double() - v).abs().max()), float(v.abs().max())
            e = d / max(vmax, GATE_FLOOR if name == "gate" else 1e-30)
            if name not in worst or e > worst[name][0]:
                worst[name] = (e, b)
            if name == "gate" and d / max(vmax, 1e-30) > gate_rel[0]:
                gate_rel = (d / max(vmax, 1e-30), b, d)
    errs = {k: v[0] for k, v in worst.items()}
    name = max(errs, key=errs.get)
    record_parity(f"{tag}_forward", {**errs, "worst_output": name, "worst_row": worst[name][1],
                                     "worst_row_out_len": int(batch["out_lens"][worst[name][1]]),
                                     "gate_row_relative": gate_rel[0], "gate_row_relative_row": gate_rel[1],
                                     "gate_row_relative_abs": gate_rel[2]})
    return [f"{tag} {k}: {v[0]:.3e} (row {v[1]}, out_len {int(batch['out_lens'][v[1]])})" for k, v in worst.items()
            if not v[0] <= FWD_BAR]


def _check_losses(tag, losses, ref, ctc_weight):
    errs = {k: abs(float(losses[k]) - ref[k]) / abs(ref[k]) for k in LOSS_BARS if k != "ctc" or ctc_weight}
    record_parity(f"{tag}_losses", errs)
    return [f"{tag} {k} loss: {v:.3e}" for k, v in errs.items() if not v <= LOSS_BARS[k]]


def _group(name):
    """Tensor group of a parameter: encoder / embedding / speaker_embedding, or flows.i.<module>."""
    parts = name.replace(".ar_step.", ".").split(".")
    if parts[0] != "flows":
        return parts[0]
    return f"flows.{parts[1]}." + ("dense+conv" if parts[2] in ("dense_layer", "conv") else parts[2])


def _check_grads(tag, grads, ref, bars):
    """Every parameter gradient against its own fp64 oracle gradient: relative L2 and cosine with no floor, or on the
    absolute scale for the analytically ~0 ones."""
    bar_rel, bar_cos = bars
    gmax = max(float(r.norm()) for r in ref.values())
    rows, small = [], []
    for name, g in grads.items():
        assert torch.isfinite(g).all(), (tag, name)
        g64, r = g.reshape(-1).double(), ref[name].reshape(-1)
        rn, dn = float(r.norm()), float((g64 - r).norm())
        if rn < SMALL * gmax:
            small.append((name, dn / gmax))
            continue
        rows.append((name, dn / rn, 1.0 - float(g64 @ r) / (float(g64.norm()) * rn)))
    worst = max(rows, key=lambda x: x[1])
    least = max(rows, key=lambda x: x[2])
    groups = {}
    for name, e, _ in rows:
        groups[_group(name)] = max(groups.get(_group(name), 0.0), e)
    record_parity(tag, {"param_rel_l2": worst[1], "param_rel_l2_tensor": worst[0], "one_minus_cos": least[2],
                        "one_minus_cos_tensor": least[0], "small_abs": max([e for _, e in small], default=0.0),
                        "small_tensors": len(small), **{f"group_{k}": v for k, v in groups.items()}})
    bad = [f"{tag} {n}: rel {e:.3e} 1-cos {c:.3e}" for n, e, c in rows if not (e <= bar_rel and c <= bar_cos)]
    return bad + [f"{tag} {n}: |g - r| = {e:.3e} of the largest norm" for n, e in small if not e <= SMALL_BAR]


@pytest.mark.parametrize("case", ["cfg1", "cfg2", "edges"])
def test_training_step_matches_fp64_oracle(oracle, case):
    """The eager training step of a benchmarked shape: forward outputs per row, losses and every parameter gradient."""
    from flowtron_b200 import _lib
    torch.cuda.reset_peak_memory_stats()
    cfg, batch, ctc_weight, ref = oracle(case)
    model = _model(cfg)
    cu = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in batch.items()}
    out, losses, _ = _fwd_bwd(model, _crit(ctc_weight), cu, ctc_weight)
    torch.cuda.synchronize()
    assert _lib.device_status() == 0
    tag = f"train_oracle_{case}"
    bad = _check_forward(tag, out, ref, batch)
    bad += _check_losses(tag, losses, ref, ctc_weight)
    bad += _check_grads(f"{tag}_grads", {n: p.grad for n, p in model.named_parameters()}, ref["grads"], BARS[case])
    record_parity(f"{tag}_memory", {"peak_gib": torch.cuda.max_memory_allocated() / 2 ** 30})
    if case == "cfg1":
        # what the gradient bars can see: one row's share of each tensor group's gradient (the shortest row's, the one a
        # kernel that drops a row's contribution would hide best); the per-row forward checks see any row directly
        short = int(batch["out_lens"].argmin())
        params = {k: v.cuda() for k, v in synth.synth_params(cfg, SEED).items()}
        one = train_step_oracle(params, batch, rows=[short])["grads"]
        share = {}
        for name, g in one.items():
            k = _group(name)
            a, r = share.get(k, (0.0, 0.0))
            share[k] = (a + float(g.norm()) ** 2, r + float(ref["grads"][name].norm()) ** 2)
        record_parity(f"{tag}_shortest_row_share", {"row": short, "out_len": int(batch["out_lens"][short]),
                                                    **{k: math.sqrt(a / r) for k, (a, r) in share.items()}})
    assert not bad, bad


def _rel_to(g, ref):
    return float((g - ref).norm()) / max(float(ref.norm()), 1e-30)


def test_cfg1_graph_replay_matches_fp64_oracle(oracle):
    """The cfg1 step as bench.py times it: zero_grad -> forward -> loss -> backward -> clip_grad_norm_(1.0) -> step() of
    the fused capturable RAdam, captured in one CUDA graph and replayed from the synth parameters.  The replayed gradients
    meet the oracle bars and agree with eager backwards; the replay's loss equals the eager loss; the device-side total norm
    equals the oracle's fp64 norm of all gradients."""
    from flowtron_b200 import _lib
    from flowtron_b200.radam import RAdam
    cfg, batch, ctc_weight, ref = oracle("cfg1")
    model = _model(cfg)
    crit = _crit(ctc_weight)
    cu = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in batch.items()}
    opt = RAdam(model.parameters(), lr=1e-3, weight_decay=1e-6, capturable=True)
    loss_static = torch.zeros((), device="cuda")
    norm_static = torch.zeros((), device="cuda")

    def step():
        opt.zero_grad()
        _, _, loss = _fwd_bwd(model, crit, cu, ctc_weight)
        norm = opt.clip_grad_norm_(1.0)
        opt.step()
        loss_static.copy_(loss)
        norm_static.copy_(norm)

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    opt.zero_grad()
    torch.cuda.synchronize()
    with torch.cuda.graph(graph):
        step()
    torch.cuda.synchronize()
    synth_p = synth.synth_params(cfg, SEED)
    params = dict(model.named_parameters())

    def restore():
        with torch.no_grad():
            for n, p in params.items():
                p.copy_(synth_p[n])

    restore()
    graph.replay()
    torch.cuda.synchronize()
    assert _lib.device_status() == 0
    replayed = {n: p.grad.clone() for n, p in params.items()}
    replay_loss, replay_norm = float(loss_static), float(norm_static)
    restore()
    eager = []
    for _ in range(3):
        opt.zero_grad()
        _, _, loss = _fwd_bwd(model, crit, cu, ctc_weight)
        torch.cuda.synchronize()
        eager.append(({n: p.grad.clone() for n, p in params.items()}, float(loss)))
    assert _lib.device_status() == 0

    bad = _check_grads("train_oracle_cfg1_replay_grads", replayed, ref["grads"], BARS["cfg1"])
    ratios = {}
    for n in params:
        spread = max(_rel_to(a[0][n], b[0][n]) for i, a in enumerate(eager) for b in eager[i + 1:])
        ratios[n] = _rel_to(replayed[n], eager[0][0][n]) / max(3.0 * spread, 1e-6)
    worst = max(ratios, key=ratios.get)
    loss_err = abs(replay_loss - eager[0][1]) / abs(eager[0][1])
    onorm = math.sqrt(sum(float(r.norm()) ** 2 for r in ref["grads"].values()))
    norm_err = abs(replay_norm - onorm) / onorm
    record_parity("train_oracle_cfg1_replay", {"replay_vs_eager_over_bar": ratios[worst], "replay_vs_eager_tensor": worst,
                                               "loss_rel": loss_err, "norm_rel": norm_err, "norm": replay_norm,
                                               "oracle_norm": onorm})
    assert not bad, bad
    assert ratios[worst] <= 1.0, (worst, ratios[worst])
    assert loss_err <= 1e-6, loss_err
    assert norm_err <= NORM_BAR, (replay_norm, onorm)
