"""GPU: fine-tuning a subset of Flowtron's parameters.  A flow step's backward computes only the gradients that are wanted
(parameters with requires_grad, d_text / d_mel when text / mel require grad) and runs only the stages they depend on
(ft_ar_step_bwd_plan, pinned on the CPU by tests/test_finetune_host.py).

1. One flow step, each subset against the fp64 oracle (the bars and the machinery of tests/test_gpu_ar_step_backward.py)
   and against the same step with every gradient wanted.
2. The whole model for the README's two fine-tuning workflows (speaker embedding only; the last flow's gate only) and for
   one whole flow: trainable gradients against a full backward, frozen parameters keep .grad None.
3. The work skipped, counted with _lib.launch_count().
4. The speaker-only and gate-only steps captured in one CUDA graph with the capturable RAdam.

"Spread": the largest relative L2 between the same gradient from three full backwards on the same inputs (fp32 atomics
make them differ); a subset's gradient must agree with the first full one within 3x that spread, with a 1e-6 floor."""
import pytest
import torch

from conftest import record_parity
from flowtron_b200 import _lib, synth
from test_gpu_ar_step_backward import BARS, _inputs, _load_flow, _oracle, _oracle_grads, _rel, _upstream

pytestmark = pytest.mark.gpu


def _rel_to(g, ref):
    return float((g - ref).norm()) / max(float(ref.norm()), 1e-30)


F = _lib.AR_WEIGHT_FIELDS
SUBSETS = {                       # name: (parameter fields, d_text, d_mel)
    "gate": (["gate_w", "gate_b"], False, False),
    "attention_lstm": ([f for f in F if f.startswith("attn_lstm_")], False, False),
    "lstm_l1": (["lstm_w_ih1", "lstm_w_hh1", "lstm_b_ih1", "lstm_b_hh1"], False, False),
    "qkv": (["att_query", "att_key", "att_value"], False, False),
    "d_text": ([], True, False),
    "d_mel": ([], False, True),
    "mixed": (["lstm_w_hh0", "lstm_b_hh1", "att_v", "dense_w1", "conv_b", "gate_b"], True, False),
}


def _spread_bar(fulls):
    spread = max(_rel_to(a, b) for i, a in enumerate(fulls) for b in fulls[i + 1:])
    return max(3.0 * spread, 1e-6)


@pytest.mark.parametrize("gate", [True, False])
@pytest.mark.parametrize("direction", ["fwd", "back"])
def test_flow_step_subsets_match_oracle_and_full_backward(direction, gate):
    flow, step, pre, params, keys, p64 = _load_flow(direction, gate)
    plist = step._param_list()
    fields = [F[next(i for i, q in enumerate(plist) if q is p)] for p in params]
    B, T, L = 5, 77, 12
    x = _inputs(B, T, L, True, seed=41)
    ref_outs, ins = _oracle(direction, pre, p64, x, 1.0)
    up = _upstream("all", x, ref_outs, gate)
    ref = dict(zip(["d_mel", "d_text"] + fields, _oracle_grads(ref_outs, ins, up)))
    bar_mel, bar_text, bar_p, bar_cos = BARS["all"]

    def run(want, d_text, d_mel):
        for p, f in zip(params, fields):
            p.requires_grad_(f in want)
        mel = x["mel"].clone().requires_grad_(d_mel)
        text = x["text"].clone().requires_grad_(d_text)
        names = (["d_mel"] if d_mel else []) + (["d_text"] if d_text else []) + [f for f in fields if f in want]
        wrt = ([mel] if d_mel else []) + ([text] if d_text else []) + [p for p, f in zip(params, fields) if f in want]
        outs = flow(mel, text, x["mask"], x["out_lens"], x["prior"])
        idx = list(up)
        gs = torch.autograd.grad([outs[i] for i in idx], wrt, [up[i].float() for i in idx])
        torch.cuda.synchronize()
        assert _lib.device_status() == 0
        assert all(p.grad is None for p in params)
        return dict(zip(names, gs))

    try:
        fulls = [run(fields, True, True) for _ in range(3)]
        for name, (want, d_text, d_mel) in SUBSETS.items():
            if name == "gate" and not gate:
                continue
            want = [f for f in want if f in fields]
            got = run(want, d_text, d_mel)
            assert set(got) == set(want) | ({"d_text"} if d_text else set()) | ({"d_mel"} if d_mel else set())
            errs, bad = {}, []
            for k, g in got.items():
                assert torch.isfinite(g).all(), (name, k)
                r = ref[k]
                if k in ("d_mel", "d_text"):
                    floor = 1e-4 * float(r.norm())
                    col = 1
                    errs[k] = max(_rel(g.select(col, b), r.select(col, b), floor) for b in range(B))
                    if not errs[k] <= (bar_mel if k == "d_mel" else bar_text):
                        bad.append((k, "oracle", errs[k]))
                else:
                    g64, r64 = g.reshape(-1).double(), r.reshape(-1)
                    rel = float((g64 - r64).norm()) / max(float(r64.norm()), 1e-300)
                    cos = float(g64 @ r64) / (float(g64.norm()) * float(r64.norm()) + 1e-300)
                    errs[k] = rel
                    if float(r64.norm()) > 0 and not (rel <= bar_p and cos >= bar_cos):
                        bad.append((k, "oracle", rel, cos))
                d_full, bar_full = _rel_to(g, fulls[0][k]), _spread_bar([f[k] for f in fulls])
                errs[k + "_vs_full"] = d_full
                if not d_full <= bar_full:
                    bad.append((k, "full", d_full, bar_full))
            record_parity(f"finetune_step_{direction}_{'gate' if gate else 'nogate'}_{name}", errs)
            assert not bad, (name, bad)
    finally:
        for p in params:
            p.requires_grad_(True)


# ------------------------------------------------------------------------------------------------ whole model
def _workflow(names, which):
    if which == "speaker":
        return {"speaker_embedding.weight"}
    if which == "gate":
        return {n for n in names if "gate_layer" in n}
    assert which == "flow1"
    return {n for n in names if n.startswith("flows.1.")}


def _model(n_flows):
    from flowtron_b200.flowtron import Flowtron
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=n_flows, n_speakers=3)
    model = Flowtron(**cfg)
    model.load_state_dict(synth.synth_params(cfg, 11), strict=True)
    model = model.cuda().train()
    model.encoder.p_dropout = 0.0
    batch = synth.synth_batch(4, 96, 14, cfg, 11, out_lens=[96, 41, 70, 1], in_lens=[14, 12, 9, 5], with_prior=True)
    cu = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in batch.items()}
    return model, cu


class _Counter:
    """Launches enqueued by the flow-step backward calls and by the loss gradient, from _lib.launch_count()."""

    def __init__(self, monkeypatch):
        self.flow, self.attn_calls, self.loss = [], 0, 0
        for name in ("ar_step_bwd_main", "ar_step_bwd_attn_lstm", "nll_grad"):
            monkeypatch.setattr(_lib, name, self._wrap(name, getattr(_lib, name)))

    def _wrap(self, name, fn):
        def call(*a, **k):
            n0 = _lib.launch_count()
            fn(*a, **k)
            n = _lib.launch_count() - n0
            if name == "nll_grad":
                self.loss += n
            else:
                self.flow.append(n)
                self.attn_calls += name == "ar_step_bwd_attn_lstm"
        return call


def _backward(model, cu, train, mel_grad=False):
    from flowtron_b200.flowtron import FlowtronLoss
    for n, p in model.named_parameters():
        p.requires_grad_(train is None or n in train)
        p.grad = None
    crit = FlowtronLoss(sigma=1.0, gate_loss=True, use_ctc_loss=True, ctc_loss_weight=0.1)
    mel = cu["mel"].clone().requires_grad_(mel_grad)
    out = model(mel, cu["speaker_ids"], cu["text"], cu["in_lens"], cu["out_lens"], cu["attn_prior"])
    nll, gl, ctc = crit(out, cu["gate_target"], cu["in_lens"], cu["out_lens"])
    loss = (nll + gl + 0.1 * ctc).sum()
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    loss.backward()
    torch.cuda.synchronize()
    assert _lib.device_status() == 0
    launches = _lib.launch_count() - n0
    return {n: (None if p.grad is None else p.grad.clone()) for n, p in model.named_parameters()}, launches


@pytest.mark.parametrize("n_flows", [2, 3])
def test_finetune_gradients_match_full_backward(n_flows, monkeypatch):
    model, cu = _model(n_flows)
    try:
        fulls = [_backward(model, cu, None) for _ in range(3)]
        n_full = fulls[0][1]
        assert all(n == n_full for _, n in fulls)
        fulls = [g for g, _ in fulls]
        names = list(fulls[0])
        bars = {n: _spread_bar([f[n] for f in fulls]) for n in names}
        launches = {}
        for which in ("speaker", "gate", "flow1"):
            train = _workflow(names, which)
            assert train
            counter = _Counter(monkeypatch)
            got, launches[which] = _backward(model, cu, train)
            monkeypatch.undo()
            errs, bad = {}, []
            for n in names:
                if n not in train:
                    assert got[n] is None, (which, n, "a frozen parameter got a gradient")
                    continue
                d = _rel_to(got[n], fulls[0][n])
                errs[n] = d
                if not d <= bars[n]:
                    bad.append((n, d, bars[n]))
            record_parity(f"finetune_model_{n_flows}flows_{which}", errs)
            assert not bad, (which, bad)
            if which == "gate":              # the last flow's backward is the gate kernel alone; the others do not run
                assert counter.flow == [1] and counter.attn_calls == 0, counter.flow
                assert launches[which] == counter.loss + 1, (launches[which], counter.loss)
        assert launches["speaker"] < n_full, (launches, n_full)
        # full training: the first flow's mel is data, so its d_mel dgrad, that dgrad's weight cast and combine_dmel are
        # skipped; a mel that requires grad brings exactly these three launches back, and the parameter gradients agree
        with_mel, n_mel = _backward(model, cu, None, mel_grad=True)
        assert n_mel == n_full + 3, (n_mel, n_full)
        for n in names:
            assert _rel_to(with_mel[n], fulls[0][n]) <= bars[n], n
    finally:
        for p in model.parameters():
            p.requires_grad_(True)


# ------------------------------------------------------------------------------------------------ CUDA graph
@pytest.mark.parametrize("which", ["speaker", "gate"])
def test_finetune_step_replays_from_one_cuda_graph(which):
    from flowtron_b200.flowtron import FlowtronLoss
    from flowtron_b200.radam import RAdam
    model, cu = _model(2)
    names = [n for n, _ in model.named_parameters()]
    train = _workflow(names, which)
    for n, p in model.named_parameters():
        p.requires_grad_(n in train)
    opt = RAdam([p for p in model.parameters() if p.requires_grad], lr=1e-3, weight_decay=1e-6, capturable=True)
    crit = FlowtronLoss(sigma=1.0, gate_loss=True, use_ctc_loss=True, ctc_loss_weight=0.1)
    assert cu["in_lens"].is_cuda and cu["out_lens"].is_cuda

    def fwd_bwd():
        out = model(cu["mel"], cu["speaker_ids"], cu["text"], cu["in_lens"], cu["out_lens"], cu["attn_prior"])
        nll, gl, ctc = crit(out, cu["gate_target"], cu["in_lens"], cu["out_lens"])
        (nll + gl + 0.1 * ctc).sum().backward()

    def step():
        opt.zero_grad()
        fwd_bwd()
        opt.clip_grad_norm_(1.0)
        opt.step()

    for _ in range(2):
        step()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    opt.zero_grad()
    torch.cuda.synchronize()
    with torch.cuda.graph(graph):
        step()
    torch.cuda.synchronize()
    params = dict(model.named_parameters())

    def eager_grads():
        opt.zero_grad()
        fwd_bwd()
        torch.cuda.synchronize()
        return {n: params[n].grad.clone() for n in train}

    for _ in range(3):
        before = {n: p.detach().clone() for n, p in params.items()}
        graph.replay()
        torch.cuda.synchronize()
        assert _lib.device_status() == 0
        replayed = {n: params[n].grad.clone() for n in train}
        after = {n: p.detach().clone() for n, p in params.items()}
        for n in names:
            if n in train:
                assert not torch.equal(after[n], before[n]), (n, "a trainable parameter was not updated")
            else:
                assert torch.equal(after[n], before[n]), (n, "a frozen parameter changed")
                assert params[n].grad is None, n
        with torch.no_grad():                    # the same gradients eagerly, at the parameters the replay started from
            for n, p in params.items():
                p.copy_(before[n])
        eager = [eager_grads() for _ in range(3)]
        for n in train:
            assert _rel_to(replayed[n], eager[0][n]) <= _spread_bar([e[n] for e in eager]), n
        with torch.no_grad():
            for n, p in params.items():
                p.copy_(after[n])
