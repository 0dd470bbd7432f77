"""GPU: one flow step's backward against torch.autograd of the fp64 oracle, one upstream gradient at a time.

The product modules (`Flowtron.flows[i]`: AR_Step / AR_Back_Step, with and without a gate) run forward and backward on
the sm_90a kernels (ft_ar_step_fwd, ft_ar_step_bwd_main, ft_ar_step_bwd_attn_lstm).  The reference is
oracle/flowtron_oracle.py in fp64 on the same fp32-valued weights and inputs; its own gradient is pinned by finite
differences in tests/test_ar_step_oracle_host.py.  The oracle runs on the GPU in fp64 only to keep the test short: it is
the same torch code that tests/test_oracle_golden.py pins on the CPU.

Each case runs each upstream gradient alone (d_z, d_log_s, d_gate, d_attn, d_attn_logprob) and then all of them together
at the relative scales FlowtronLoss + the attention-CTC loss produce.  Upstream gradients are zero on padded positions
(frames t >= out_len, and keys l >= in_len for attn / attn_logprob), as every masked loss makes them.  d_mel and d_text
are compared per utterance, so an error confined to one row of a ragged batch cannot hide in a tensor norm.

The base case adds a dynamic-range path: d_z at 1e-4 of d_attn_logprob.  A flow's backward runs at one loss scale, chosen
from its largest incoming gradient, so here the attention side sets it and the coupling path's gradients (conv, dense,
lstm layers 0 and 1) sit far down the fp16 range; they must still meet the bars."""
import pytest
import torch

from conftest import record_parity
from flowtron_b200 import synth

pytestmark = pytest.mark.gpu

CFG = synth.DEFAULT_MODEL_CONFIG
SEED = 5
M, A, E = CFG["n_mel_channels"], CFG["n_attn_channels"], CFG["n_text_dim"] + CFG["n_speaker_dim"]
OUTPUTS = ("d_z", "d_log_s", "d_gate", "d_attn", "d_attn_logprob")     # upstream gradient of output i of a flow step

# Bars per path (see _check): worst relative L2 of d_mel and of d_text over utterances, worst relative L2 and cosine over
# the parameter gradients, each against its own oracle gradient.  Each bar is about 3x the worst value measured over every
# case and both directions (NVIDIA H100 80GB HBM3, 700 W); repeated runs move these errors by a few percent (fp32
# atomics).  The errors come from the backward's fp16 tensor-core operands; d_mel of d_z alone stays in fp32 and is two
# orders tighter.  In the dynamic-range path the coupling tensors (conv, dense, lstm layers 0 and 1) stay at <= 1.07e-3,
# as accurate as the attention side that sets the loss scale.  Two parameter bars are 1e-2, about 2.5x the worst: the
# attention `v` weight under d_log_s at T = 320 (4.02e-3) and the attention-LSTM biases at T = 1 (3.82e-3, a sum over only
# B rows of fp16-rounded gate gradients).
BARS = {                         # d_mel    d_text   params   cosine         measured worst
    "d_z": (7.1e-05, 3.1e-03, 5.9e-03, 1 - 5.8e-06),               # 2.37e-05  1.06e-03  1.98e-03  1 - 1.9e-06
    "d_log_s": (3.1e-03, 3.3e-03, 1.0e-02, 1 - 2.3e-05),           # 1.06e-03  1.12e-03  4.02e-03  1 - 7.8e-06
    "d_gate": (1.5e-03, 1.6e-03, 3.1e-03, 1 - 1.6e-06),            # 5.24e-04  5.36e-04  1.04e-03  1 - 5.4e-07
    "d_attn": (2.4e-03, 1.8e-03, 3.6e-03, 1 - 2.1e-06),            # 8.22e-04  6.01e-04  1.21e-03  1 - 7.3e-07
    "d_attn_logprob": (2.5e-03, 3.3e-03, 2.4e-03, 1 - 9.6e-07),    # 8.62e-04  1.12e-03  8.01e-04  1 - 3.2e-07
    "all": (5.8e-04, 2.1e-03, 1.0e-02, 1 - 2.1e-05),               # 1.95e-04  7.11e-04  3.82e-03  1 - 7.3e-06
    "range": (2.2e-03, 1.0e-03, 3.3e-03, 1 - 1.8e-06),             # 7.50e-04  3.42e-04  1.12e-03  1 - 6.3e-07
}
FWD_BAR = 1e-3                   # forward outputs on valid positions, relative to the tensor's max |value|


# (direction, gate) -> (n_flows, flow index): only the last flow of a model has a gate
_WHERE = {("fwd", True): (1, 0), ("back", True): (2, 1), ("fwd", False): (2, 0), ("back", False): (3, 1)}


def _load_flow(direction, gate):
    """The flow module on the GPU, its inner AR_Step, its parameters and their oracle names, and fp64 oracle weights."""
    from flowtron_b200.flowtron import Flowtron
    n_flows, i = _WHERE[(direction, gate)]
    cfg = dict(CFG, n_flows=n_flows)
    params = synth.synth_params(cfg, SEED)
    model = Flowtron(**cfg)
    model.load_state_dict(params, strict=True)
    flow = model.flows[i].cuda()
    step = flow.ar_step if direction == "back" else flow
    assert hasattr(step, "gate_layer") == gate
    names = [n for n, _ in flow.named_parameters()]
    keys = [f"flows.{i}.{n}" for n in names]
    p64 = {k: params[k].double().cuda() for k in keys}
    return flow, step, f"flows.{i}", [p for _, p in flow.named_parameters()], keys, p64


@pytest.fixture(scope="module")
def flows():
    """_load_flow, each (direction, gate) loaded once for this module and released when it ends."""
    cache = {}

    def get(direction, gate):
        if (direction, gate) not in cache:
            cache[(direction, gate)] = _load_flow(direction, gate)
        return cache[(direction, gate)]
    yield get
    cache.clear()
    torch.cuda.empty_cache()


def _lengths(B, hi, g, descending):
    """B ragged lengths in [1, hi] that include 1 and hi (B = 1: hi)."""
    v = torch.randint(1, hi + 1, (B,), generator=g)
    v[0] = hi
    if B > 1:
        v[1] = 1
    if descending:                                # the collate's order for text lengths
        return v.sort(descending=True).values
    return v[torch.randperm(B, generator=g)]


def _inputs(B, T, L, with_prior, seed):
    g = torch.Generator().manual_seed(seed)
    out_lens = _lengths(B, T, g, descending=False)
    in_lens = _lengths(B, L, g, descending=True)
    vt = torch.arange(T)[:, None] < out_lens[None, :]                         # [T,B] valid frames
    vk = torch.arange(L)[None, :] < in_lens[:, None]                          # [B,L] valid keys
    mel = torch.randn(T, B, M, generator=g) * vt[..., None]
    text = 0.5 * torch.randn(L, B, E, generator=g)                            # pad rows non-zero on purpose
    prior = None
    if with_prior:
        prior = torch.zeros(B, T, L)
        for b in range(B):
            t, l = int(out_lens[b]), int(in_lens[b])
            prior[b, :t, :l] = torch.from_numpy(synth.beta_binomial_prior(l, t)).float()
    mask = ~vk[..., None]
    cu = lambda x: None if x is None else x.cuda()
    return dict(mel=cu(mel), text=cu(text), mask=cu(mask), out_lens=cu(out_lens), in_lens=cu(in_lens), prior=cu(prior),
                vt=cu(vt), vk=cu(vk), g=g)


def _upstream(path, x, ref_outs, has_gate):
    """{output index: upstream gradient} of a path, zero on padded positions."""
    vt, vk, g = x["vt"].double(), x["vk"].double(), x["g"]
    T, B = vt.shape
    L = vk.shape[1]
    vtl = vt.t()[:, :, None] * vk[:, None, :]
    N = float(vt.sum())
    rnd = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64).cuda()
    shapes = [(T, B, M), (T, B, M), (T, B, 1), (B, T, L), (B, T, L)]
    masks = [vt[..., None], vt[..., None], vt[..., None], vtl, vtl]
    if path in OUTPUTS:
        i = OUTPUTS.index(path)
        return {i: rnd(*shapes[i]) * masks[i]}
    if path == "all":                  # FlowtronLoss (nll + gate) and attention-CTC scales
        up = {0: ref_outs[0].detach() * masks[0] / (N * M),
              1: -masks[1].expand(T, B, M) / (N * M),
              3: 1e-3 * rnd(*shapes[3]) * masks[3],
              4: 1e-3 * rnd(*shapes[4]) * masks[4]}
        if has_gate:
            up[2] = (torch.rand(T, B, 1, generator=g, dtype=torch.float64).cuda() - 0.5) * masks[2] / N
        return up
    assert path == "range"             # d_z 1e-4 of d_attn_logprob: the attention side sets the loss scale
    return {0: 1e-7 * rnd(*shapes[0]) * masks[0], 4: 1e-3 * rnd(*shapes[4]) * masks[4]}


def _oracle(direction, pre, p64, x, temperature):
    from oracle import flowtron_oracle as O
    fn = O.ar_back_step_forward if direction == "back" else O.ar_step_forward
    ins = [x["mel"].double().requires_grad_(True), x["text"].double().requires_grad_(True)]
    ins += [v.clone().requires_grad_(True) for v in p64.values()]
    prior = None if x["prior"] is None else x["prior"].double()
    outs = fn(dict(zip(p64, ins[2:])), pre, ins[0], ins[1], x["mask"], x["out_lens"], prior, temperature)
    return outs, ins


def _oracle_grads(outs, ins, up):
    idx = list(up)
    gs = torch.autograd.grad([outs[i] for i in idx], ins, [up[i] for i in idx], retain_graph=True, allow_unused=True)
    return [torch.zeros_like(x) if g is None else g for g, x in zip(gs, ins)]


def _gpu(flow, params, x, up):
    """Forward + torch.autograd.grad through the product module: (outputs, [d_mel, d_text, *parameter gradients])."""
    from flowtron_b200 import _lib
    mel, text = x["mel"].clone().requires_grad_(True), x["text"].clone().requires_grad_(True)
    outs = flow(mel, text, x["mask"], x["out_lens"], x["prior"])
    idx = list(up)
    grads = torch.autograd.grad([outs[i] for i in idx], [mel, text, *params], [up[i].float() for i in idx])
    torch.cuda.synchronize()
    assert _lib.device_status() == 0
    return outs, grads


def _rel(a, b, floor):
    return float((a.double() - b).norm()) / max(float(b.norm()) + floor, 1e-300)


def _check_forward(tag, outs, ref, x):
    vt, vk = x["vt"], x["vk"]
    vtl = vt.t()[:, :, None] & vk[:, None, :]
    errs = {}
    for name, o, r, m in zip(("z", "log_s", "gate", "attn", "attn_logprob"), outs, ref, (vt, vt, vt, vtl, vtl)):
        if r is None:
            assert o is None
            continue
        a, b = o.detach().double()[m], r.detach()[m]
        errs[name] = float((a - b).abs().max()) / max(float(b.abs().max()), 1e-30)
    record_parity(f"{tag}_forward", errs)
    bad = {k: v for k, v in errs.items() if not v <= FWD_BAR}
    assert not bad, bad


def _check(tag, path, gpu, ref, keys, x):
    """Exact: every gradient finite, d_mel zero on padded frames, d_text zero on padded keys, and a parameter gradient
    that the path does not reach (oracle gradient exactly zero) is exactly zero.  Per utterance: d_mel and d_text relative
    L2 against the oracle's slice (floor 1e-4 of the whole tensor's norm).  Every other parameter gradient: relative L2
    and cosine against its own oracle gradient, with no floor, so a small tensor (the coupling path's, when the attention
    side dominates) is held to the same bar as a large one."""
    bar_mel, bar_text, bar_p, bar_cos = BARS[path]
    d_mel, d_text, *pg = gpu
    r_mel, r_text, *pr = ref
    for name, t in zip(["d_mel", "d_text"] + keys, gpu):
        assert torch.isfinite(t).all(), (tag, name)
    assert (d_mel[~x["vt"]] == 0).all(), (tag, "d_mel is not zero on padded frames")
    assert (d_text.transpose(0, 1)[~x["vk"]] == 0).all(), (tag, "d_text is not zero on padded keys")
    errs = {}
    for name, g, r in (("d_mel", d_mel, r_mel), ("d_text", d_text, r_text)):
        floor = 1e-4 * float(r.norm())
        per = [_rel(g[:, b], r[:, b], floor) for b in range(g.shape[1])]
        errs[name] = max(per)
        errs[name + "_row"] = per.index(errs[name])
    rows, unreached = [], []
    for name, g, r in zip(keys, pg, pr):
        g64, r64 = g.reshape(-1).double(), r.reshape(-1)
        rn = float(r64.norm())
        if rn == 0.0:
            unreached.append((name, float(g64.norm())))
            continue
        rows.append((name, float((g64 - r64).norm()) / rn, float(g64 @ r64) / (float(g64.norm()) * rn + 1e-300)))
    worst = max(rows, key=lambda r: r[1], default=("", 0.0, 1.0))           # L = 1: attn / attn_logprob reach nothing
    least = min(rows, key=lambda r: r[2], default=("", 0.0, 1.0))
    errs.update(param_rel_l2=worst[1], param_rel_l2_tensor=worst[0], param_cos=least[2], param_cos_tensor=least[0])
    errs["unreached_norm"] = max([n for _, n in unreached], default=0.0)
    record_parity(tag, errs)
    bad = [f"{n}: not reached by this path, yet |grad| = {v:.3e}" for n, v in unreached if v != 0.0]
    bad += [f"{k}={errs[k]:.3e} (row {errs[k + '_row']})" for k, bar in (("d_mel", bar_mel), ("d_text", bar_text))
           if not errs[k] <= bar]
    bad += [f"{n}: rel {e:.3e} cos {c:.6f}" for n, e, c in rows if not (e <= bar_p and c >= bar_cos)]
    assert not bad, (tag, bad)


CASES = {
    # name: (B, T, L, prior, gate, temperature)
    "base": (5, 77, 12, True, True, 1.0),
    "no_prior": (5, 77, 12, False, True, 1.0),
    "no_gate": (5, 77, 12, True, False, 1.0),
    "temperature": (4, 60, 10, True, True, 0.5),   # Flowtron.infer(temperature=...) leaves it set for later training
    "temperature_no_prior": (4, 60, 10, False, True, 0.5),
    "t1": (3, 1, 9, True, True, 1.0),              # Rm = 0: no recurrent weight-gradient rows
    "t2": (3, 2, 9, True, True, 1.0),
    "t101": (3, 101, 9, True, True, 1.0),          # a one-step tail chunk of the 100-step layer pipeline
    "t320": (3, 320, 9, True, True, 1.0),          # the first T with the attention-LSTM overlap (256 + 64)
    "b1": (1, 40, 11, True, True, 1.0),
    "b17": (17, 40, 11, True, True, 1.0),          # N padded to 32 in the recurrences
    "b32": (32, 40, 11, True, True, 1.0),
    "l1": (3, 48, 1, True, True, 1.0),
    "l256": (3, 48, 256, True, True, 1.0),         # the last short-text attention variant
    "l257": (3, 48, 257, True, True, 1.0),         # the first long-text attention variant
    "l673": (3, 48, 673, True, True, 1.0),         # the first length whose attention rows go through global memory
    "l1024": (2, 40, 1024, True, True, 1.0),
}


@pytest.mark.parametrize("direction", ["fwd", "back"])
@pytest.mark.parametrize("case", list(CASES))
def test_flow_step_backward_matches_fp64_oracle(flows, case, direction):
    """Forward outputs, then d_mel, d_text and every parameter gradient of each path against the fp64 oracle."""
    B, T, L, with_prior, gate, temperature = CASES[case]
    flow, step, pre, params, keys, p64 = flows(direction, gate)
    x = _inputs(B, T, L, with_prior, seed=17 + list(CASES).index(case))
    ref_outs, ins = _oracle(direction, pre, p64, x, temperature)
    paths = [p for p in OUTPUTS if gate or p != "d_gate"] + ["all"] + (["range"] if case == "base" else [])
    step.attention_layer.temperature = temperature
    try:
        for k, path in enumerate(paths):
            up = _upstream(path, x, ref_outs, gate)
            outs, gpu = _gpu(flow, params, x, up)
            tag = f"ar_step_bwd_{case}_{direction}_{path}"
            if k == 0:
                _check_forward(f"ar_step_bwd_{case}_{direction}", outs, ref_outs, x)
            _check(tag, path, gpu, _oracle_grads(ref_outs, ins, up), keys, x)
    finally:
        step.attention_layer.temperature = 1.0


@pytest.mark.parametrize("present", [("d_mel_out",), ("d_logprob",), ("d_log_s", "d_attn")])
def test_null_upstream_gradients_equal_zero_filled(flows, present):
    """The C backward takes NULL for an absent upstream gradient (autograd always hands it zero-filled tensors instead).
    Both forms must give the same d_mel, d_text and parameter gradients up to the order of fp32 atomics."""
    from flowtron_b200 import _lib
    B, T, L = 5, 77, 12
    step = flows("fwd", True)[1]
    x = _inputs(B, T, L, True, seed=3)
    i32 = lambda t: t.to(torch.int32).contiguous()
    in_lens, out_lens = i32(x["in_lens"]), i32(x["out_lens"])
    mel, text, prior = x["mel"].contiguous(), x["text"].contiguous(), x["prior"].contiguous()
    vt, vk = x["vt"].float(), x["vk"].float()
    g = x["g"]
    rnd = lambda *s: torch.randn(*s, generator=g).cuda()
    up = {"d_mel_out": rnd(T, B, M) * vt[..., None], "d_log_s": rnd(T, B, M) * vt[..., None],
          "d_gates": rnd(T, B, 1) * vt[..., None],
          "d_attn": rnd(B, T, L) * vt.t()[:, :, None] * vk[:, None, :],
          "d_logprob": rnd(B, T, L) * vt.t()[:, :, None] * vk[:, None, :]}
    plist = [p.detach() for p in step._param_list()]
    desc = _lib.FtArStepDesc(T, B, L, M, CFG["n_hidden"], A, E, 0, 1, 1, 1.0)
    saved_bytes, scratch_bytes = _lib.ar_step_sizes(desc)

    def run(zeros):
        saved = torch.empty(saved_bytes, dtype=torch.uint8, device="cuda")
        scratch = torch.empty(scratch_bytes, dtype=torch.uint8, device="cuda")
        carry = torch.empty(_lib.ar_step_bwd_carry_bytes(desc), dtype=torch.uint8, device="cuda")
        outs = [torch.empty(T, B, M, device="cuda"), torch.empty(T, B, M, device="cuda"), torch.empty(T, B, 1, device="cuda"),
                torch.empty(B, T, L, device="cuda"), torch.empty(B, T, L, device="cuda")]
        w = _lib.make_weights(plist)
        _lib.ar_step_fwd(desc, w, mel, text, in_lens, out_lens, prior, *outs, saved, scratch)
        d = {k: (v if k in present else (torch.zeros_like(v) if zeros else None)) for k, v in up.items()}
        d_mel, d_text = torch.full_like(mel, float("nan")), torch.full_like(text, float("nan"))
        grads = [torch.full_like(p, float("nan")) for p in plist]
        gw = _lib.make_weights(grads)
        _lib.ar_step_bwd_main(desc, w, mel, in_lens, out_lens, outs[3], d["d_mel_out"], d["d_log_s"], d["d_gates"], d["d_attn"],
                              d["d_logprob"], d_text, gw, saved, scratch, carry)
        _lib.ar_step_bwd_attn_lstm(desc, w, out_lens, d_mel, gw, saved, scratch, carry)
        torch.cuda.synchronize()
        assert _lib.device_status() == 0
        return [d_mel, d_text] + grads

    a, b = run(False), run(True)
    gmax = max(float(t.norm()) for t in b)
    for name, u, v in zip(["d_mel", "d_text"] + _lib.AR_WEIGHT_FIELDS, a, b):
        assert torch.isfinite(u).all() and torch.isfinite(v).all(), name
        dn = float((u - v).norm())
        assert dn <= 1e-3 * (float(v.norm()) + 1e-4 * gmax), (name, dn, float(v.norm()))
