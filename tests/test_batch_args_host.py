"""CPU: the argument checks of Flowtron's padded-batch entry points (encode, convert, align, score, infer_batch,
infer_aligned, infer_durations), all made before any device work.  One table of bad lengths, batch sizes and texts runs
against every entry point; the checks only one entry point makes follow it.  With valid arguments, CPU tensors raise
FlowtronB200Error: the sm_90a kernels are the only implementation.  The ``cpu_model`` fixture here is the one the other
host tests that need a Flowtron use."""
import pytest
import torch

from flowtron_b200 import synth
from flowtron_b200._lib import FlowtronB200Error

B, T, L = 3, 20, 9
IN_LENS, FRAMES = [9, 4, 6], [20, 7, 13]


@pytest.fixture(scope="module")
def cpu_model():
    from flowtron_b200.flowtron import Flowtron
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=2, n_speakers=2)
    m = Flowtron(**cfg)
    m.load_state_dict(synth.synth_params(cfg, 3), strict=True)
    return m.eval()


def _spk(n=B):
    return torch.zeros(n, dtype=torch.long)


def _text(n_tokens=L):
    return torch.zeros(B, n_tokens, dtype=torch.long)


def _maps(x, text, frames=None):
    """One forced alignment per flow for infer_aligned, [B, Ta, L] with Ta = the frames of x unless given."""
    return [torch.zeros(text.size(0), x.size(-1) if frames is None else frames, text.size(-1))] * 2


# entry point -> (call(model, x, text, in_lens, frames), name of its per-row frame lengths or None).  x is the [B, 80, T]
# mel or residual; every other argument is built to fit, so only the case under test is wrong.
ENTRIES = {
    "encode": (lambda m, x, text, il, fl: m.encode(x, _spk(), text, il, fl), "out_lens"),
    "convert": (lambda m, x, text, il, fl: m.convert(x, _spk(), _spk(x.size(0)), text, il, fl), "out_lens"),
    "align": (lambda m, x, text, il, fl: m.align(x, _spk(), text, il, fl), "out_lens"),
    "score": (lambda m, x, text, il, fl: m.score(x, _spk(), text, il, fl), "out_lens"),
    "infer_batch": (lambda m, x, text, il, fl: m.infer_batch(x, _spk(), text, il, max_frames=fl), "max_frames"),
    "infer_aligned": (lambda m, x, text, il, fl: m.infer_aligned(x, _spk(), text, il, _maps(x, text), fl), "n_frames"),
    "infer_durations": (lambda m, x, text, il, fl: m.infer_durations(x, _spk(), text, il,
                                                                     torch.ones(text.shape, dtype=torch.long)), None),
}

# (case, in_lens, frames): every length case names the argument it breaks
LENGTH_CASES = [
    ("in_lens count", [9, 4], FRAMES),
    ("in_lens zero", [9, 0, 4], FRAMES),
    ("in_lens above L", [9, 10, 4], [20, 12, 13]),
    ("in_lens float", [9.0, 4.0, 6.0], FRAMES),
    ("in_lens tensor of the wrong length", torch.tensor([9, 4, 4, 4]), FRAMES),
    ("frames count", IN_LENS, [20, 7]),
    ("frames zero", IN_LENS, [20, 0, 13]),
    ("frames above T", IN_LENS, [20, 21, 13]),
    ("frames float", IN_LENS, [20.0, 7.0, 13.0]),
    ("frames tensor of the wrong length", IN_LENS, torch.tensor([20, 5])),
]


@pytest.mark.parametrize("entry,case,in_lens,frames", [
    pytest.param(entry, *c, id=f"{entry}-{c[0]}") for entry in ENTRIES for c in LENGTH_CASES
    if c[0].startswith("in_lens") or ENTRIES[entry][1] is not None])        # infer_durations: durations, checked below
def test_bad_lengths(cpu_model, entry, case, in_lens, frames):
    call, frames_name = ENTRIES[entry]
    with pytest.raises(ValueError, match="in_lens" if case.startswith("in_lens") else frames_name):
        call(cpu_model, torch.zeros(B, 80, T), _text(), in_lens, frames)


@pytest.mark.parametrize("entry", ENTRIES)
def test_bad_shapes_and_texts(cpu_model, entry):
    call, _ = ENTRIES[entry]
    mel = torch.zeros(B, 80, T)
    with pytest.raises(ValueError, match="batch sizes disagree"):
        call(cpu_model, mel[:2], _text(), IN_LENS, FRAMES)
    with pytest.raises(ValueError, match=r"expects \w+ \[B, n_mel, T\]"):
        call(cpu_model, mel[0], _text(), IN_LENS, FRAMES)
    with pytest.raises(ValueError, match=r"1024 tokens \(MAX_TEXT_LEN\)"):
        call(cpu_model, mel, _text(1025), IN_LENS, FRAMES)


@pytest.mark.parametrize("entry", ENTRIES)
def test_cpu_tensors_need_the_kernels(cpu_model, entry):
    call, _ = ENTRIES[entry]
    mel = torch.zeros(B, 80, T)
    with pytest.raises(FlowtronB200Error, match="needs CUDA tensors"):
        call(cpu_model, mel, _text(), IN_LENS, FRAMES)
    with pytest.raises(FlowtronB200Error, match="needs CUDA tensors"):
        call(cpu_model, mel, _text(), torch.tensor(IN_LENS), torch.tensor(FRAMES))


@pytest.mark.parametrize("entry", ["encode", "convert", "align", "score"])
def test_attn_prior_shape(cpu_model, entry):
    m, mel, spk, text = cpu_model, torch.zeros(B, 80, T), _spk(), _text()
    args = {"encode": lambda p: m.encode(mel, spk, text, IN_LENS, FRAMES, p),
            "convert": lambda p: m.convert(mel, spk, spk, text, IN_LENS, FRAMES, p),
            "align": lambda p: m.align(mel, spk, text, IN_LENS, FRAMES, p),
            "score": lambda p: m.score(mel, spk, text, IN_LENS, FRAMES, p)}[entry]
    with pytest.raises(ValueError, match="attn_prior"):
        args(torch.zeros(B, T, L + 1))
    with pytest.raises(FlowtronB200Error):
        args(torch.zeros(B, T, L))


def test_encode_arguments(cpu_model):
    mel, spk, text = torch.zeros(B, 80, T), _spk(), _text()
    with pytest.raises(ValueError, match="out_lens"):
        cpu_model.encode(mel, spk, text, IN_LENS, [20, 21, 13], return_attns=True)
    with pytest.raises(FlowtronB200Error):
        cpu_model.encode(mel, spk, text, IN_LENS, FRAMES, return_attns=True)


def test_convert_arguments(cpu_model):
    mel, spk, text = torch.zeros(B, 80, T), _spk(), _text()
    with pytest.raises(ValueError, match="target_speaker_ids"):
        cpu_model.convert(mel, spk, spk[:2], text, IN_LENS, FRAMES)


def test_align_arguments(cpu_model):
    mel, spk, text = torch.zeros(B, 80, T), _spk(), _text()
    for flow in (2, -1, True, 0.0):
        with pytest.raises(ValueError, match="flow"):
            cpu_model.align(mel, spk, text, IN_LENS, FRAMES, flow=flow)
    with pytest.raises(ValueError, match="at least as many frames as tokens"):
        cpu_model.align(mel, spk, text, [9, 4, 4], [20, 3, 13])            # 3 frames for 4 tokens
    with pytest.raises(FlowtronB200Error):
        cpu_model.align(mel, spk, text, IN_LENS, FRAMES, flow=1)


def test_score_arguments(cpu_model):
    mel, spk, text = torch.zeros(B, 80, T), _spk(), _text()
    for gate_target in (torch.zeros(B, T + 1), torch.zeros(T, B)):          # must be [B, T]
        with pytest.raises(ValueError, match="gate_target"):
            cpu_model.score(mel, spk, text, IN_LENS, FRAMES, gate_target=gate_target)
    with pytest.raises(FlowtronB200Error):
        cpu_model.score(mel, spk, text, IN_LENS, FRAMES, gate_target=torch.zeros(B, T))


def test_infer_batch_arguments(cpu_model):
    res, spk, text = torch.zeros(B, 80, T), _spk(), _text()
    for kw in (dict(attns=[torch.zeros(T, L)] * 2), dict(attn_prior=torch.zeros(B, T, L))):
        with pytest.raises(ValueError, match="attns or attn_prior"):
            cpu_model.infer_batch(res, spk, text, IN_LENS, **kw)
    with pytest.raises(ValueError, match="256"):                            # longer than the kernel's 256 keys
        cpu_model.infer_batch(res, spk, _text(257), IN_LENS)
    with pytest.raises(FlowtronB200Error):                                  # max_frames defaults to T for every row
        cpu_model.infer_batch(res, spk, text, torch.tensor(IN_LENS))


def test_infer_aligned_arguments(cpu_model):
    res, spk, text = torch.zeros(B, 80, T), _spk(), _text()
    attns = _maps(res, text)
    bad = [
        attns[:1],                                               # one map per flow
        attns + attns[:1],
        attns[0],                                                # not a list
        [torch.zeros(B, T, L), torch.zeros(B, T, L + 1)],
        [torch.zeros(T, B, L)] * 2,                              # time-major
        [torch.zeros(B, T, L, dtype=torch.long)] * 2,
    ]
    for a in bad:
        with pytest.raises(ValueError, match="attns"):
            cpu_model.infer_aligned(res, spk, text, IN_LENS, a, FRAMES)
    with pytest.raises(ValueError, match="n_frames"):          # the maps cover 12 frames, row 0 wants 20
        cpu_model.infer_aligned(res, spk, text, IN_LENS, _maps(res, text, 12), FRAMES)
    with pytest.raises(FlowtronB200Error):                       # shorter maps are fine when no row needs more
        cpu_model.infer_aligned(res, spk, text, IN_LENS, _maps(res, text, 12), torch.tensor([12, 7, 9]))
    with pytest.raises(FlowtronB200Error):                       # texts past 256 tokens are accepted
        cpu_model.infer_aligned(res, spk, _text(300), [300, 4, 4], _maps(res, _text(300)), FRAMES)


def test_infer_durations_arguments(cpu_model):
    res, spk, text = torch.zeros(B, 80, T), _spk(), _text()
    dur = torch.tensor([[2] * 9, [3, 1, 1, 2] + [0] * 5, [1] * 6 + [0] * 3])
    bad = [
        dur.float(),
        dur[:2],
        dur[:, :8],
        dur.tolist(),
        torch.cat([dur[:2], -dur[2:]]),                                     # negative
        torch.cat([dur[:2], torch.zeros(1, L, dtype=torch.long)]),         # an empty row
        torch.cat([dur[:1] * 2, dur[1:]]),                                  # 36 frames > T
    ]
    for d in bad:
        with pytest.raises(ValueError, match="durations"):
            cpu_model.infer_durations(res, spk, text, IN_LENS, d)
    with pytest.raises(FlowtronB200Error):
        cpu_model.infer_durations(res, spk, text, IN_LENS, dur)
