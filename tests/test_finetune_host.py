"""CPU: the dependency rule of a flow step's backward (ft_ar_step_bwd_plan), which decides what the two backward calls
launch when only some parameter gradients, d_text or d_mel are wanted (fine-tuning a subset of the model)."""
import pytest

from flowtron_b200 import _lib

FIELDS = _lib.AR_WEIGHT_FIELDS
CHAIN = {"COUPLING", "CONV_DGRAD", "DENSE1_DGRAD", "DENSE0_DGRAD", "LSTM1", "LSTM0"}    # loss scale down to dd = dG0 W_ih0
WGRADS = {k for k in _lib.BWD_STAGES if k.startswith("G_")}
GROUPS = {                        # parameter group -> (its fields, its G_ bit)
    "attention_lstm": ([f for f in FIELDS if f.startswith("attn_lstm_")], "G_ATTN_LSTM"),
    "lstm_l0": (["lstm_w_ih0", "lstm_w_hh0", "lstm_b_ih0", "lstm_b_hh0"], "G_LSTM0"),
    "lstm_l1": (["lstm_w_ih1", "lstm_w_hh1", "lstm_b_ih1", "lstm_b_hh1"], "G_LSTM1"),
    "query": (["att_query"], "G_QUERY"),
    "key": (["att_key"], "G_KEY"),
    "value": (["att_value"], "G_VALUE"),
    "v": (["att_v"], "G_V"),
    "dense_0": (["dense_w0", "dense_b0"], "G_DENSE0"),
    "dense_1": (["dense_w1", "dense_b1"], "G_DENSE1"),
    "conv": (["conv_w", "conv_b"], "G_CONV"),
    "gate": (["gate_w", "gate_b"], "G_GATE"),
}


def _desc(gate=True):
    return _lib.FtArStepDesc(1000, 32, 160, 80, 1024, 640, 640, 0, int(gate), 1, 1.0)


def _plan(fields=(), d_text=False, d_mel=False, gate=True):
    want = [f in fields for f in FIELDS]
    return _lib.ar_step_bwd_plan(_desc(gate), want, d_text, d_mel)


def test_everything_wanted_runs_every_stage():
    assert _plan(FIELDS, True, True) == set(_lib.BWD_STAGES)
    assert _plan(FIELDS, True, True, gate=False) == set(_lib.BWD_STAGES) - {"GATE_DD", "G_GATE"}


def test_nothing_wanted_runs_nothing():
    assert _plan() == set()
    assert _plan(["gate_w", "gate_b"], gate=False) == set()       # a flow without a gate ignores gate entries


@pytest.mark.parametrize("fields", [["gate_w", "gate_b"], ["gate_w"], ["gate_b"]])
def test_gate_only_is_the_gate_parameter_stage(fields):
    assert _plan(fields) == {"G_GATE"}


def test_speaker_style_step_skips_the_attention_lstm_and_every_weight_gradient():
    m = _plan(d_text=True)
    assert m == CHAIN | {"GATE_DD", "ATTN", "D_TEXT"}
    assert not m & ({"ATTN_LSTM", "QUERY_DGRAD", "D_MEL"} | WGRADS)


def test_d_mel_alone_runs_the_full_bptt_chain_without_weight_gradients():
    m = _plan(d_mel=True)
    assert m == CHAIN | {"GATE_DD", "ATTN", "QUERY_DGRAD", "ATTN_LSTM", "D_MEL"}
    assert _plan(d_mel=True, gate=False) == m - {"GATE_DD"}


EXPECTED = {                      # group -> stages beside its own G_ bit
    "attention_lstm": CHAIN | {"GATE_DD", "ATTN", "QUERY_DGRAD", "ATTN_LSTM"},
    "lstm_l0": set(CHAIN),
    "lstm_l1": {"COUPLING", "CONV_DGRAD", "DENSE1_DGRAD", "DENSE0_DGRAD", "LSTM1"},
    "query": CHAIN | {"GATE_DD", "ATTN"},
    "key": CHAIN | {"GATE_DD", "ATTN"},
    "value": CHAIN | {"GATE_DD", "ATTN"},
    "v": CHAIN | {"GATE_DD", "ATTN"},
    "dense_0": {"COUPLING", "CONV_DGRAD", "DENSE1_DGRAD"},
    "dense_1": {"COUPLING", "CONV_DGRAD"},
    "conv": {"COUPLING"},
    "gate": set(),
}


@pytest.mark.parametrize("group", list(GROUPS))
def test_each_parameter_group_turns_on_exactly_its_chain(group):
    fields, bit = GROUPS[group]
    assert _plan(fields) == EXPECTED[group] | {bit}
    for f in fields:                          # one member of the group asks for the same work
        assert _plan([f]) == EXPECTED[group] | {bit}
    if group != "gate":
        assert _plan(fields, gate=False) == (EXPECTED[group] | {bit}) - {"GATE_DD"}


def test_stages_are_monotone_in_what_is_wanted():
    """Wanting more never runs less: the union of two requests plans at least the union of their plans."""
    reqs = [(GROUPS[g][0], False, False) for g in GROUPS] + [((), True, False), ((), False, True)]
    for a in reqs:
        for b in reqs:
            both = _plan(list(a[0]) + list(b[0]), a[1] or b[1], a[2] or b[2])
            assert _plan(*a) | _plan(*b) <= both


def test_plan_rejects_null_arguments():
    from ctypes import byref, c_uint
    L = _lib.lib()
    m = c_uint(0)
    assert L.ft_ar_step_bwd_plan(None, byref(_lib.FtArStepWeights()), 1, 1, byref(m)) != 0
    assert L.ft_ar_step_bwd_plan(byref(_desc()), None, 1, 1, byref(m)) != 0
    assert L.ft_ar_step_bwd_plan(byref(_desc()), byref(_lib.FtArStepWeights()), 1, 1, None) != 0
