"""CPU: the float32 MAS restatement (oracle/align_oracle.py) on hand-worked cases and against exhaustive search, its
one-hot maps, the argument checks of align.mas / align.hard_attention, and the register budget of the alignment kernels."""
import itertools
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from conftest import ROOT
from oracle import align_oracle as O

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
HAVE_NVCC = os.path.exists(NVCC) or shutil.which("nvcc") is not None


def _one(s, reversed_=False):
    s = np.asarray(s, dtype=np.float32)
    d, tok = O.mas(s[None], [s.shape[1]], [s.shape[0]], reversed_)
    return d[0], tok[0]


def test_oracle_hand_worked_path():
    # paths 0,0,1 (0 - 1 - 0.5 = -1.5) and 0,1,1 (0 - 2 - 0.5 = -2.5): the first wins
    d, tok = _one([[0.0, -5.0], [-1.0, -2.0], [-3.0, -0.5]])
    assert tok.tolist() == [0, 0, 1] and d.tolist() == [2, 1]


def test_oracle_diagonal_map():
    T, L = 12, 4
    s = np.full((T, L), -10.0, dtype=np.float32)
    for t in range(T):
        s[t, t * L // T] = 0.0                  # three frames per token
    d, tok = _one(s)
    assert d.tolist() == [3, 3, 3, 3]
    assert tok.tolist() == [t * L // T for t in range(T)]


@pytest.mark.parametrize("c", [0.0, -1.25, 3.0])
def test_oracle_exact_ties_stay_on_the_token(c):
    """Uniform rows: every path ties, and the walk back moves only when it must, so the last token takes the slack."""
    T, L = 9, 5
    d, tok = _one(np.full((T, L), c))
    assert d.tolist() == [1, 1, 1, 1, T - L + 1]
    assert tok.tolist() == [0, 1, 2, 3] + [4] * (T - L + 1)


def test_oracle_one_frame_per_token_and_no_path():
    g = np.random.default_rng(0)
    d, tok = _one(g.standard_normal((6, 6)))
    assert d.tolist() == [1] * 6 and tok.tolist() == list(range(6))
    s = g.standard_normal((2, 5, 7)).astype(np.float32)
    d, tok = O.mas(s, [7, 3], [5, 5])            # row 0: 5 frames, 7 tokens
    assert (d[0] == 0).all() and (tok[0] == -1).all()
    assert d[1, :3].sum() == 5 and (d[1, 3:] == 0).all() and (d[1, :3] >= 1).all()


def test_oracle_finds_the_best_path():
    """Against exhaustive search over every monotonic path (random inputs: no ties)."""
    g = np.random.default_rng(1)
    for T, L in [(1, 1), (4, 1), (5, 2), (6, 3), (7, 4), (8, 5)]:
        for _ in range(3):
            s = g.standard_normal((T, L)).astype(np.float32)
            best, arg = -np.inf, None
            for steps in itertools.combinations(range(1, T), L - 1):     # frames at which the token advances
                tok = np.cumsum([1 if t in steps else 0 for t in range(T)])
                v = float(s[np.arange(T), tok].astype(np.float64).sum())
                if v > best:
                    best, arg = v, tok
            d, tok = _one(s)
            assert tok.tolist() == arg.tolist(), (T, L)
            assert d.sum() == T and (d >= 1).all()


def test_oracle_reversed_rows_and_padding():
    g = np.random.default_rng(2)
    B, T, L = 3, 20, 7
    lp = g.standard_normal((B, T, L)).astype(np.float32)
    in_lens, out_lens = [7, 3, 5], [20, 9, 14]
    flipped = np.full_like(lp, np.nan)
    for b in range(B):
        flipped[b, :out_lens[b], :in_lens[b]] = lp[b, :out_lens[b], :in_lens[b]][::-1]
    d0, t0 = O.mas(lp, in_lens, out_lens)
    d1, t1 = O.mas(flipped, in_lens, out_lens, time_reversed=True)
    assert (d0 == d1).all() and (t0 == t1).all()
    for b in range(B):
        assert d0[b].sum() == out_lens[b] and (t0[b, out_lens[b]:] == -1).all() and (d0[b, in_lens[b]:] == 0).all()


def test_oracle_hard_attention_is_one_hot_of_the_path():
    g = np.random.default_rng(3)
    B, T, L = 2, 15, 6
    lp = g.standard_normal((B, T, L)).astype(np.float32)
    in_lens, out_lens = [6, 4], [15, 10]
    d, tok = O.mas(lp, in_lens, out_lens)
    fwd = O.hard_attention(d, in_lens, T)
    back = O.hard_attention(d, in_lens, T, time_reversed=True)
    for b in range(B):
        n = out_lens[b]
        ref = np.zeros((T, L), dtype=np.float32)
        ref[np.arange(n), tok[b, :n]] = 1.0
        assert (fwd[b] == ref).all()
        assert (back[b, :n] == ref[:n][::-1]).all() and (back[b, n:] == 0).all()


def test_mas_and_hard_attention_argument_validation():
    from flowtron_b200 import align
    from flowtron_b200._lib import FlowtronB200Error
    lp = torch.zeros(3, 20, 9)
    ok = dict(in_lens=[9, 4, 4], out_lens=[20, 7, 13])
    bad = [
        dict(ok, in_lens=[9, 4]),
        dict(ok, in_lens=[9, 0, 4]),
        dict(ok, in_lens=[9, 10, 4]),
        dict(ok, in_lens=[9.0, 4.0, 4.0]),
        dict(ok, out_lens=[20, 21, 13]),
        dict(ok, out_lens=[20, 0, 13]),
        dict(ok, out_lens=[20, 3, 13]),                          # 3 frames for 4 tokens
    ]
    for kw in bad:
        with pytest.raises(ValueError):
            align.mas(lp, **kw)
    for x in (torch.zeros(20, 9), torch.zeros(3, 20, 9, dtype=torch.long), torch.zeros(0, 20, 9)):
        with pytest.raises(ValueError):
            align.mas(x, **ok)
    with pytest.raises(ValueError, match="1024"):
        align.mas(torch.zeros(1, 2000, 1025), [1025], [2000])
    with pytest.raises(FlowtronB200Error):
        align.mas(lp, **ok)
    dur = torch.ones(3, 9, dtype=torch.long)
    for args in [(dur.float(), [9, 4, 4], 20), (dur[0], [9, 4, 4], 20), (dur, [9, 4], 20), (dur, [9, 4, 10], 20),
                 (dur, [9, 4, 4], 0), (dur, [9, 4, 4], 2.5)]:
        with pytest.raises(ValueError):
            align.hard_attention(*args)
    with pytest.raises(FlowtronB200Error):
        align.hard_attention(dur, [9, 4, 4], 20)


@pytest.mark.skipif(not HAVE_NVCC, reason="nvcc not available")
def test_alignment_kernels_do_not_spill(tmp_path):
    r = subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr",
                        "-Xptxas", "-v", "-c", os.path.join(ROOT, "flowtron_b200", "csrc", "align.cu"), "-o",
                        str(tmp_path / "align.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    logs = {}
    for part in r.stderr.split("Compiling entry function")[1:]:
        logs[re.match(r"\s*'(\S+)'", part).group(1)] = part
    want = [k for k in logs if "mas_kernel" in k or "durations_to_attn_kernel" in k]
    assert len(want) == 3, sorted(logs)
    for k in want:
        regs = int(re.search(r"Used (\d+) registers", logs[k]).group(1))
        spill = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", logs[k])
        assert regs <= 255 and spill.groups() == ("0", "0"), logs[k]
