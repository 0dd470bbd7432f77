"""GPU: hard alignments -- align.mas (ft_mas_align) identical to the float32 restatement in oracle/align_oracle.py on ragged,
tied, long and time-reversed inputs; align.hard_attention (ft_durations_to_attn); Flowtron.align against the oracle on each
row's own B = 1 forward; Flowtron.infer_durations against infer_aligned with maps built in numpy."""
import numpy as np
import pytest
import torch

from conftest import record_parity
from flowtron_b200 import synth
from oracle import align_oracle as O

pytestmark = pytest.mark.gpu


def _logp(seed, B, T, L, ties=False):
    """Attention-like log-probabilities [B, T, L]: log_softmax of random scores, or small integers when `ties`."""
    g = torch.Generator().manual_seed(seed)
    if ties:
        return torch.randint(-2, 1, (B, T, L), generator=g).float()
    return torch.log_softmax(3.0 * torch.randn(B, T, L, generator=g), -1)


def _lens(seed, B, T, L):
    g = np.random.default_rng(seed)
    in_lens = g.integers(1, L + 1, B)
    out_lens = np.array([g.integers(n, T + 1) for n in in_lens])
    in_lens[0], out_lens[-1] = L, T                              # the padded sizes are reached; order is unsorted
    return in_lens.tolist(), out_lens.tolist()


def _flip_rows(lp, in_lens, out_lens, fill):
    """Each row's valid block in flipped time (row q = natural frame out_lens[b]-1-q), `fill` elsewhere."""
    out = torch.full_like(lp, fill)
    for b, (nl, nt) in enumerate(zip(in_lens, out_lens)):
        out[b, :nt, :nl] = lp[b, :nt, :nl].flip(0)
    return out


def _padded(lp, in_lens, out_lens, fill):
    out = torch.full_like(lp, fill)
    for b, (nl, nt) in enumerate(zip(in_lens, out_lens)):
        out[b, :nt, :nl] = lp[b, :nt, :nl]
    return out


CASES = {                       # name: (B, T, L, ties)
    "b1_l1": (1, 37, 1, False),
    "b40_ragged": (40, 300, 90, False),
    "l256": (6, 700, 256, False),
    "l257": (6, 700, 257, False),
    "l1024": (3, 2100, 1024, False),
    "t4096": (2, 4096, 400, False),
    "ties": (12, 200, 60, True),
}


@pytest.mark.parametrize("reversed_", [False, True])
@pytest.mark.parametrize("name", sorted(CASES))
def test_mas_matches_the_oracle(name, reversed_):
    from flowtron_b200 import _lib, align
    B, T, L, ties = CASES[name]
    seed = sorted(CASES).index(name)
    lp = _logp(seed, B, T, L, ties)
    in_lens, out_lens = _lens(seed + 100, B, T, L)
    if ties:
        lp[0] = -1.0
        in_lens[0], out_lens[0] = L, T
    if name == "b1_l1":
        in_lens, out_lens = [1], [T]
    ref_d, ref_t = O.mas(lp.numpy(), in_lens, out_lens)
    x = _flip_rows(lp, in_lens, out_lens, float("nan")) if reversed_ else _padded(lp, in_lens, out_lens, float("nan"))
    d, tok = align.mas(x.cuda(), in_lens, out_lens, time_reversed=reversed_)
    torch.cuda.synchronize()
    assert _lib.device_status() == 0
    assert d.dtype == tok.dtype == torch.int64 and tuple(d.shape) == (B, L) and tuple(tok.shape) == (B, T)
    bad = [b for b in range(B) if not (np.array_equal(d[b].cpu().numpy(), ref_d[b])
                                       and np.array_equal(tok[b].cpu().numpy(), ref_t[b]))]
    record_parity(f"mas_{name}_{'rev' if reversed_ else 'fwd'}", {"rows": B, "rows_differing": len(bad)})
    assert not bad, bad
    assert d.sum(1).tolist() == out_lens and bool((d[:, :1] >= 1).all())
    if ties:                     # row 0 is uniform: every path ties and the last token takes the slack
        assert d[0].tolist() == [1] * (L - 1) + [T - L + 1]


def test_mas_rows_without_a_path_and_padding_values():
    """CUDA lengths with fewer frames than tokens give zero durations and -1; what lies outside the lengths is never read."""
    from flowtron_b200 import align
    B, T, L = 4, 50, 30
    lp = _logp(7, B, T, L)
    in_lens, out_lens = [30, 12, 20, 5], [50, 11, 40, 5]
    ref_d, ref_t = O.mas(lp.numpy(), in_lens, out_lens)
    outs = []
    for fill in (0.0, float("nan"), float("inf"), -float("inf")):
        outs.append(align.mas(_padded(lp, in_lens, out_lens, fill).cuda(), torch.tensor(in_lens, device="cuda"),
                              torch.tensor(out_lens, device="cuda")))
    for d, tok in outs:
        assert np.array_equal(d.cpu().numpy(), ref_d) and np.array_equal(tok.cpu().numpy(), ref_t)
    assert (outs[0][0][1] == 0).all() and (outs[0][1][1] == -1).all()


def test_mas_graph_replay_equals_eager():
    from flowtron_b200 import align
    B, T, L = 16, 600, 300
    lp = _logp(11, B, T, L).cuda()
    in_lens, out_lens = _lens(12, B, T, L)
    il, ol = torch.tensor(in_lens, device="cuda"), torch.tensor(out_lens, device="cuda")
    eager = align.mas(lp, il, ol, time_reversed=True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        align.mas(lp, il, ol, time_reversed=True)                 # warm-up on the capture stream: scratch is allocated
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            out = align.mas(lp, il, ol, time_reversed=True)
    torch.cuda.current_stream().wait_stream(s)
    for _ in range(2):
        graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out[0], eager[0]) and torch.equal(out[1], eager[1])


@pytest.mark.parametrize("reversed_", [False, True])
def test_hard_attention_matches_the_oracle(reversed_):
    from flowtron_b200 import align
    g = torch.Generator().manual_seed(21)
    B, L = 9, 700
    in_lens = torch.randint(1, L + 1, (B,), generator=g)
    in_lens[3] = L
    dur = torch.randint(0, 4, (B, L), generator=g)
    dur[5] = torch.randint(1, 9, (L,), generator=g)              # longer than Ta: cut
    dur[1, 0] = 25
    Ta = int(dur.sum(1).max()) - 40
    ref = O.hard_attention(dur.numpy(), in_lens.tolist(), Ta, reversed_)
    out = align.hard_attention(dur.cuda(), in_lens.tolist(), Ta, time_reversed=reversed_)
    assert np.array_equal(out.cpu().numpy(), ref)
    out_dev = align.hard_attention(dur.cuda().int(), in_lens.cuda(), Ta, time_reversed=reversed_)
    assert torch.equal(out_dev, out)


def _model(n_flows, seed):
    from flowtron_b200.flowtron import Flowtron
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=n_flows, n_speakers=2)
    m = Flowtron(**cfg)
    m.load_state_dict(synth.synth_params(cfg, seed), strict=True)
    return m.cuda().eval(), cfg


@pytest.mark.parametrize("prior", [False, True])
@pytest.mark.parametrize("n_flows", [2, 3])
def test_flowtron_align_rows_match_the_oracle_on_their_own_forward(n_flows, prior):
    from flowtron_b200 import _lib
    from flowtron_b200.align import hard_attention
    from flowtron_b200.flowtron import AR_Back_Step
    m, cfg = _model(n_flows, 40 + n_flows)
    B, T, L = 4, 340, 30
    bt = synth.synth_batch(B, T, L, cfg, 5 + n_flows, out_lens=[90, 340, 41, 200], in_lens=[22, 30, 9, 25], with_prior=True,
                           logmel_stats=True)
    perm = [2, 0, 3, 1]                                          # unsorted rows; one past the 320-frame split
    out_lens, in_lens = bt["out_lens"][perm].tolist(), bt["in_lens"][perm].tolist()
    mel, text, spk = bt["mel"][perm].cuda(), bt["text"][perm].cuda(), bt["speaker_ids"][perm].cuda()
    pr = bt["attn_prior"][perm].cuda() if prior else None
    errs = {}
    for f in range(n_flows):
        d, tok = m.align(mel, spk, text, in_lens, out_lens, attn_prior=pr, flow=f)
        assert d.sum(1).tolist() == out_lens
        rev = isinstance(m.flows[f], AR_Back_Step)
        maps = hard_attention(d, in_lens, T, time_reversed=rev)
        for b in range(B):
            nl, nt = in_lens[b], out_lens[b]
            with torch.no_grad():
                out = m(mel[b:b + 1, :, :nt].contiguous(), spk[b:b + 1], text[b:b + 1, :nl].contiguous(),
                        torch.tensor([nl], device="cuda"), torch.tensor([nt], device="cuda"),
                        None if pr is None else pr[b:b + 1, :nt, :nl].contiguous())
            rd, rt = O.mas(out[4][f].float().cpu().numpy(), [nl], [nt], time_reversed=rev)
            assert np.array_equal(d[b, :nl].cpu().numpy(), rd[0]) and (d[b, nl:] == 0).all(), (f, b)
            assert np.array_equal(tok[b, :nt].cpu().numpy(), rt[0]) and (tok[b, nt:] == -1).all(), (f, b)
            d1, t1 = m.align(mel[b:b + 1, :, :nt].contiguous(), spk[b:b + 1], text[b:b + 1, :nl].contiguous(), [nl], [nt],
                             None if pr is None else pr[b:b + 1, :nt, :nl].contiguous(), flow=f)
            assert torch.equal(d1[0], d[b, :nl]) and torch.equal(t1[0], tok[b, :nt]), (f, b)
            onehot = torch.zeros(T, L, device="cuda")
            onehot[torch.arange(nt, device="cuda"), tok[b, :nt]] = 1.0
            ref_map = torch.cat([onehot[:nt].flip(0), onehot[nt:]]) if rev else onehot
            assert torch.equal(maps[b], ref_map), (f, b)
        errs[f"flow{f}_rows"] = B
    torch.cuda.synchronize()
    assert _lib.device_status() == 0
    record_parity(f"flowtron_align_f{n_flows}_{'prior' if prior else 'noprior'}", errs)


def test_infer_durations_equals_infer_aligned_on_numpy_maps():
    from flowtron_b200 import _lib
    from flowtron_b200.flowtron import AR_Back_Step
    m, _ = _model(3, 51)
    B, T, L = 5, 120, 24
    g = torch.Generator().manual_seed(52)
    res = (torch.randn(B, 80, T, generator=g) * 0.5).cuda()
    text = torch.randint(0, 185, (B, L), generator=g).cuda()
    spk = torch.randint(0, 2, (B,), generator=g).cuda()
    in_lens = [24, 7, 15, 3, 20]
    dur = torch.zeros(B, L, dtype=torch.long)
    for b, n in enumerate(in_lens):
        dur[b, :n] = torch.randint(1, 5, (n,), generator=g)
    n_frames = dur.sum(1).tolist()
    assert max(n_frames) + 4 <= T                                # room for the doubled token below
    maps = [torch.from_numpy(O.hard_attention(dur.numpy(), in_lens, T, isinstance(f, AR_Back_Step))).cuda() for f in m.flows]
    ref, ref_lens = m.infer_aligned(res, spk, text, in_lens, maps, n_frames)
    mel, mel_lens = m.infer_durations(res, spk, text, in_lens, dur.cuda())
    mel_h, _ = m.infer_durations(res, spk, text, in_lens, dur)
    torch.cuda.synchronize()
    assert _lib.device_status() == 0
    assert mel_lens.tolist() == ref_lens.tolist() == n_frames
    assert torch.equal(mel, ref) and torch.equal(mel_h, ref)
    # doubling one token's duration lengthens that row by exactly that many frames and leaves the others alone
    k, b = 2, 2
    dur2 = dur.clone()
    dur2[b, k] *= 2
    mel2, lens2 = m.infer_durations(res, spk, text, torch.tensor(in_lens, device="cuda"), dur2.cuda())
    torch.cuda.synchronize()
    assert lens2[b].item() == n_frames[b] + int(dur[b, k]) and (mel2[b, :, lens2[b]:] == 0).all()
    for r in range(B):
        if r != b:
            assert lens2[r].item() == n_frames[r] and torch.equal(mel2[r], mel[r]), r
    record_parity("infer_durations", {"rows": B, "bit_identical": 1})
