"""CPU: the mixture-synthesis oracle against the unmodified reference (tests/make_golden_gmm_sample.py), the sampler's counter
hash, the responsibilities' normalisation and log normaliser, and the argument checks of Flowtron.mixture,
style.sample_mixture and style.gmm_responsibilities, all raised before any device work."""
import os

import numpy as np
import pytest
import torch

import gmm_sample_oracle as O
from conftest import GOLDEN
from flowtron_b200 import synth

CASES = ["gmm_sample_learned", "gmm_sample_fixed"]


def _case(name):
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=2, n_components=int(g["K"]), fixed_gaussian=bool(g["fixed_gaussian"]),
               mean_scale=float(g["mean_scale"]))
    return g, cfg, synth.synth_gmm_params(cfg, int(g["seed"]))


@pytest.mark.parametrize("name", CASES)
def test_oracle_mixture_matches_the_reference_one_utterance_at_a_time(name):
    g, cfg, params = _case(name)
    emb, mean, log_var, prob = O.mixture(params, torch.from_numpy(g["mel"]), g["out_lens"], cfg["n_components"],
                                         cfg["fixed_gaussian"])
    for key, got in (("mel_embedding", emb), ("mean", mean), ("log_var", log_var), ("prob", prob)):
        ref = torch.from_numpy(g[key]).double()
        assert got.shape == ref.shape, key
        scale = max(ref.abs().max().item(), 1e-30)
        assert (got - ref).abs().max().item() <= 1e-5 * scale, (key, (got - ref).abs().max().item() / scale)
    assert len(set(g["out_lens"].tolist())) == len(g["out_lens"])         # rows of different lengths


@pytest.mark.parametrize("name", CASES)
def test_responsibilities_normalise_and_their_log_normaliser_is_the_reference_nll(name):
    g, _, _ = _case(name)
    lens = g["out_lens"]
    r, lse = O.responsibilities(g["z"], lens, g["mean"], g["log_var"], g["prob"])
    assert np.allclose(r.sum(1), 1.0, rtol=0, atol=1e-12)
    assert (r >= 0).all()
    # FlowtronLoss(gm_loss=True) with zero log_s: -sum_valid lse / (n_valid * 80)
    nll = -lse.sum() / (lens.sum() * 80)
    assert abs(nll - float(g["loss"])) <= 2e-6 * abs(float(g["loss"])), (nll, float(g["loss"]))


def test_counter_hash_reproduces_known_words():
    # words of the splitmix64 finaliser over (seed, counter, element), worked out with Python integers
    assert O.hash3(0, 0, 0) == 0xE220A839
    assert O.hash3(1, 0, 0) == 0x910A2DEC
    assert O.hash3(0x1234, 7, 5) == 0x89BCD30C
    assert O.hash3(0, 0, np.array([0, 1, 2], dtype=np.uint64)).tolist() == [0xE220A839, 0x2D0F28C7, 0x3C5B6687]


def test_oracle_draw_depends_only_on_the_element():
    gen = np.random.default_rng(3)
    K, T = 4, 20
    mean = gen.normal(size=(3, 80, K)).astype(np.float32)
    log_var = gen.normal(size=(3, 80, K)).astype(np.float32) * 0.3
    prob = np.full((3, K), 0.25, dtype=np.float32)
    z3, k3 = O.sample(mean, log_var, prob, [20, 7, 13], T, 0.8, 11, 5)
    z1, k1 = O.sample(mean[:1], log_var[:1], prob[:1], [20], T + 9, 0.8, 11, 5)
    assert np.array_equal(z3[0], z1[0, :, :T]) and np.array_equal(k3[0], k1[0, :, :T])
    assert (z3[1, :, 7:] == 0).all() and (k3[1, :, 7:] == -1).all()
    z_next, _ = O.sample(mean, log_var, prob, [20, 7, 13], T, 0.8, 11, 6)
    assert not np.array_equal(z3[0], z_next[0])
    one_hot = np.zeros((3, K), dtype=np.float32)
    one_hot[:, 2] = 1.0
    _, k = O.sample(mean, log_var, one_hot, [20, 7, 13], T, 1.0, 11, 5)
    assert set(np.unique(k[k >= 0]).tolist()) == {2}
    _, k = O.sample(mean, log_var, prob, [20, 7, 13], T, 1.0, 11, 5, component=[1, -1, 3])
    assert (k[0, :, :20] == 1).all() and (k[2, :, :13] == 3).all() and len(np.unique(k[1, :, :7])) > 1


def _mixture_inputs(B=2, K=4, per_row=True):
    mean = torch.zeros(B if per_row else 1, 80, K)
    return mean, torch.zeros_like(mean), torch.full((B, K), 1.0 / K)


def test_sample_mixture_rejects_bad_arguments_before_device_work():
    from flowtron_b200 import style
    from flowtron_b200._lib import FlowtronB200Error
    mean, log_var, prob = _mixture_inputs()
    bad = [
        dict(mean=mean[:, :, :3]),                            # K disagrees with prob
        dict(log_var=log_var[:1]),                             # mean and log_var differ
        dict(mean=torch.zeros(3, 80, 4), log_var=torch.zeros(3, 80, 4)),   # neither per-row nor shared
        dict(mean=torch.zeros(2, 81, 4), log_var=torch.zeros(2, 81, 4)),   # more than 80 channels
        dict(prob=torch.full((3, 4), 0.25)),                   # prob of the wrong size
        dict(prob=torch.full((2,), 0.5)),
        dict(mean=torch.zeros(2, 80, 33), log_var=torch.zeros(2, 80, 33), prob=torch.full((2, 33), 1 / 33)),   # K > 32
        dict(component=[0, 4]),                                # component out of range
        dict(component=[0, -2]),
        dict(component=[0]),
        dict(component=[0.0, 1.0]),
        dict(n_frames=[5, 11]),                                # past T
        dict(n_frames=[5, 0]),
        dict(n_frames=[5]),
        dict(T=0),
        dict(sigma=-1.0),
        dict(sigma=float("nan")),
        dict(rng_state=torch.zeros(3, dtype=torch.int64)),
    ]
    for kw in bad:
        args = dict(mean=mean, log_var=log_var, prob=prob, n_frames=[5, 10], T=10)
        args.update(kw)
        with pytest.raises(ValueError):
            style.sample_mixture(**args)
    with pytest.raises(FlowtronB200Error):                     # valid shapes, CPU tensors
        style.sample_mixture(mean, log_var, prob, [5, 10], 10, component=[-1, 3])


def test_gmm_responsibilities_rejects_bad_arguments_before_device_work():
    from flowtron_b200 import style
    from flowtron_b200._lib import FlowtronB200Error
    mean, log_var, prob = _mixture_inputs(per_row=False)
    z = torch.zeros(2, 80, 10)
    bad = [
        dict(z=torch.zeros(80, 10)),
        dict(z=torch.zeros(2, 40, 10)),                        # channels disagree with mean
        dict(prob=torch.full((3, 4), 0.25)),
        dict(mean=torch.zeros(1, 80, 5), log_var=torch.zeros(1, 80, 5)),
        dict(mean=torch.zeros(1, 80, 33), log_var=torch.zeros(1, 80, 33), prob=torch.full((2, 33), 1 / 33)),
        dict(out_lens=[3, 11]),
        dict(out_lens=[0, 4]),
    ]
    for kw in bad:
        args = dict(z=z, out_lens=[3, 10], mean=mean, log_var=log_var, prob=prob)
        args.update(kw)
        with pytest.raises(ValueError):
            style.gmm_responsibilities(**args)
    with pytest.raises(FlowtronB200Error):
        style.gmm_responsibilities(z, [3, 10], mean, log_var, prob)


def test_mixture_rejects_bad_arguments_and_models_without_a_mixture():
    from flowtron_b200._lib import FlowtronB200Error
    from flowtron_b200.flowtron import Flowtron
    cfg = dict(synth.DEFAULT_MODEL_CONFIG, n_flows=2, n_components=4, fixed_gaussian=False, mean_scale=0.0)
    m = Flowtron(**cfg)
    mel = torch.zeros(2, 80, 12)
    for bad_mel, lens in ((torch.zeros(80, 12), [12, 5]), (torch.zeros(2, 40, 12), [12, 5]), (mel, [12, 13]),
                          (mel, [0, 5]), (mel, [12]), (mel, [1.5, 2.0])):
        with pytest.raises(ValueError):
            m.mixture(bad_mel, lens)
    with pytest.raises(FlowtronB200Error):
        m.mixture(mel, [12, 5])
    plain = Flowtron(**dict(cfg, n_components=0))
    with pytest.raises(ValueError, match="mixture"):
        plain.mixture(mel, [12, 5])


def test_abi_symbols_are_declared_and_exported():
    import re
    from conftest import ROOT
    from flowtron_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "flowtron_b200.h")).read()
    L = _lib.lib()
    for sym in ("ft_gmm_sample", "ft_gmm_responsibilities"):
        assert re.search(r"\b" + sym + r"\(", hdr), sym
        assert hasattr(L, sym), sym
