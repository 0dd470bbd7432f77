"""CPU: the Gaussian-mixture prior's host layer (MelEncoder, GaussianMixture, Flowtron(n_components > 1),
FlowtronLoss(gm_loss=True)): state_dict layout against the reference fixtures, strict loads, CPU-tensor and K > 32 rejections,
the C ABI of the mel-encoder and mixture-NLL kernels, both encoders' kernels unchanged by sharing their device and host
code, and the byte layouts of both encoders' saved / scratch buffers."""
import os
import re

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT
from flowtron_b200 import synth
from kernel_pins import HAVE_NVCC, _assert_kernels_pinned, _compile


def _cfg(K=8, fixed=True, mean_scale=3.0, n_flows=2):
    return dict(synth.DEFAULT_MODEL_CONFIG, n_flows=n_flows, n_components=K, fixed_gaussian=fixed, mean_scale=mean_scale)


@pytest.mark.parametrize("fixed", [True, False])
def test_state_dict_keys_and_shapes(fixed):
    from flowtron_b200.flowtron import Flowtron
    cfg = _cfg(K=8, fixed=fixed)
    sd = Flowtron(**cfg).state_dict()
    want = dict(synth.param_shapes(dict(cfg, n_components=0)), **synth.gmm_param_shapes(cfg))
    if fixed:
        want["gaussian_mixture.mean"] = (1, 80, 8)
        want["gaussian_mixture.log_var"] = (1, 80, 8)
        assert "gaussian_mixture.mean_layer.linear_layer.weight" not in sd
    else:
        assert want["gaussian_mixture.mean_layer.linear_layer.weight"] == (640, 512)
    assert {k: tuple(v.shape) for k, v in sd.items()} == want
    assert want["mel_encoder.convolutions.0.0.conv.weight"] == (512, 80, 3)
    assert want["mel_encoder.convolutions.1.0.conv.weight"] == (512, 512, 3)


def test_fixed_means_are_scaled_unit_vectors():
    from flowtron_b200.flowtron import Flowtron
    m = Flowtron(**_cfg(K=8, fixed=True, mean_scale=3.0)).gaussian_mixture.mean
    assert m.shape == (1, 80, 8)
    assert torch.equal((m != 0).sum(1), torch.ones(1, 8, dtype=torch.long)) and torch.all(m.sum(1) == 3.0)
    assert len(set(m[0].argmax(0).tolist())) == 8


@pytest.mark.parametrize("name", ["gmm_f2_fixed", "gmm_f3_learned", "gmm_b1_learned", "gmm_b1_fixed"])
def test_reference_key_set_loads_strict_both_ways(name):
    from flowtron_b200.flowtron import Flowtron
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    cfg = _cfg(K=int(g["K"]), fixed=bool(g["fixed_gaussian"]), mean_scale=float(g["mean_scale"]), n_flows=int(g["n_flows"]))
    params = synth.synth_gmm_params(cfg, int(g["seed"]))
    assert sorted(params) == sorted(g["state_keys"].tolist())        # the reference model's own state_dict keys
    m = Flowtron(**cfg)
    m.load_state_dict(params, strict=True)
    back = Flowtron(**cfg)
    back.load_state_dict(m.state_dict(), strict=True)
    if cfg["fixed_gaussian"]:
        assert torch.equal(back.gaussian_mixture.mean, torch.from_numpy(g["fixed_mean"]))


def test_sizes_the_kernels_are_not_built_for_raise():
    from flowtron_b200.flowtron import MelEncoder, MaskedInstanceNorm1d
    MelEncoder(512)
    for kw in (dict(encoder_embedding_dim=256), dict(encoder_kernel_size=5), dict(encoder_n_convolutions=3),
               dict(norm_fn=torch.nn.BatchNorm1d)):
        with pytest.raises(NotImplementedError):
            MelEncoder(**dict(dict(norm_fn=MaskedInstanceNorm1d), **kw))
    with pytest.raises(NotImplementedError):
        MelEncoder().infer(torch.zeros(1, 80, 4))


def test_cpu_tensors_raise():
    from flowtron_b200._lib import FlowtronB200Error
    from flowtron_b200.flowtron import Flowtron, FlowtronLoss
    cfg = _cfg(K=4, fixed=False)
    m = Flowtron(**cfg)
    with pytest.raises(FlowtronB200Error):
        m.mel_encoder(torch.zeros(2, 80, 8), torch.tensor([8, 5]))
    T, B = 8, 2
    out = (torch.zeros(T, B, 80), [torch.zeros(T, B, 80)], None, [], [], torch.zeros(B, 80, 4), torch.zeros(B, 80, 4),
           torch.full((B, 4), 0.25))
    with pytest.raises(FlowtronB200Error):
        FlowtronLoss(gm_loss=True, gate_loss=False)(out, None, torch.tensor([3, 3]), torch.tensor([8, 5]))


def test_more_than_32_components_raise():
    from flowtron_b200 import _lib
    from flowtron_b200.flowtron import _GmmNllFn
    z = torch.zeros(4, 2, 80)
    with pytest.raises(ValueError, match="32"):
        _GmmNllFn.apply(z, torch.tensor([4, 3]), torch.zeros(1, 80, 33), torch.zeros(1, 80, 33), torch.full((2, 33), 1 / 33))
    L = _lib.lib()
    ok, bad = _lib.FtGmmDesc(T=4, B=2, M=80, K=32, per_row=1), _lib.FtGmmDesc(T=4, B=2, M=80, K=33, per_row=1)
    assert L.ft_gmm_nll_scratch_bytes(ok) > 0
    assert L.ft_gmm_nll_scratch_bytes(bad) == 0
    assert b"32" in L.ft_last_error()


def test_mel_encoder_batch_limit_matches_the_header():
    from flowtron_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "flowtron_b200.h")).read()
    assert int(re.search(r"#define\s+FT_MEL_ENC_MAX_BATCH\s+(\d+)", hdr).group(1)) == _lib.MEL_ENC_MAX_BATCH == 64
    assert int(re.search(r"#define\s+FT_GMM_MAX_COMPONENTS\s+(\d+)", hdr).group(1)) == _lib.GMM_MAX_COMPONENTS == 32
    L = _lib.lib()
    assert L.ft_mel_encoder_saved_bytes(_lib.FtMelEncoderDesc(B=64, T=2000, eps=1e-5, dropout_p=0.5)) > 0
    assert L.ft_mel_encoder_saved_bytes(_lib.FtMelEncoderDesc(B=65, T=16, eps=1e-5, dropout_p=0.5)) == 0


def test_abi_symbols_are_declared_and_exported():
    from flowtron_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "flowtron_b200.h")).read()
    L = _lib.lib()
    for sym in ("ft_mel_encoder_saved_bytes", "ft_mel_encoder_fwd_scratch_bytes", "ft_mel_encoder_bwd_scratch_bytes",
                "ft_mel_encoder_fwd", "ft_mel_encoder_bwd", "ft_gmm_nll_scratch_bytes", "ft_gmm_nll_reduce", "ft_gmm_nll_grad"):
        assert re.search(r"\b" + sym + r"\(", hdr), sym
        assert hasattr(L, sym), sym


# The text encoder's kernels as the parent commit compiled them: registers / spills (-Xptxas -v) and a hash of each
# kernel's SASS instructions (cuobjdump -sass, addresses and encodings stripped).  encoder.cu now shares its device code
# with mel_encoder.cu through encoder_kernels.cuh; the kernels themselves must not change.
_ENC_KERNELS = {
    "_ZN2ft21enc_bilstm_bwd_kernelILi2EEEvNS_16EncLstmBwdParamsE": (255, ("40", "40"), "5a443a14b0107575"),
    "_ZN2ft21enc_bilstm_bwd_kernelILi1EEEvNS_16EncLstmBwdParamsE": (255, ("40", "40"), "108c2bec41f68b77"),
    "_ZN2ft21enc_bilstm_fwd_kernelILi2EEEvNS_16EncLstmFwdParamsE": (255, ("36", "36"), "9333b9f4100a06be"),
    "_ZN2ft21enc_bilstm_fwd_kernelILi1EEEvNS_16EncLstmFwdParamsE": (255, ("36", "36"), "56ca3fe645041ac4"),
    "_ZN2ft22enc_rng_advance_kernelEPy": (8, ("0", "0"), "a0e3aedf0534f89f"),
    "_ZN2ft19enc_norm_bwd_kernelEPKfPK6__halfS1_PKiiS1_S1_S1_fS1_PS2_PfS8_": (32, ("0", "0"), "c843761297c1f250"),
    "_ZN2ft19enc_norm_fwd_kernelEPKfPKiiS1_S1_ffPKyiP6__halfPfS8_": (32, ("0", "0"), "a311cddb04e8ad57"),
    "_ZN2ft27enc_unpack_conv_grad_kernelEPKfPf": (32, ("0", "0"), "d34ba1a8698ec2d8"),
    "_ZN2ft22enc_colsum_hilo_kernelEPK6__halfxiPKfPf": (32, ("0", "0"), "2019169276341926"),
    "_ZN2ft19enc_pack_wih_kernelEPKfP6__halfS3_": (18, ("0", "0"), "2440e59be516a81f"),
    "_ZN2ft20enc_pack_conv_kernelEPKfP6__halfS3_": (22, ("0", "0"), "d06270cf268c23b0"),
    "_ZN2ft19enc_out_grad_kernelEPKfPKiiiS1_Pf": (32, ("0", "0"), "9caac83c413733aa"),
    "_ZN2ft21enc_embed_grad_kernelEPKfPKxiPKiiiS1_Pf": (18, ("0", "0"), "e7311297c2d99df6"),
    "_ZN2ft16enc_embed_kernelEPKxPKfiPKiiiP6__half": (16, ("0", "0"), "4b94feaca877ddd4"),
    "_ZN2ft13enc_in_kernelEPKfPKiiiP6__half": (30, ("0", "0"), "c60cffb8967a4040"),
}


# mel_encoder.cu's own kernels, pinned the same way: both encoders run one host path, and no kernel of either file changed.
_MEL_ENC_KERNELS = {
    "_ZN2ft20mel_enc_dmean_kernelEPKfS1_iPf": (12, ("0", "0"), "6d1f30673583bfae"),
    "_ZN2ft19mel_enc_mean_kernelEPKfPKiiS3_iPfS4_": (31, ("0", "0"), "7f19eac91b247e2f"),
    "_ZN2ft27mel_unpack_conv_grad_kernelEPKfiiPf": (34, ("0", "0"), "269da6964b47df28"),
    "_ZN2ft20mel_pack_conv_kernelEPKfiiP6__halfS3_": (26, ("0", "0"), "85844aa1e43c1bb0"),
    "_ZN2ft17mel_enc_in_kernelEPKfPKiiP6__half": (32, ("0", "0"), "ce3d8fc79dfcf961"),
}


@pytest.mark.skipif(not HAVE_NVCC, reason="nvcc not available")
def test_text_encoder_kernels_are_unchanged(tmp_path):
    _assert_kernels_pinned("encoder.cu", _ENC_KERNELS, tmp_path)


@pytest.mark.skipif(not HAVE_NVCC, reason="nvcc not available")
def test_mel_encoder_kernels_are_unchanged(tmp_path):
    _assert_kernels_pinned("mel_encoder.cu", _MEL_ENC_KERNELS, tmp_path)


@pytest.mark.skipif(not HAVE_NVCC, reason="nvcc not available")
def test_new_kernels_do_not_spill(tmp_path):
    for src in ("mel_encoder.cu", "gmm.cu"):
        _, regs = _compile(src, tmp_path)
        assert regs, src
        for name, (_, spill) in regs.items():
            assert spill == ("0", "0"), name


# (saved, forward scratch, backward scratch) bytes of each encoder, as laid out before the two encoders shared one host path;
# the masked flag and the dropout probability do not change them.  Callers allocate these buffers, so the regions, their
# order and their sizes are part of what the host path must keep.
_ENC_BYTES = {  # (B, L)
    (1, 1): (145920, 29925632, 19486208), (1, 7): (305664, 29974784, 19590656),
    (1, 256): (6935040, 32014592, 23925248), (1, 1024): (27382272, 38306048, 37294592),
    (2, 1): (291328, 29966592, 19573248), (2, 7): (610816, 30064896, 19782144),
    (2, 256): (13869568, 34144512, 28451328), (2, 1024): (54764032, 46727424, 55190016),
    (33, 1): (4798976, 31236352, 22271488), (33, 7): (10070528, 32858368, 25718272),
    (33, 256): (228839936, 100172032, 168759808), (33, 1024): (903598592, 307790080, 609948160),
    (64, 1): (9306880, 32506112, 24969728), (64, 7): (19530496, 35651840, 31654400),
    (64, 256): (443810560, 166199552, 309068288), (64, 1024): (1752433408, 568852736, 1164706304),
}
_MEL_ENC_BYTES = {  # (B, T)
    (1, 1): (104960, 12232960, 14245376), (1, 100): (2005760, 13246720, 15968768),
    (1, 2000): (38485760, 32702720, 49043968), (17, 1): (1772032, 12921088, 15670784),
    (17, 100): (34085632, 30155008, 44968448), (17, 2000): (654245632, 360907008, 607246848),
    (64, 1): (6669312, 14942464, 19857920), (64, 100): (128320512, 79823104, 130155008),
    (64, 2000): (2463040512, 1325007104, 2246967808),
}


def test_encoder_buffer_sizes_are_pinned():
    from flowtron_b200 import _lib
    L = _lib.lib()
    for (B, T), want in _ENC_BYTES.items():
        for masked in (0, 1):
            for p in (0.0, 0.5):
                d = _lib.encoder_desc(B, T, masked, p)
                got = (L.ft_encoder_saved_bytes(d), L.ft_encoder_fwd_scratch_bytes(d), L.ft_encoder_bwd_scratch_bytes(d))
                assert got == want, (B, T, masked, p)
    for (B, T), want in _MEL_ENC_BYTES.items():
        for p in (0.0, 0.5):
            d = _lib.FtMelEncoderDesc(B=B, T=T, eps=1e-5, dropout_p=p)
            got = (L.ft_mel_encoder_saved_bytes(d), L.ft_mel_encoder_fwd_scratch_bytes(d), L.ft_mel_encoder_bwd_scratch_bytes(d))
            assert got == want, (B, T, p)
    bad_text = [_lib.encoder_desc(65, 8, 1, 0.0), _lib.encoder_desc(2, 8, 1, 0.0)]
    bad_text[1].C = 256
    for d in bad_text:
        assert (L.ft_encoder_saved_bytes(d), L.ft_encoder_fwd_scratch_bytes(d), L.ft_encoder_bwd_scratch_bytes(d)) == (0, 0, 0)
    for d in (_lib.FtMelEncoderDesc(B=65, T=8, eps=1e-5, dropout_p=0.0), _lib.FtMelEncoderDesc(B=2, T=0, eps=1e-5, dropout_p=0.0)):
        assert (L.ft_mel_encoder_saved_bytes(d), L.ft_mel_encoder_fwd_scratch_bytes(d), L.ft_mel_encoder_bwd_scratch_bytes(d)) == (0, 0, 0)


def test_mixture_parameters_reach_the_gradient_buckets_and_the_optimizer_order():
    from flowtron_b200 import distributed
    from flowtron_b200.flowtron import Flowtron
    m = Flowtron(**_cfg(K=8, fixed=False))
    bucketed = [id(p) for b in distributed._default_buckets(m) for p in b]
    assert sorted(bucketed) == sorted(id(p) for p in m.parameters())
    names = {id(p): n for n, p in m.named_parameters()}
    assert any(names[i].startswith("mel_encoder.") for i in bucketed)
    assert any(names[i].startswith("gaussian_mixture.mean_layer") for i in bucketed)
    assert "gaussian_mixture.mean" not in names.values()          # learned Gaussians: no buffers
    fixed = Flowtron(**_cfg(K=8, fixed=True))
    assert "gaussian_mixture.mean" not in dict(fixed.named_parameters())   # buffers never reach the optimizer
