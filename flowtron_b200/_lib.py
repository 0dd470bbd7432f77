"""ctypes binding of libflowtron_b200.so (the C ABI in include/flowtron_b200.h).

There is deliberately NO fallback: if the shared library is missing or a call fails the product path
raises.  torch is used only for device memory, streams and torch.distributed.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, Structure, byref, c_char_p, c_double, c_float, c_int, c_longlong, c_size_t, c_void_p

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libflowtron_b200.so")

FT_F16, FT_BF16, FT_TF32 = 0, 1, 2
_FMT = {torch.float16: FT_F16, torch.bfloat16: FT_BF16, torch.float32: FT_TF32}

_lib = None


class FtArStepDesc(Structure):
    _fields_ = [("T", c_int), ("B", c_int), ("L", c_int), ("n_mel", c_int), ("n_hidden", c_int), ("n_attn", c_int),
                ("n_text", c_int), ("reversed", c_int), ("has_gate", c_int), ("has_prior", c_int),
                ("temperature", c_float), ("no_d_mel", c_int)]


AR_WEIGHT_FIELDS = ["attn_lstm_w_ih", "attn_lstm_w_hh", "attn_lstm_b_ih", "attn_lstm_b_hh",
                    "lstm_w_ih0", "lstm_w_hh0", "lstm_b_ih0", "lstm_b_hh0",
                    "lstm_w_ih1", "lstm_w_hh1", "lstm_b_ih1", "lstm_b_hh1",
                    "att_query", "att_key", "att_value", "att_v",
                    "dense_w0", "dense_b0", "dense_w1", "dense_b1", "conv_w", "conv_b", "gate_w", "gate_b"]


class FtArStepWeights(Structure):
    _fields_ = [(n, c_void_p) for n in AR_WEIGHT_FIELDS]


class FtEncoderDesc(Structure):
    _fields_ = [("B", c_int), ("L", c_int), ("C", c_int), ("n_convs", c_int), ("ksize", c_int), ("masked", c_int),
                ("dropout_p", c_float), ("eps", c_float)]


ENC_PARAM_FIELDS = [("conv_w", 3), ("conv_b", 3), ("norm_w", 3), ("norm_b", 3), ("w_ih", 2), ("w_hh", 2), ("b_ih", 2), ("b_hh", 2)]


class FtEncoderWeights(Structure):
    _fields_ = [(n, c_void_p * k) for n, k in ENC_PARAM_FIELDS]


class FtEncoderGrads(Structure):
    _fields_ = [("d_" + n, c_void_p * k) for n, k in ENC_PARAM_FIELDS]


class FtMelEncoderDesc(Structure):
    _fields_ = [("B", c_int), ("T", c_int), ("eps", c_float), ("dropout_p", c_float)]


MEL_ENC_PARAM_FIELDS = [("conv_w", 2), ("conv_b", 2), ("norm_w", 2), ("norm_b", 2), ("w_ih", 2), ("w_hh", 2), ("b_ih", 2), ("b_hh", 2)]
MEL_ENC_MAX_BATCH = 64          # FT_MEL_ENC_MAX_BATCH
GMM_MAX_COMPONENTS = 32         # FT_GMM_MAX_COMPONENTS


class FtMelEncoderWeights(Structure):
    _fields_ = [(n, c_void_p * k) for n, k in MEL_ENC_PARAM_FIELDS]


class FtMelEncoderGrads(Structure):
    _fields_ = [("d_" + n, c_void_p * k) for n, k in MEL_ENC_PARAM_FIELDS]


class FtGmmDesc(Structure):
    _fields_ = [("T", c_int), ("B", c_int), ("M", c_int), ("K", c_int), ("per_row", c_int)]


class FtWaveGlowDesc(Structure):
    _fields_ = [("n_mel", c_int), ("n_flows", c_int), ("n_group", c_int), ("n_early_every", c_int), ("n_early_size", c_int),
                ("n_layers", c_int), ("n_channels", c_int), ("kernel_size", c_int), ("B", c_int), ("F_max", c_int),
                ("frames", POINTER(c_int))]


WG_MAX_FLOWS, WG_MAX_LAYERS = 16, 8


class FtWaveGlowWeights(Structure):
    _fields_ = [("up_w", c_void_p), ("up_b", c_void_p)] + \
        [(n, (c_void_p * WG_MAX_LAYERS) * WG_MAX_FLOWS) for n in ("in_w", "in_b", "rs_w", "rs_b")] + \
        [(n, c_void_p * WG_MAX_FLOWS) for n in ("start_w", "start_b", "end_w", "end_b", "inv_w")]


class FtWaveGlowTrainDesc(Structure):
    _fields_ = [("n_mel", c_int), ("n_flows", c_int), ("n_group", c_int), ("n_early_every", c_int), ("n_early_size", c_int),
                ("n_layers", c_int), ("n_channels", c_int), ("kernel_size", c_int), ("B", c_int), ("F", c_int), ("N", c_int)]


class FtWaveGlowTrainWeights(Structure):
    _fields_ = [("up_w", c_void_p), ("up_b", c_void_p)] + \
        [(n, (c_void_p * WG_MAX_LAYERS) * WG_MAX_FLOWS) for n in ("in_w", "in_b", "rs_w", "rs_b", "in_wT", "rs_wT")] + \
        [(n, c_void_p * WG_MAX_FLOWS) for n in ("start_w", "start_b", "end_w", "end_b", "conv_w")]


class FtWaveGlowTrainGrads(Structure):
    _fields_ = [("up_w", c_void_p), ("up_b", c_void_p), ("in_w", ((c_void_p * 4) * WG_MAX_LAYERS) * WG_MAX_FLOWS)] + \
        [(n, (c_void_p * WG_MAX_LAYERS) * WG_MAX_FLOWS) for n in ("in_b", "rs_w", "rs_b")] + \
        [(n, c_void_p * WG_MAX_FLOWS) for n in ("start_w", "start_b", "end_w", "end_b", "conv_w")]


class FtAttentionDesc(Structure):
    _fields_ = [("T", c_int), ("B", c_int), ("L", c_int), ("Dq", c_int), ("E", c_int), ("A", c_int), ("has_prior", c_int),
                ("attn_given", c_int), ("temperature", c_float)]


class FtAttentionWeights(Structure):
    _fields_ = [("query", c_void_p), ("key", c_void_p), ("value", c_void_p), ("v", c_void_p)]


class FlowtronB200Error(RuntimeError):
    pass


# Longest text (tokens) the flow-step kernels take in training and inference: FT_MAX_TEXT_LEN in include/flowtron_b200.h
# (ft_max_text_len()).  Texts of up to 256 tokens run the short-text kernel variants, longer ones the long-text variants.
MAX_TEXT_LEN = 1024


def check_text_len(L: int, where: str) -> None:
    """ValueError for a padded text length the kernels do not take, before any allocation or launch."""
    if L > MAX_TEXT_LEN:
        raise ValueError(f"{where}: text length {L} > {MAX_TEXT_LEN} tokens (MAX_TEXT_LEN) is not supported")


def ragged_lengths(v, B: int, hi: int, name: str) -> torch.Tensor:
    """Per-row lengths of a padded batch: a CUDA tensor is trusted (only its size is checked, nothing is read on the
    host); host values must be B integers in [1, hi] and come back as a CPU tensor."""
    if torch.is_tensor(v) and v.is_cuda:
        if v.dim() != 1 or v.numel() != B:
            raise ValueError(f"{name} must hold {B} values, got shape {tuple(v.shape)}")
        return v
    t = torch.as_tensor(v)
    if t.dim() != 1 or t.numel() != B:
        raise ValueError(f"{name} must hold {B} values, got shape {tuple(t.shape)}")
    if t.is_floating_point() or t.dtype == torch.bool:
        raise ValueError(f"{name} must be integers")
    if bool((t < 1).any()) or bool((t > hi).any()):
        raise ValueError(f"{name} must lie in [1, {hi}], got {t.tolist()}")
    return t


def check_frames_cover_tokens(in_lens, out_lens) -> None:
    """ValueError unless every row has at least as many frames as tokens, which a monotonic alignment needs.  Checked
    only when both lengths are on the host (and of one shape); CUDA lengths are trusted and not read."""
    if any(torch.is_tensor(v) and v.is_cuda for v in (in_lens, out_lens)):
        return
    il, ol = torch.as_tensor(in_lens), torch.as_tensor(out_lens)
    if il.shape == ol.shape and bool((ol < il).any()):
        raise ValueError(f"every row needs at least as many frames as tokens: out_lens {ol.tolist()}, "
                         f"in_lens {il.tolist()}")


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise FlowtronB200Error(
                f"{LIB_PATH} not built: run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(the CUDA extension is mandatory; there is no CPU fallback)")
        _lib = ctypes.CDLL(LIB_PATH)
        _lib.ft_last_error.restype = c_char_p
        _lib.ft_launch_count.restype = c_longlong
        _declare(_lib)
    return _lib


def _declare(L):
    L.ft_gemm.argtypes = [c_int, c_int, c_int, c_void_p, c_longlong, c_int, c_int, c_void_p, c_longlong, c_int, c_int,
                          c_void_p, c_void_p, c_int, c_int, c_float, c_void_p, c_longlong, c_void_p, c_longlong,
                          c_int, c_void_p]
    L.ft_gemm.restype = c_int


    L.ft_lstm_fwd.argtypes = [c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_longlong, c_void_p, c_void_p,
                              c_void_p, c_longlong, c_void_p, c_void_p]
    L.ft_lstm_fwd.restype = c_int
    L.ft_lstm_bwd.argtypes = [c_int, c_int, c_void_p, c_longlong, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                              c_void_p, c_void_p]
    L.ft_lstm_bwd.restype = c_int


    L.ft_max_text_len.restype = c_int
    L.ft_ar_step_saved_bytes.argtypes = [POINTER(FtArStepDesc)]
    L.ft_ar_step_saved_bytes.restype = c_size_t
    L.ft_ar_step_scratch_bytes.argtypes = [POINTER(FtArStepDesc)]
    L.ft_ar_step_scratch_bytes.restype = c_size_t
    L.ft_ar_step_saved_lookup.argtypes = [POINTER(FtArStepDesc), c_char_p, POINTER(c_size_t), POINTER(c_size_t)]
    L.ft_ar_step_saved_lookup.restype = c_int
    L.ft_ar_step_fwd.argtypes = [POINTER(FtArStepDesc), POINTER(FtArStepWeights)] + [c_void_p] * 14
    L.ft_ar_step_fwd.restype = c_int
    L.ft_ar_step_bwd.argtypes = [POINTER(FtArStepDesc), POINTER(FtArStepWeights)] + [c_void_p] * 11 + \
        [POINTER(FtArStepWeights), c_void_p, c_void_p, c_void_p]
    L.ft_ar_step_bwd.restype = c_int
    L.ft_ar_step_bwd_carry_bytes.argtypes = [POINTER(FtArStepDesc)]
    L.ft_ar_step_bwd_carry_bytes.restype = c_size_t
    L.ft_ar_step_bwd_main.argtypes = [POINTER(FtArStepDesc), POINTER(FtArStepWeights)] + [c_void_p] * 10 + \
        [POINTER(FtArStepWeights), c_void_p, c_void_p, c_void_p, c_void_p]
    L.ft_ar_step_bwd_main.restype = c_int
    L.ft_ar_step_bwd_attn_lstm.argtypes = [POINTER(FtArStepDesc), POINTER(FtArStepWeights), c_void_p, c_void_p,
                                           POINTER(FtArStepWeights), c_void_p, c_void_p, c_void_p, c_void_p]
    L.ft_ar_step_bwd_attn_lstm.restype = c_int
    L.ft_ar_step_bwd_plan.argtypes = [POINTER(FtArStepDesc), POINTER(FtArStepWeights), c_int, c_int, POINTER(ctypes.c_uint)]
    L.ft_ar_step_bwd_plan.restype = c_int
    L.ft_ar_step_infer_scratch_bytes.argtypes = [POINTER(FtArStepDesc)]
    L.ft_ar_step_infer_scratch_bytes.restype = c_size_t
    L.ft_ar_step_infer.argtypes = [POINTER(FtArStepDesc), POINTER(FtArStepWeights)] + [c_void_p] * 6 + \
        [c_int, c_float, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]
    L.ft_ar_step_infer.restype = c_int
    L.ft_mel_scratch_bytes.argtypes = [c_int, c_longlong]
    L.ft_mel_scratch_bytes.restype = c_size_t
    L.ft_mel_spectrogram.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_longlong, c_void_p, c_void_p, c_void_p, c_void_p,
                                     c_int, c_int, c_int, c_float, c_void_p, c_void_p, c_longlong, c_void_p]
    L.ft_mel_spectrogram.restype = c_int
    L.ft_mel_spectrogram_fused.argtypes = [c_void_p, c_int, c_void_p, c_void_p, c_int, c_longlong, c_void_p, c_void_p, c_void_p,
                                           c_void_p, c_int, c_int, c_int, c_float, c_void_p, c_void_p]
    L.ft_mel_spectrogram_fused.restype = c_int
    L.ft_stft_transform.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_longlong, c_void_p, c_int, c_int, c_void_p, c_void_p,
                                    c_void_p]
    L.ft_stft_transform.restype = c_int
    L.ft_stft_inverse.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_longlong, c_void_p, c_int, c_int, c_void_p,
                                  c_float, c_void_p, c_void_p]
    L.ft_stft_inverse.restype = c_int
    L.ft_stft_pack_rows.argtypes = [c_void_p, c_int, c_longlong, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]
    L.ft_stft_pack_rows.restype = c_int
    L.ft_attn_prior.argtypes = [c_void_p, c_void_p, c_int, c_int, c_int, c_float, c_float, c_void_p, c_void_p]
    L.ft_attn_prior.restype = c_int
    L.ft_collate_mel.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]
    L.ft_collate_mel.restype = c_int
    L.ft_attn_ctc_scratch_bytes.argtypes = [c_int, c_int, c_int]
    L.ft_attn_ctc_scratch_bytes.restype = c_size_t
    L.ft_attn_ctc_loss.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_float, c_void_p, c_void_p, c_void_p,
                                   c_void_p]
    L.ft_attn_ctc_loss.restype = c_int
    L.ft_nll_reduce.argtypes = [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]
    L.ft_nll_reduce.restype = c_int
    L.ft_nll_rows.argtypes = [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]
    L.ft_nll_rows.restype = c_int
    L.ft_nll_grad.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_float, c_void_p, c_void_p,
                              c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]
    L.ft_nll_grad.restype = c_int
    L.ft_sumsq_partials.argtypes = [c_void_p, c_longlong, c_void_p, c_void_p]
    L.ft_sumsq_partials.restype = c_int
    L.ft_clip_coef.argtypes = [c_void_p, c_int, c_float, c_void_p, c_void_p]
    L.ft_clip_coef.restype = c_int
    L.ft_radam_step.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_longlong, c_double, c_double, c_double, c_double,
                                c_double, c_int, c_void_p, c_void_p]
    L.ft_radam_step.restype = c_int
    L.ft_radam_step_dev.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_longlong, c_double, c_double, c_double, c_double,
                                    c_double, c_void_p, c_void_p, c_void_p]
    L.ft_radam_step_dev.restype = c_int
    L.ft_step_increment.argtypes = [c_void_p, c_void_p]
    L.ft_step_increment.restype = c_int
    for fn in ("ft_encoder_saved_bytes", "ft_encoder_fwd_scratch_bytes", "ft_encoder_bwd_scratch_bytes"):
        getattr(L, fn).argtypes = [POINTER(FtEncoderDesc)]
        getattr(L, fn).restype = c_size_t
    L.ft_encoder_fwd.argtypes = [POINTER(FtEncoderDesc), POINTER(FtEncoderWeights), c_void_p, c_void_p, c_void_p, c_void_p,
                                 c_longlong, c_longlong, c_void_p, c_void_p, c_void_p]
    L.ft_encoder_fwd.restype = c_int
    L.ft_encoder_bwd.argtypes = [POINTER(FtEncoderDesc), POINTER(FtEncoderWeights), c_void_p, c_longlong, c_longlong, c_void_p,
                                 c_void_p, POINTER(FtEncoderGrads), c_void_p, c_void_p]
    L.ft_encoder_bwd.restype = c_int
    L.ft_encoder_fwd_tokens.argtypes = [POINTER(FtEncoderDesc), POINTER(FtEncoderWeights), c_void_p, c_void_p, c_int, c_void_p, c_void_p,
                                        c_void_p, c_longlong, c_longlong, c_void_p, c_void_p, c_void_p]
    L.ft_encoder_fwd_tokens.restype = c_int
    L.ft_encoder_bwd_tokens.argtypes = [POINTER(FtEncoderDesc), POINTER(FtEncoderWeights), c_void_p, c_longlong, c_longlong, c_void_p,
                                        c_void_p, c_int, c_void_p, POINTER(FtEncoderGrads), c_void_p, c_void_p]
    L.ft_encoder_bwd_tokens.restype = c_int
    L.ft_waveglow_scratch_bytes.argtypes = [POINTER(FtWaveGlowDesc)]
    L.ft_waveglow_scratch_bytes.restype = c_size_t
    L.ft_waveglow_infer.argtypes = [POINTER(FtWaveGlowDesc), POINTER(FtWaveGlowWeights), c_void_p, c_void_p, c_float, c_void_p,
                                    c_void_p, c_void_p]
    L.ft_waveglow_infer.restype = c_int
    L.ft_waveglow_infer_dev.argtypes = [POINTER(FtWaveGlowDesc), POINTER(FtWaveGlowWeights), c_void_p, c_void_p, c_float,
                                        c_void_p, c_void_p, c_void_p, c_void_p]
    L.ft_waveglow_infer_dev.restype = c_int
    for fn in ("ft_waveglow_train_saved_bytes", "ft_waveglow_train_scratch_bytes"):
        getattr(L, fn).argtypes = [POINTER(FtWaveGlowTrainDesc)]
        getattr(L, fn).restype = c_size_t
    L.ft_waveglow_train_fwd.argtypes = [POINTER(FtWaveGlowTrainDesc), POINTER(FtWaveGlowTrainWeights), c_void_p, c_void_p,
                                        c_void_p, POINTER(c_void_p), c_void_p, c_void_p, c_void_p]
    L.ft_waveglow_train_fwd.restype = c_int
    L.ft_waveglow_train_bwd.argtypes = [POINTER(FtWaveGlowTrainDesc), POINTER(FtWaveGlowTrainWeights), c_void_p,
                                        POINTER(c_void_p), c_void_p, POINTER(FtWaveGlowTrainGrads), c_void_p, c_void_p]
    L.ft_waveglow_train_bwd.restype = c_int
    L.ft_posterior_mean.argtypes = [c_void_p, c_int, c_int, c_int, c_void_p, c_int, c_int, c_float, c_void_p, c_void_p]
    L.ft_posterior_mean.restype = c_int
    L.ft_mas_align_scratch_bytes.argtypes = [c_int, c_int, c_int]
    L.ft_mas_align_scratch_bytes.restype = c_size_t
    L.ft_mas_align.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]
    L.ft_mas_align.restype = c_int
    L.ft_durations_to_attn.argtypes = [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]
    L.ft_durations_to_attn.restype = c_int
    for fn in ("ft_mel_encoder_saved_bytes", "ft_mel_encoder_fwd_scratch_bytes", "ft_mel_encoder_bwd_scratch_bytes"):
        getattr(L, fn).argtypes = [POINTER(FtMelEncoderDesc)]
        getattr(L, fn).restype = c_size_t
    L.ft_mel_encoder_fwd.argtypes = [POINTER(FtMelEncoderDesc), POINTER(FtMelEncoderWeights), c_void_p, c_void_p, c_void_p, c_int,
                                     c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]
    L.ft_mel_encoder_fwd.restype = c_int
    L.ft_mel_encoder_bwd.argtypes = [POINTER(FtMelEncoderDesc), POINTER(FtMelEncoderWeights), c_void_p, c_void_p,
                                     POINTER(FtMelEncoderGrads), c_void_p, c_void_p]
    L.ft_mel_encoder_bwd.restype = c_int
    L.ft_gmm_nll_scratch_bytes.argtypes = [POINTER(FtGmmDesc)]
    L.ft_gmm_nll_scratch_bytes.restype = c_size_t
    L.ft_gmm_nll_reduce.argtypes = [POINTER(FtGmmDesc)] + [c_void_p] * 8
    L.ft_gmm_nll_reduce.restype = c_int
    L.ft_gmm_nll_rows.argtypes = [POINTER(FtGmmDesc)] + [c_void_p] * 8
    L.ft_gmm_nll_rows.restype = c_int
    L.ft_gmm_nll_grad.argtypes = [POINTER(FtGmmDesc)] + [c_void_p] * 11
    L.ft_gmm_nll_grad.restype = c_int
    L.ft_gmm_sample.argtypes = [POINTER(FtGmmDesc)] + [c_void_p] * 5 + [c_float, c_void_p, c_void_p, c_void_p]
    L.ft_gmm_sample.restype = c_int
    L.ft_gmm_responsibilities.argtypes = [POINTER(FtGmmDesc)] + [c_void_p] * 8
    L.ft_gmm_responsibilities.restype = c_int
    for fn in ("ft_attention_saved_bytes", "ft_attention_scratch_bytes"):
        getattr(L, fn).argtypes = [POINTER(FtAttentionDesc)]
        getattr(L, fn).restype = c_size_t
    L.ft_attention_fwd.argtypes = [POINTER(FtAttentionDesc), POINTER(FtAttentionWeights)] + [c_void_p] * 11
    L.ft_attention_fwd.restype = c_int
    L.ft_attention_bwd.argtypes = [POINTER(FtAttentionDesc), POINTER(FtAttentionWeights)] + [c_void_p] * 12 + \
        [POINTER(FtAttentionWeights), c_void_p, c_void_p, c_void_p]
    L.ft_attention_bwd.restype = c_int


def check(rc: int, what: str = ""):
    if rc != 0:
        raise FlowtronB200Error(f"{what} failed (rc={rc}): {lib().ft_last_error().decode()}")


def ptr(t):
    return None if t is None else c_void_p(t.data_ptr())


def stream_ptr():
    return c_void_p(torch.cuda.current_stream().cuda_stream)


def device_status() -> int:
    return int(lib().ft_device_status())


def launch_count() -> int:
    return int(lib().ft_launch_count())


def reset_launch_count():
    lib().ft_reset_launch_count()


def timing(enable: bool):
    lib().ft_timing_reset()
    lib().ft_timing_enable(1 if enable else 0)


def timing_report():
    """[(name, m, n, k, count, total_ms)] aggregated per kernel and shape; synchronises the device."""
    buf = ctypes.create_string_buffer(1 << 16)
    lib().ft_timing_report.argtypes = [c_char_p, c_int]
    n = lib().ft_timing_report(buf, len(buf))
    out = []
    for line in buf.raw[:n].decode().splitlines():
        name, m, nn, k, cnt, ms = line.split()
        out.append((name, int(m), int(nn), int(k), int(cnt), float(ms)))
    return out


def _need_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise FlowtronB200Error("flowtron_b200 kernels need CUDA tensors (no CPU fallback exists)")


def set_gemm_pair_mode(mode: int):
    """0 = single-CTA tiles (default), 1 = CTA pairs for big contractions, 2 = CTA pairs whenever eligible."""
    lib().ft_set_gemm_pair_mode(int(mode))


def gemm(A, B, *, a_mn=False, b_mn=False, bias=None, bias2=None, act=0, beta=0, alpha=1.0,
         out32=None, out16=None):
    """C = act(alpha * A @ B^T + bias + bias2) (+ out32 if beta).  A:[M,K] (or [K,M] if a_mn), B:[N,K] (or [K,N])."""
    _need_cuda(A, B)
    if a_mn:
        K, M = A.shape
    else:
        M, K = A.shape
    if b_mn:
        Kb, N = B.shape
    else:
        N, Kb = B.shape
    assert K == Kb, (A.shape, B.shape)
    assert A.stride(-1) == 1 and B.stride(-1) == 1
    c16_fmt = 0
    if out16 is not None:
        c16_fmt = _FMT[out16.dtype]
    check(lib().ft_gemm(M, N, K, ptr(A), A.stride(0), _FMT[A.dtype], int(a_mn), ptr(B), B.stride(0), _FMT[B.dtype],
                        int(b_mn), ptr(bias), ptr(bias2), act, beta, float(alpha),
                        ptr(out32), 0 if out32 is None else out32.stride(0),
                        ptr(out16), 0 if out16 is None else out16.stride(0), c16_fmt, stream_ptr()), "ft_gemm")


def lstm_fwd(xproj, whh16, lens, hseq16, gates16=None, cstate=None, h32=None):
    """xproj [T,B,4096] f32, whh16 [4096,1024] f16, lens int32 [B]|None, hseq16 [T,B,>=1024 view] f16 (written)."""
    _need_cuda(xproj, whh16, hseq16)
    T, B = xproj.shape[0], xproj.shape[1]
    assert xproj.is_contiguous() and whh16.dtype == torch.float16 and hseq16.dtype == torch.float16
    assert hseq16.stride(1) == hseq16.stride(0) // B or T == 1
    flags = torch.empty(T * 16, dtype=torch.int32, device=xproj.device)
    check(lib().ft_lstm_fwd(T, B, ptr(xproj), ptr(whh16), ptr(lens), ptr(hseq16), hseq16.stride(1), ptr(gates16),
                            ptr(cstate), ptr(h32), 0 if h32 is None else h32.stride(1), ptr(flags), stream_ptr()),
          "ft_lstm_fwd")


def lstm_bwd(dh_ext, whhT16, gates16, cstate, lens, dG16):
    """dh_ext [T,B,ld view] f32, whhT16 [1024,4096] f16, dG16 [T,B,4096] f16 (written, saturating)."""
    _need_cuda(dh_ext, whhT16, dG16)
    T, B = dG16.shape[0], dG16.shape[1]
    assert whhT16.dtype == torch.float16 and dG16.dtype == torch.float16 and dG16.is_contiguous()
    flags = torch.empty(T * 64, dtype=torch.int32, device=dG16.device)
    check(lib().ft_lstm_bwd(T, B, ptr(dh_ext), dh_ext.stride(1), ptr(whhT16), ptr(gates16), ptr(cstate), ptr(lens),
                            ptr(dG16), ptr(flags), stream_ptr()), "ft_lstm_bwd")


# ----------------------------------------------------------------------------------------------- AR step
_scratch = {}


def scratch_buffer(nbytes: int, device) -> torch.Tensor:
    """Per-(device, stream) transient work area shared by every flow on that stream (grown on demand)."""
    key = (device.type, device.index, torch.cuda.current_stream(device).cuda_stream)
    buf = _scratch.get(key)
    if buf is None or buf.numel() < nbytes:
        buf = None
        _scratch[key] = None
        buf = torch.empty(int(nbytes), dtype=torch.uint8, device=device)
        _scratch[key] = buf
    return buf


def make_weights(tensors) -> FtArStepWeights:
    w = FtArStepWeights()
    for name, t in zip(AR_WEIGHT_FIELDS, tensors):
        if t is not None:
            assert t.dtype == torch.float32 and t.is_contiguous() and t.is_cuda, name
            setattr(w, name, t.data_ptr())
        else:
            setattr(w, name, None)
    return w


def ar_step_sizes(desc: FtArStepDesc):
    L = lib()
    return int(L.ft_ar_step_saved_bytes(byref(desc))), int(L.ft_ar_step_scratch_bytes(byref(desc)))


def ar_step_saved_view(desc: FtArStepDesc, saved: torch.Tensor, name: str, dtype) -> torch.Tensor:
    off, nb = c_size_t(), c_size_t()
    check(lib().ft_ar_step_saved_lookup(byref(desc), name.encode(), byref(off), byref(nb)), "ft_ar_step_saved_lookup")
    return saved[off.value: off.value + nb.value].view(dtype)


def ar_step_fwd(desc, weights, mel, text, in_lens, out_lens, prior, mel_out, log_s, gates, attn, logprob, saved, scratch,
                text_ready=None):
    """text_ready: a recorded torch.cuda.Event (or None) that the call waits for before it first reads `text`."""
    check(lib().ft_ar_step_fwd(byref(desc), byref(weights), ptr(mel), ptr(text), ptr(in_lens), ptr(out_lens), ptr(prior),
                               ptr(mel_out), ptr(log_s), ptr(gates), ptr(attn), ptr(logprob), ptr(saved), ptr(scratch),
                               None if text_ready is None else c_void_p(text_ready.cuda_event), stream_ptr()),
          "ft_ar_step_fwd")


def ar_step_bwd(desc, weights, mel, in_lens, out_lens, attn, d_mel_out, d_log_s, d_gates, d_attn, d_logprob, d_mel, d_text,
                grads, saved, scratch):
    check(lib().ft_ar_step_bwd(byref(desc), byref(weights), ptr(mel), ptr(in_lens), ptr(out_lens), ptr(attn),
                               ptr(d_mel_out), ptr(d_log_s), ptr(d_gates), ptr(d_attn), ptr(d_logprob), ptr(d_mel),
                               ptr(d_text), byref(grads), ptr(saved), ptr(scratch), stream_ptr()), "ft_ar_step_bwd")


def ar_step_bwd_carry_bytes(desc) -> int:
    return int(lib().ft_ar_step_bwd_carry_bytes(byref(desc)))


def ar_step_bwd_main(desc, weights, mel, in_lens, out_lens, attn, d_mel_out, d_log_s, d_gates, d_attn, d_logprob, d_text, grads,
                     saved, scratch, carry):
    check(lib().ft_ar_step_bwd_main(byref(desc), byref(weights), ptr(mel), ptr(in_lens), ptr(out_lens), ptr(attn), ptr(d_mel_out),
                                    ptr(d_log_s), ptr(d_gates), ptr(d_attn), ptr(d_logprob), ptr(d_text), byref(grads), ptr(saved),
                                    ptr(scratch), ptr(carry), stream_ptr()), "ft_ar_step_bwd_main")


# Stage bits of ft_ar_step_bwd_plan (include/flowtron_b200.h)
BWD_STAGES = {"COUPLING": 0, "CONV_DGRAD": 1, "DENSE1_DGRAD": 2, "DENSE0_DGRAD": 3, "LSTM1": 4, "LSTM0": 5, "GATE_DD": 6,
              "ATTN": 7, "QUERY_DGRAD": 8, "D_TEXT": 9, "ATTN_LSTM": 10, "D_MEL": 11, "G_CONV": 16, "G_DENSE1": 17,
              "G_DENSE0": 18, "G_LSTM1": 19, "G_LSTM0": 20, "G_QUERY": 21, "G_KEY": 22, "G_VALUE": 23, "G_V": 24,
              "G_ATTN_LSTM": 25, "G_GATE": 26}


def ar_step_bwd_plan(desc, want, want_d_text: bool, want_d_mel: bool) -> set:
    """Names of the backward stages ft_ar_step_bwd_main / ft_ar_step_bwd_attn_lstm run when the parameter gradients with
    a true entry in `want` (24 flags in AR_WEIGHT_FIELDS order) and d_text / d_mel as given are wanted.  Host only: the
    non-NULL gradient pointers are never dereferenced."""
    g = FtArStepWeights()
    for name, w in zip(AR_WEIGHT_FIELDS, want):
        setattr(g, name, 1 if w else None)
    m = ctypes.c_uint(0)
    check(lib().ft_ar_step_bwd_plan(byref(desc), byref(g), int(want_d_text), int(want_d_mel), byref(m)), "ft_ar_step_bwd_plan")
    return {k for k, b in BWD_STAGES.items() if m.value >> b & 1}


def ar_step_bwd_attn_lstm(desc, weights, out_lens, d_mel, grads, saved, scratch, carry):
    check(lib().ft_ar_step_bwd_attn_lstm(byref(desc), byref(weights), ptr(out_lens), ptr(d_mel), byref(grads), ptr(saved),
                                         ptr(scratch), ptr(carry), stream_ptr()), "ft_ar_step_bwd_attn_lstm")


def nll_reduce(z, log_s_list, gate, gate_target, out_lens, sums):
    """log_s_list: list of f32 CUDA tensors [T,B,M] (one per flow); their pointers travel as a host array."""
    T, B, M = z.shape
    arr = (c_void_p * len(log_s_list))(*[t.data_ptr() for t in log_s_list])
    check(lib().ft_nll_reduce(ptr(z), arr, len(log_s_list), ptr(gate), ptr(gate_target), ptr(out_lens), T, B, M,
                              ptr(sums), stream_ptr()), "ft_nll_reduce")


def nll_rows(z, log_s_list, gate, gate_target, out_lens, rows):
    """ft_nll_rows: rows [B, 4] = per utterance {sum z^2, sum_flows sum log_s, sum gate BCE, frames}."""
    _need_cuda(z, *log_s_list, gate, gate_target, out_lens, rows)
    T, B, M = z.shape
    arr = (c_void_p * max(1, len(log_s_list)))(*[t.data_ptr() for t in log_s_list])
    check(lib().ft_nll_rows(ptr(z), arr, len(log_s_list), ptr(gate), ptr(gate_target), ptr(out_lens), T, B, M,
                            ptr(rows), stream_ptr()), "ft_nll_rows")


def nll_grad(z, gate, gate_target, out_lens, sigma, sums, g_nll, g_gate, dz, dlog_s, dgate):
    T, B, M = z.shape
    check(lib().ft_nll_grad(ptr(z), ptr(gate), ptr(gate_target), ptr(out_lens), T, B, M, float(sigma), ptr(sums),
                            ptr(g_nll), ptr(g_gate), ptr(dz), ptr(dlog_s), ptr(dgate), stream_ptr()), "ft_nll_grad")


SUMSQ_PARTIALS = 1024


def sumsq_partials(x, partials):
    """x: flat f32 CUDA tensor; partials: f32 [1024] (written)."""
    _need_cuda(x, partials)
    assert x.dtype == torch.float32 and x.is_contiguous() and partials.numel() >= SUMSQ_PARTIALS
    check(lib().ft_sumsq_partials(ptr(x), x.numel(), ptr(partials), stream_ptr()), "ft_sumsq_partials")


def clip_coef(partials, n_partials, max_norm, norm_coef):
    _need_cuda(partials, norm_coef)
    check(lib().ft_clip_coef(ptr(partials), int(n_partials), float(max_norm), ptr(norm_coef), stream_ptr()), "ft_clip_coef")


def radam_step(p, g, m, v, beta1, beta2, eps, weight_decay_lr, step_size, use_denom, grad_coef=None):
    """In-place fused RAdam update of flat f32 CUDA tensors (radam.py:77-122)."""
    _need_cuda(p, g, m, v)
    n = p.numel()
    assert g.numel() == n and m.numel() == n and v.numel() == n
    for t in (p, g, m, v):
        assert t.dtype == torch.float32 and t.is_contiguous()
    check(lib().ft_radam_step(ptr(p), ptr(g), ptr(m), ptr(v), n, float(beta1), float(beta2), float(eps),
                              float(weight_decay_lr), float(step_size), 1 if use_denom else 0, ptr(grad_coef), stream_ptr()),
          "ft_radam_step")


def sumsq_partials_raw(x_ptr: int, n: int, partials_ptr: int):
    check(lib().ft_sumsq_partials(c_void_p(x_ptr), int(n), c_void_p(partials_ptr), stream_ptr()), "ft_sumsq_partials")


def radam_step_raw(p_ptr, g_ptr, m_ptr, v_ptr, n, beta1, beta2, eps, weight_decay_lr, step_size, use_denom, coef_ptr=0):
    """Raw-pointer form used by flowtron_b200.radam (runs of parameters inside flat buffers)."""
    check(lib().ft_radam_step(c_void_p(p_ptr), c_void_p(g_ptr), c_void_p(m_ptr), c_void_p(v_ptr), int(n), float(beta1),
                              float(beta2), float(eps), float(weight_decay_lr), float(step_size), 1 if use_denom else 0,
                              c_void_p(coef_ptr) if coef_ptr else None, stream_ptr()), "ft_radam_step")


def ar_step_infer(desc, weights, residual, text, in_lens, frame_lens, prior, attn_forced, gate_threshold, out, attn_out,
                  n_frames):
    """in_lens / frame_lens: int32 CUDA [B] or None (all L / all T); attn_forced: f32 CUDA [B, Ta, L] contiguous or None."""
    nbytes = int(lib().ft_ar_step_infer_scratch_bytes(byref(desc)))
    scratch = scratch_buffer(nbytes, residual.device)
    Ta = 0 if attn_forced is None else int(attn_forced.size(1))
    check(lib().ft_ar_step_infer(byref(desc), byref(weights), ptr(residual), ptr(text), ptr(in_lens), ptr(frame_lens), ptr(prior),
                                 ptr(attn_forced), Ta, float(gate_threshold), ptr(out), ptr(attn_out), ptr(n_frames),
                                 ptr(scratch), stream_ptr()), "ft_ar_step_infer")


def mel_spectrogram(wav, sample_offsets, frame_offsets, n_utt, total_frames, window, basis, band_lo, band_hi, n_fft, hop,
                    clip, mel_out, chunk_frames=131072):
    chunk = int(min(chunk_frames, max(1, total_frames)))
    scratch = scratch_buffer(int(lib().ft_mel_scratch_bytes(n_fft, chunk)), wav.device)
    check(lib().ft_mel_spectrogram(ptr(wav), ptr(sample_offsets), ptr(frame_offsets), n_utt, total_frames, ptr(window),
                                   ptr(basis), ptr(band_lo), ptr(band_hi), basis.shape[0], n_fft, hop, float(clip),
                                   ptr(mel_out), ptr(scratch), chunk, stream_ptr()), "ft_mel_spectrogram")


def mel_spectrogram_fused(wav, sample_offsets, frame_offsets, n_utt, total_frames, window, basis, band_lo, band_hi, n_fft, hop,
                          clip, mel_out):
    """wav: flat f32 (in [-1,1]) or int16 PCM CUDA tensor.  One kernel, no scratch (csrc/mel_fused.cu)."""
    _need_cuda(wav, mel_out)
    fmt = {torch.float32: 0, torch.int16: 1}[wav.dtype]
    check(lib().ft_mel_spectrogram_fused(ptr(wav), fmt, ptr(sample_offsets), ptr(frame_offsets), int(n_utt), int(total_frames),
                                         ptr(window), ptr(basis), ptr(band_lo), ptr(band_hi), basis.shape[0], int(n_fft),
                                         int(hop), float(clip), ptr(mel_out), stream_ptr()), "ft_mel_spectrogram_fused")


def stft_transform(wav, sample_offsets, frame_offsets, n_utt, total_frames, window, n_fft, hop, magnitude, phase):
    _need_cuda(wav, magnitude, phase)
    check(lib().ft_stft_transform(ptr(wav), ptr(sample_offsets), ptr(frame_offsets), int(n_utt), int(total_frames), ptr(window),
                                  int(n_fft), int(hop), ptr(magnitude), ptr(phase), stream_ptr()), "ft_stft_transform")


def stft_pack_rows(audio, lengths, n_fft, hop, packed, sample_offsets, frame_offsets):
    """audio f32 [B, N] CUDA (contiguous), lengths int64 CUDA [B] -> packed rows and their int64 [B + 1] sample / frame
    offsets, planned on the device (ft_stft_pack_rows: rows of at most n_fft / 2 samples come out empty)."""
    _need_cuda(audio, lengths, packed, sample_offsets, frame_offsets)
    assert audio.dtype == packed.dtype == torch.float32 and audio.is_contiguous() and lengths.dtype == torch.int64
    assert sample_offsets.dtype == frame_offsets.dtype == torch.int64 and lengths.is_contiguous()
    B, N = audio.shape
    check(lib().ft_stft_pack_rows(ptr(audio), int(B), int(N), ptr(lengths), int(n_fft), int(hop), ptr(packed),
                                  ptr(sample_offsets), ptr(frame_offsets), stream_ptr()), "ft_stft_pack_rows")


STFT_INVERSE_HOPS = (128, 256, 512)


def stft_inverse(magnitude, phase, frame_offsets, out_offsets, n_utt, total_frames, window, n_fft, hop, out, bias=None,
                 strength=0.0):
    """magnitude / phase: per-utterance [513, F_u] blocks (f32 CUDA, ft_stft_transform's layout); frame_offsets int64 [n_utt+1];
    out_offsets int64 [n_utt] (where utterance u's (F_u - 1) * hop samples go in ``out``); bias: optional f32 [513], applied as
    max(m - strength * bias, 0).  One kernel (csrc/istft.cu)."""
    if n_fft != 1024 or hop not in STFT_INVERSE_HOPS:
        raise NotImplementedError(f"the inverse STFT kernel is built for filter_length 1024 and hop 128, 256 or 512 "
                                  f"(got {n_fft}, {hop})")
    _need_cuda(magnitude, phase, frame_offsets, out_offsets, window, out, bias)
    assert magnitude.dtype == phase.dtype == torch.float32 and magnitude.is_contiguous() and phase.is_contiguous()
    assert frame_offsets.dtype == out_offsets.dtype == torch.int64 and out.dtype == torch.float32
    assert bias is None or (bias.dtype == torch.float32 and bias.is_contiguous() and bias.numel() == n_fft // 2 + 1)
    check(lib().ft_stft_inverse(ptr(magnitude), ptr(phase), ptr(frame_offsets), ptr(out_offsets), int(n_utt), int(total_frames),
                                ptr(window), int(n_fft), int(hop), ptr(bias), float(strength), ptr(out), stream_ptr()),
          "ft_stft_inverse")


def attn_prior(in_lens, out_lens, T, L, scaling, threshold, prior):
    """in_lens / out_lens: int32 CUDA [B]; prior: f32 CUDA [B,T,L] (written)."""
    _need_cuda(in_lens, out_lens, prior)
    assert in_lens.dtype == torch.int32 and out_lens.dtype == torch.int32 and prior.is_contiguous()
    check(lib().ft_attn_prior(ptr(in_lens), ptr(out_lens), in_lens.numel(), int(T), int(L), float(scaling), float(threshold),
                              ptr(prior), stream_ptr()), "ft_attn_prior")


def collate_mel(mel_packed, frame_offsets, order, n_mel, T, mel_padded, gate_padded, out_lens):
    _need_cuda(mel_packed, frame_offsets, order, mel_padded, gate_padded, out_lens)
    assert order.dtype == torch.int32 and out_lens.dtype == torch.int32 and frame_offsets.dtype == torch.int64
    check(lib().ft_collate_mel(ptr(mel_packed), ptr(frame_offsets), ptr(order), order.numel(), int(n_mel), int(T),
                               ptr(mel_padded), ptr(gate_padded), ptr(out_lens), stream_ptr()), "ft_collate_mel")


def attn_ctc_loss(logprob, in_lens, out_lens, time_reversed, blank_logprob, cost, dlogprob):
    """logprob [B,T,L] f32 CUDA (one flow), in_lens / out_lens int32 CUDA [B]; cost [B], dlogprob [B,T,L] written."""
    _need_cuda(logprob, in_lens, out_lens, cost, dlogprob)
    B, T, L = logprob.shape
    assert logprob.is_contiguous() and dlogprob.is_contiguous() and in_lens.dtype == torch.int32 and out_lens.dtype == torch.int32
    scratch = scratch_buffer(int(lib().ft_attn_ctc_scratch_bytes(B, T, L)), logprob.device)
    check(lib().ft_attn_ctc_loss(ptr(logprob), ptr(in_lens), ptr(out_lens), B, T, L, 1 if time_reversed else 0,
                                 float(blank_logprob), ptr(cost), ptr(dlogprob), ptr(scratch), stream_ptr()), "ft_attn_ctc_loss")


POSTERIOR_BATCH, POSTERIOR_TIME_AND_BATCH = 0, 1


def posterior_mean(z, out_lens, n_frames, mode, scale, out):
    """z f32 [T,B,M] contiguous CUDA, out_lens int32 CUDA [B]; out f32 [M, n_frames] (mode 0) or [M] (mode 1), written.
    One launch (csrc/style.cu)."""
    _need_cuda(z, out_lens, out)
    T, B, M = z.shape
    assert z.dtype == torch.float32 and z.is_contiguous() and out_lens.dtype == torch.int32 and out.is_contiguous()
    check(lib().ft_posterior_mean(ptr(z), int(T), int(B), int(M), ptr(out_lens), int(n_frames), int(mode), float(scale),
                                  ptr(out), stream_ptr()), "ft_posterior_mean")


def mas_align(logp, in_lens, out_lens, time_reversed, durations, token_of_frame):
    """logp [B,T,L] f32 CUDA, in_lens / out_lens int32 CUDA [B]; durations int32 [B,L], token_of_frame int32 [B,T] written.
    One launch (csrc/align.cu)."""
    _need_cuda(logp, in_lens, out_lens, durations, token_of_frame)
    B, T, L = logp.shape
    assert logp.dtype == torch.float32 and logp.is_contiguous() and in_lens.dtype == torch.int32 and out_lens.dtype == torch.int32
    assert durations.dtype == torch.int32 and token_of_frame.dtype == torch.int32
    scratch = scratch_buffer(int(lib().ft_mas_align_scratch_bytes(B, T, L)), logp.device)
    check(lib().ft_mas_align(ptr(logp), ptr(in_lens), ptr(out_lens), B, T, L, 1 if time_reversed else 0, ptr(durations),
                             ptr(token_of_frame), ptr(scratch), stream_ptr()), "ft_mas_align")


def durations_to_attn(durations, in_lens, time_reversed, out):
    """durations int32 CUDA [B,L], in_lens int32 CUDA [B]; out f32 [B,Ta,L] (written).  One launch (csrc/align.cu)."""
    _need_cuda(durations, in_lens, out)
    B, Ta, L = out.shape
    assert durations.dtype == torch.int32 and durations.is_contiguous() and in_lens.dtype == torch.int32
    assert out.dtype == torch.float32 and out.is_contiguous()
    check(lib().ft_durations_to_attn(ptr(durations), ptr(in_lens), B, L, Ta, 1 if time_reversed else 0, ptr(out),
                                     stream_ptr()), "ft_durations_to_attn")


def radam_step_dev_raw(p_ptr, g_ptr, m_ptr, v_ptr, n, beta1, beta2, eps, weight_decay, lr, step_dev, coef_ptr=0):
    """Capturable update: the step count is read from the int32 CUDA tensor ``step_dev`` by the kernel."""
    check(lib().ft_radam_step_dev(c_void_p(p_ptr), c_void_p(g_ptr), c_void_p(m_ptr), c_void_p(v_ptr), int(n), float(beta1),
                                  float(beta2), float(eps), float(weight_decay), float(lr), ptr(step_dev),
                                  c_void_p(coef_ptr) if coef_ptr else None, stream_ptr()), "ft_radam_step_dev")


def step_increment(step_dev):
    check(lib().ft_step_increment(ptr(step_dev), stream_ptr()), "ft_step_increment")


# ------------------------------------------------------------------------------------------------ text encoder
def encoder_desc(B, L, masked, dropout_p, eps=1e-5):
    return FtEncoderDesc(B=B, L=L, C=512, n_convs=3, ksize=5, masked=1 if masked else 0, dropout_p=float(dropout_p), eps=float(eps))


def _enc_struct(cls, prefix, tensors, fields):
    """tensors: dict name -> list of tensors, in `fields` order (ENC_PARAM_FIELDS or MEL_ENC_PARAM_FIELDS)."""
    st = cls()
    for n, k in fields:
        setattr(st, prefix + n, (c_void_p * k)(*[c_void_p(t.data_ptr()) for t in tensors[n]]))
    return st


def encoder_fwd(desc, params, x, in_lens_i32, rng_state, out, out_stride_b, out_stride_l, tokens=None, emb_weight=None):
    """ft_encoder_fwd (x [B,512,L] given) or ft_encoder_fwd_tokens (tokens int64 [B,L] + embedding weight).  params: dict name ->
    list of fp32 CUDA tensors (ENC_PARAM_FIELDS).  Returns the `saved` buffer."""
    _need_cuda(x if tokens is None else tokens, out)
    L = lib()
    saved = torch.empty(L.ft_encoder_saved_bytes(byref(desc)), dtype=torch.uint8, device=out.device)
    scratch = torch.empty(L.ft_encoder_fwd_scratch_bytes(byref(desc)), dtype=torch.uint8, device=out.device)
    w = _enc_struct(FtEncoderWeights, "", params, ENC_PARAM_FIELDS)
    if tokens is None:
        check(L.ft_encoder_fwd(byref(desc), byref(w), ptr(x), ptr(in_lens_i32), ptr(rng_state), ptr(out), out_stride_b, out_stride_l,
                               ptr(saved), ptr(scratch), stream_ptr()), "ft_encoder_fwd")
    else:
        check(L.ft_encoder_fwd_tokens(byref(desc), byref(w), ptr(tokens), ptr(emb_weight), emb_weight.size(0), ptr(in_lens_i32),
                                      ptr(rng_state), ptr(out), out_stride_b, out_stride_l, ptr(saved), ptr(scratch), stream_ptr()),
              "ft_encoder_fwd_tokens")
    return saved


def encoder_bwd(desc, params, d_out, saved, need_dx=True, tokens=None, emb_weight=None):
    """ft_encoder_bwd / ft_encoder_bwd_tokens.  Returns (d_x [B,512,L] -- or d_emb_weight in the token form -- or None, dict of
    gradient tensors like `params`)."""
    _need_cuda(d_out, saved)
    L = lib()
    dev = d_out.device
    grads = {n: [torch.empty_like(t) for t in params[n]] for n, _ in ENC_PARAM_FIELDS}
    scratch = torch.empty(L.ft_encoder_bwd_scratch_bytes(byref(desc)), dtype=torch.uint8, device=dev)
    w = _enc_struct(FtEncoderWeights, "", params, ENC_PARAM_FIELDS)
    g = _enc_struct(FtEncoderGrads, "d_", grads, ENC_PARAM_FIELDS)
    if tokens is None:
        d_x = torch.empty(desc.B, 512, desc.L, dtype=torch.float32, device=dev) if need_dx else None
        check(L.ft_encoder_bwd(byref(desc), byref(w), ptr(d_out), d_out.stride(0), d_out.stride(1), ptr(saved), ptr(d_x), byref(g),
                               ptr(scratch), stream_ptr()), "ft_encoder_bwd")
        return d_x, grads
    d_emb = torch.empty_like(emb_weight)
    check(L.ft_encoder_bwd_tokens(byref(desc), byref(w), ptr(d_out), d_out.stride(0), d_out.stride(1), ptr(saved), ptr(tokens),
                                  emb_weight.size(0), ptr(d_emb), byref(g), ptr(scratch), stream_ptr()), "ft_encoder_bwd_tokens")
    return d_emb, grads


# ------------------------------------------------------------------------------------------------ mel encoder (GMM prior)
def mel_encoder_fwd(params, mel, out_lens_i32, all_lens_i32, rng_state, dropout_p, eps, emb):
    """ft_mel_encoder_fwd on mel [B, 80, T] (B <= 64) -> emb [B, 512] (written).  all_lens_i32: the whole batch's lengths (their
    maximum divides the time sum).  Returns (desc, saved) for mel_encoder_bwd."""
    _need_cuda(mel, out_lens_i32, all_lens_i32, emb)
    L = lib()
    desc = FtMelEncoderDesc(B=mel.size(0), T=mel.size(2), eps=float(eps), dropout_p=float(dropout_p))
    saved = torch.empty(L.ft_mel_encoder_saved_bytes(byref(desc)), dtype=torch.uint8, device=mel.device)
    scratch = torch.empty(L.ft_mel_encoder_fwd_scratch_bytes(byref(desc)), dtype=torch.uint8, device=mel.device)
    w = _enc_struct(FtMelEncoderWeights, "", params, MEL_ENC_PARAM_FIELDS)
    check(L.ft_mel_encoder_fwd(byref(desc), byref(w), ptr(mel), ptr(out_lens_i32), ptr(all_lens_i32), all_lens_i32.numel(),
                               ptr(rng_state), ptr(emb), ptr(saved), ptr(scratch), stream_ptr()), "ft_mel_encoder_fwd")
    return desc, saved


def mel_encoder_bwd(desc, params, d_emb, saved):
    """ft_mel_encoder_bwd: dict of weight gradients like `params`."""
    _need_cuda(d_emb, saved)
    L = lib()
    grads = {n: [torch.empty_like(t) for t in params[n]] for n, _ in MEL_ENC_PARAM_FIELDS}
    scratch = torch.empty(L.ft_mel_encoder_bwd_scratch_bytes(byref(desc)), dtype=torch.uint8, device=d_emb.device)
    w = _enc_struct(FtMelEncoderWeights, "", params, MEL_ENC_PARAM_FIELDS)
    g = _enc_struct(FtMelEncoderGrads, "d_", grads, MEL_ENC_PARAM_FIELDS)
    check(L.ft_mel_encoder_bwd(byref(desc), byref(w), ptr(d_emb), ptr(saved), byref(g), ptr(scratch), stream_ptr()),
          "ft_mel_encoder_bwd")
    return grads


# ------------------------------------------------------------------------------------------------ mixture NLL
def gmm_nll_reduce(z, out_lens_i32, mean, log_var, prob, per_row, sums):
    """ft_gmm_nll_reduce: sums[0] = NLL, sums[1] = valid frames.  z [T, B, M], mean / log_var [B or 1, M, K], prob [B, K]."""
    _need_cuda(z, out_lens_i32, mean, log_var, prob, sums)
    T, B, M = z.shape
    desc = FtGmmDesc(T=T, B=B, M=M, K=prob.size(1), per_row=int(per_row))
    scratch = torch.empty(lib().ft_gmm_nll_scratch_bytes(byref(desc)), dtype=torch.uint8, device=z.device)
    check(lib().ft_gmm_nll_reduce(byref(desc), ptr(z), ptr(out_lens_i32), ptr(mean), ptr(log_var), ptr(prob), ptr(sums),
                                  ptr(scratch), stream_ptr()), "ft_gmm_nll_reduce")


def gmm_nll_rows(z, out_lens_i32, mean, log_var, prob, per_row, rows):
    """ft_gmm_nll_rows: rows [B] = each utterance's mixture NLL (no division by its element count)."""
    _need_cuda(z, out_lens_i32, mean, log_var, prob, rows)
    T, B, M = z.shape
    desc = FtGmmDesc(T=T, B=B, M=M, K=prob.size(1), per_row=int(per_row))
    scratch = torch.empty(lib().ft_gmm_nll_scratch_bytes(byref(desc)), dtype=torch.uint8, device=z.device)
    check(lib().ft_gmm_nll_rows(byref(desc), ptr(z), ptr(out_lens_i32), ptr(mean), ptr(log_var), ptr(prob), ptr(rows),
                                ptr(scratch), stream_ptr()), "ft_gmm_nll_rows")


def gmm_nll_grad(z, out_lens_i32, mean, log_var, prob, per_row, g_nll, dz, dmean, dlog_var, dprob):
    """ft_gmm_nll_grad: gradients of g_nll[0] * NLL (dmean / dlog_var None for shared Gaussians)."""
    _need_cuda(z, out_lens_i32, mean, log_var, prob, g_nll, dz, dprob)
    T, B, M = z.shape
    desc = FtGmmDesc(T=T, B=B, M=M, K=prob.size(1), per_row=int(per_row))
    scratch = torch.empty(lib().ft_gmm_nll_scratch_bytes(byref(desc)), dtype=torch.uint8, device=z.device)
    check(lib().ft_gmm_nll_grad(byref(desc), ptr(z), ptr(out_lens_i32), ptr(mean), ptr(log_var), ptr(prob), ptr(g_nll), ptr(dz),
                                ptr(dmean), ptr(dlog_var), ptr(dprob), ptr(scratch), stream_ptr()), "ft_gmm_nll_grad")


def gmm_sample(mean, log_var, prob, per_row, n_frames_i32, component_i32, sigma, rng_state, z):
    """ft_gmm_sample: z [B, M, T] (written) from mean / log_var [B or 1, M, K], prob [B, K]; component_i32 [B] or None;
    rng_state int64 [2] = {seed, counter}, its counter advanced on the device.  Two launches, no allocation."""
    _need_cuda(mean, log_var, prob, n_frames_i32, component_i32, rng_state, z)
    B, M, T = z.shape
    desc = FtGmmDesc(T=T, B=B, M=M, K=prob.size(1), per_row=int(per_row))
    check(lib().ft_gmm_sample(byref(desc), ptr(mean), ptr(log_var), ptr(prob), ptr(n_frames_i32), ptr(component_i32),
                              float(sigma), ptr(rng_state), ptr(z), stream_ptr()), "ft_gmm_sample")


def gmm_responsibilities(z, out_lens_i32, mean, log_var, prob, per_row, resp):
    """ft_gmm_responsibilities: resp [B, K] (written) for z [T, B, M]."""
    _need_cuda(z, out_lens_i32, mean, log_var, prob, resp)
    T, B, M = z.shape
    desc = FtGmmDesc(T=T, B=B, M=M, K=prob.size(1), per_row=int(per_row))
    scratch = torch.empty(lib().ft_gmm_nll_scratch_bytes(byref(desc)), dtype=torch.uint8, device=z.device)
    check(lib().ft_gmm_responsibilities(byref(desc), ptr(z), ptr(out_lens_i32), ptr(mean), ptr(log_var), ptr(prob),
                                        ptr(resp), ptr(scratch), stream_ptr()), "ft_gmm_responsibilities")


# ------------------------------------------------------------------------------------------------ WaveGlow
def waveglow_infer(desc, weights, mel, noise, sigma, audio, frames_dev=None):
    """mel f32 [B,80,F_max], noise f32 [B,8,32 F_max], audio f32 [B,256 F_max] (written).  The frame counts are either
    desc.frames (host) or frames_dev (int32 CUDA [B], with desc.frames NULL: ft_waveglow_infer_dev)."""
    _need_cuda(mel, noise, audio, frames_dev)
    nbytes = int(lib().ft_waveglow_scratch_bytes(byref(desc)))
    if nbytes == 0:
        raise FlowtronB200Error(f"ft_waveglow_scratch_bytes rejected the configuration: {lib().ft_last_error().decode()}")
    scratch = scratch_buffer(nbytes, mel.device)
    if frames_dev is None:
        check(lib().ft_waveglow_infer(byref(desc), byref(weights), ptr(mel), ptr(noise), float(sigma), ptr(audio), ptr(scratch),
                                      stream_ptr()), "ft_waveglow_infer")
    else:
        assert frames_dev.dtype == torch.int32 and frames_dev.is_contiguous() and frames_dev.numel() == desc.B
        check(lib().ft_waveglow_infer_dev(byref(desc), byref(weights), ptr(mel), ptr(noise), float(sigma), ptr(frames_dev),
                                          ptr(audio), ptr(scratch), stream_ptr()), "ft_waveglow_infer_dev")


def _wg_train_bytes(desc):
    saved = int(lib().ft_waveglow_train_saved_bytes(byref(desc)))
    scratch = int(lib().ft_waveglow_train_scratch_bytes(byref(desc)))
    if saved == 0 or scratch == 0:
        raise FlowtronB200Error(f"ft_waveglow_train rejected the configuration: {lib().ft_last_error().decode()}")
    return saved, scratch


def waveglow_train_saved_bytes(desc) -> int:
    return _wg_train_bytes(desc)[0]


def waveglow_train_fwd(desc, weights, mel, audio, z, log_s_list, saved):
    """mel f32 [B,80,F], audio f32 [B,N] -> z f32 [B,8,N/8], log_s_list[k] f32 [B,n_half_k,N/8] (written); saved: uint8 of
    waveglow_train_saved_bytes(desc), kept for waveglow_train_bwd."""
    _need_cuda(mel, audio, z, saved, *log_s_list)
    _, nscratch = _wg_train_bytes(desc)
    scratch = scratch_buffer(nscratch, mel.device)
    ls = (c_void_p * len(log_s_list))(*[t.data_ptr() for t in log_s_list])
    check(lib().ft_waveglow_train_fwd(byref(desc), byref(weights), ptr(mel), ptr(audio), ptr(z), ls, ptr(saved), ptr(scratch),
                                      stream_ptr()), "ft_waveglow_train_fwd")


def waveglow_train_bwd(desc, weights, d_z, d_log_s_list, saved, grads):
    """d_z f32 [B,8,N/8] or None, d_log_s_list[k] f32 [B,n_half_k,N/8] or None -> grads (FtWaveGlowTrainGrads, written)."""
    _, nscratch = _wg_train_bytes(desc)
    scratch = scratch_buffer(nscratch, saved.device)
    dls = (c_void_p * len(d_log_s_list))(*[None if t is None else t.data_ptr() for t in d_log_s_list])
    check(lib().ft_waveglow_train_bwd(byref(desc), byref(weights), ptr(d_z), dls, ptr(saved), byref(grads), ptr(scratch),
                                      stream_ptr()), "ft_waveglow_train_bwd")


# ------------------------------------------------------------------------------------------------ Attention module
def attention_weights(query, key, value, v) -> FtAttentionWeights:
    """fp32 contiguous CUDA tensors (or None) -> the pointer struct of ft_attention_fwd / ft_attention_bwd (also used for the
    weight gradients)."""
    return FtAttentionWeights(*[None if t is None else t.data_ptr() for t in (query, key, value, v)])


def attention_sizes(desc: FtAttentionDesc):
    """(saved, scratch) bytes of ft_attention_fwd / ft_attention_bwd."""
    saved, scratch = int(lib().ft_attention_saved_bytes(byref(desc))), int(lib().ft_attention_scratch_bytes(byref(desc)))
    if saved == 0 or scratch == 0:
        raise FlowtronB200Error(f"ft_attention rejected the configuration: {lib().ft_last_error().decode()}")
    return saved, scratch


def attention_fwd(desc, weights, queries, keys, values, in_lens, prior, output, attn, logprob, saved, scratch):
    _need_cuda(values, output, attn, saved, scratch)
    check(lib().ft_attention_fwd(byref(desc), byref(weights), ptr(queries), ptr(keys), ptr(values), ptr(in_lens), ptr(prior),
                                 ptr(output), ptr(attn), ptr(logprob), ptr(saved), ptr(scratch), stream_ptr()), "ft_attention_fwd")


def attention_bwd(desc, weights, queries, keys, values, in_lens, attn, d_output, d_attn, d_logprob, d_queries, d_keys, d_values,
                  d_attn_given, grads, saved, scratch):
    check(lib().ft_attention_bwd(byref(desc), byref(weights), ptr(queries), ptr(keys), ptr(values), ptr(in_lens), ptr(attn),
                                 ptr(d_output), ptr(d_attn), ptr(d_logprob), ptr(d_queries), ptr(d_keys), ptr(d_values),
                                 ptr(d_attn_given), byref(grads), ptr(saved), ptr(scratch), stream_ptr()), "ft_attention_bwd")
