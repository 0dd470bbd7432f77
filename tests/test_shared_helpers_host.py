"""CPU: the helpers the CUDA sources share (one workspace planner, one set of GEMM role launchers, one per-stream cache of
the flow step's streams and events, and the device helpers in ptx.cuh / mel_fft.cuh) change no kernel and no byte count a
caller allocates by, and every stream-ordering, memset and memcpy call's result is checked."""
import json
import os
import re
from ctypes import byref, c_int, c_size_t

import pytest

from conftest import GOLDEN, ROOT
from kernel_pins import HAVE_NVCC, _assert_kernels_pinned

CSRC = os.path.join(ROOT, "flowtron_b200", "csrc")

# Every kernel of each source whose device code includes a helper that now lives in one place (the m16n8k16 mma.sync, the
# frame-to-utterance search, the AR_Back_Step time flip), as compiled before the helpers were shared:
# {kernel: (registers, (spill stores, spill loads), SASS hash)}.
_KERNELS = {
    "attention.cu": {
        "_ZN2ft15attn_bwd_kernelILb0EEEvNS_13AttnBwdParamsE": (126, ("0", "0"), "3438583b48d7c9d7"),
        "_ZN2ft15attn_bwd_kernelILb1EEEvNS_13AttnBwdParamsE": (128, ("48", "48"), "aab5b82bc76f9bbf"),
        "_ZN2ft15attn_fwd_kernelILb0EEEvNS_13AttnFwdParamsE": (96, ("0", "0"), "99e46530ba22a3d2"),
        "_ZN2ft15attn_fwd_kernelILb1EEEvNS_13AttnFwdParamsE": (96, ("0", "0"), "f215711c6f54329a"),
    },
    "attention_module.cu": {
        "_ZN2ft_GLOBAL__N_15attn_bmm_kernelEiiiNS0_10BmmOperandES1_PfxxxPKfi": (80, ("0", "0"), "146e6f55fe6a7053"),
        "_ZN2ft_GLOBAL__N_17attn_split_kernelEPKfxiiP6__half": (24, ("0", "0"), "0a0626a21d22bf4a"),
        "_ZN2ft_GLOBAL__N_21attn_transpose_kernelEPKfxxiiPfxxS2_": (34, ("0", "0"), "705b5e6ce94e0f89"),
    },
    "elementwise.cu": {
        "_ZN2ft11cast_kernelI13__nv_bfloat16fEEvPKT_PT0_x": (32, ("0", "0"), "91a316142a9921c8"),
        "_ZN2ft11cast_kernelI6__half13__nv_bfloat16EEvPKT_PT0_x": (32, ("0", "0"), "f88773fdefd50b01"),
        "_ZN2ft11cast_kernelI6__halffEEvPKT_PT0_x": (32, ("0", "0"), "5185a521d8aaa2d5"),
        "_ZN2ft11cast_kernelIf13__nv_bfloat16EEvPKT_PT0_x": (32, ("0", "0"), "f97475f6f4b39e86"),
        "_ZN2ft11cast_kernelIf6__halfEEvPKT_PT0_x": (32, ("0", "0"), "aa44969337648d8e"),
        "_ZN2ft13absmax_kernelEPKfxS1_xS1_xPj": (32, ("0", "0"), "2038dbfb8b7546de"),
        "_ZN2ft13colsum_kernelI13__nv_bfloat16EEvPKT_xxiPfPKf": (26, ("0", "0"), "60d4f54d98082565"),
        "_ZN2ft13colsum_kernelI6__halfEEvPKT_xxiPfPKf": (26, ("0", "0"), "4296ea3e367aeb0b"),
        "_ZN2ft13colsum_kernelIfEEvPKT_xxiPfPKf": (26, ("0", "0"), "1980aab6bd6e4e9f"),
        "_ZN2ft15gate_bwd_kernelILb0EEEvPK6__halfxiPKfS5_xPfxS6_S6_S5_": (38, ("0", "0"), "222a6b033120a23e"),
        "_ZN2ft15gate_bwd_kernelILb1EEEvPK6__halfxiPKfS5_xPfxS6_S6_S5_": (40, ("0", "0"), "9ff4fa48b7bad5bc"),
        "_ZN2ft15gate_fwd_kernelEPK6__halfxiPKfS4_xPf": (30, ("0", "0"), "7a68f88b82b28c0a"),
        "_ZN2ft15nll_grad_kernelEPKfS1_S1_PKiiiifS1_S1_S1_PfS4_S4_": (40, ("0", "0"), "df57a41fe4537665"),
        "_ZN2ft15nll_rows_kernelEPKfNS_8LogSListEiS1_S1_PKiiiiPf": (40, ("0", "0"), "aaf489adb6bf2000"),
        "_ZN2ft15prep_mel_kernelEPKfPKiiiiiP6__halfPf": (30, ("0", "0"), "9304dfec6466780a"),
        "_ZN2ft17affine_bwd_kernelEPKfS1_S1_S1_PKiiiiiP6__halfPfS1_": (30, ("0", "0"), "defcd33b5161595d"),
        "_ZN2ft17affine_fwd_kernelEPKfS1_PKiiiiiPfS4_": (32, ("0", "0"), "5e71b41de9b54fd9"),
        "_ZN2ft17nll_reduce_kernelEPKfNS_8LogSListEiS1_S1_PKiiiiPf": (40, ("0", "0"), "3fc3a15728a44e0e"),
        "_ZN2ft19combine_dmel_kernelEPKfS1_PKiiiiiPfS1_": (34, ("0", "0"), "d587ead1211c3543"),
        "_ZN2ft19gate_fwd_f32_kernelEPKfxiS1_xiS1_S1_xPf": (38, ("0", "0"), "f5363b9aeddf26f5"),
        "_ZN2ft21scale_finalize_kernelEPKjfPf": (14, ("0", "0"), "f2c3c445abff7bb7"),
        "_ZN2ft25transpose_cast_f16_kernelEPKfP6__halfii": (19, ("0", "0"), "e215acf8c8056154"),
    },
    "infer.cu": {
        "_ZN2ft12infer_kernelILb0ELb0ELb0EEEvNS_11InferParamsE": (128, ("0", "0"), "cad4c7f15723e530"),
        "_ZN2ft12infer_kernelILb0ELb0ELb1EEEvNS_11InferParamsE": (127, ("0", "0"), "1950fc8f4e1c6b07"),
        "_ZN2ft12infer_kernelILb0ELb1ELb0EEEvNS_11InferParamsE": (128, ("0", "0"), "a1c488385110f8c7"),
        "_ZN2ft12infer_kernelILb0ELb1ELb1EEEvNS_11InferParamsE": (128, ("0", "0"), "74eb4aeb8176a57b"),
        "_ZN2ft12infer_kernelILb1ELb0ELb0EEEvNS_11InferParamsE": (127, ("0", "0"), "820c378a7f56caba"),
        "_ZN2ft12infer_kernelILb1ELb0ELb1EEEvNS_11InferParamsE": (127, ("0", "0"), "2dbca7155c3c7923"),
        "_ZN2ft12infer_kernelILb1ELb1ELb0EEEvNS_11InferParamsE": (125, ("0", "0"), "2eb11e43219b428d"),
        "_ZN2ft12infer_kernelILb1ELb1ELb1EEEvNS_11InferParamsE": (128, ("0", "0"), "e99aebf98a368917"),
        "_ZN2ft19infer_finish_kernelEPfS0_PKiiiiii": (24, ("0", "0"), "f30bfdfcd6f88e4c"),
        "_ZN2ft19pack_weights_kernelEP6__halfPfPKfiiS4_iS4_S4_iiii": (32, ("0", "0"), "779fe86e51c17890"),
    },
    "istft.cu": {
        "_ZN2ft12istft_kernelENS_11IstftParamsE": (128, ("0", "0"), "556e9786fd002058"),
        "_ZN2ft16stft_pack_kernelEPKfxPKxiiPfPxS5_": (40, ("0", "0"), "6cf480ae7a9a5425"),
    },
    "mel.cu": {
        "_ZN2ft12frame_kernelEPKfPKxS3_ixxS1_iiPf": (32, ("0", "0"), "b206e8ffd7953b66"),
        "_ZN2ft14mag_mel_kernelEPK6float2PKxixxiPKfPKiS8_ifPf": (30, ("0", "0"), "f4b3ddcd7ca5acba"),
    },
    "mel_fused.cu": {
        "_ZN2ft16mel_fused_kernelILi0ELb0EEEvNS_14MelFusedParamsE": (75, ("0", "0"), "781dfca27e455672"),
        "_ZN2ft16mel_fused_kernelILi0ELb1EEEvNS_14MelFusedParamsE": (79, ("0", "0"), "fab81a8ee1fd80dd"),
        "_ZN2ft16mel_fused_kernelILi1ELb0EEEvNS_14MelFusedParamsE": (78, ("0", "0"), "81c456f32c1b33fa"),
    },
    "waveglow.cu": {
        "_ZN2ft14wg_gemm_kernelENS_12WgGemmParamsE": (120, ("0", "0"), "eb5ce5b3b5d05038"),
        "_ZN2ft14wg_mela_kernelEPKNS_7WgBatchEPKiPK6__halfiPS5_": (24, ("0", "0"), "ec32ec94c74a641a"),
        "_ZN2ft14wg_plan_kernelENS_8WgFramesEPKiiiiPNS_7WgBatchE": (29, ("0", "0"), "05b42d5d1da08af1"),
        "_ZN2ft14wg_prep_kernelEPKNS_7WgBatchEPKfiP6__halfPiS7_": (24, ("0", "0"), "15f178781f2df7e6"),
        "_ZN2ft14wg_tail_kernelENS_12WgTailParamsE": (40, ("0", "0"), "3e3b8da76754463e"),
        "_ZN2ft20wg_scale_cast_kernelEPKfxS1_P6__half": (13, ("0", "0"), "6359b6cdc29beb47"),
        "_ZN2ft20wg_train_tail_kernelENS_12WtTailParamsE": (40, ("0", "0"), "bba784002cd6ab5e"),
        "_ZN2ft22wg_train_bwd_in_kernelENS_11WtBwdParamsE": (124, ("0", "0"), "3231314bde316242"),
        "_ZN2ft23wg_train_bwd_out_kernelENS_11WtBwdParamsE": (128, ("0", "0"), "17ad48da5dfc4f83"),
        "_ZN2ft24wg_train_bwd_skip_kernelENS_11WtBwdParamsE": (32, ("0", "0"), "db71d12b5897794b"),
    },
}


@pytest.mark.skipif(not HAVE_NVCC, reason="nvcc not available")
@pytest.mark.parametrize("src", sorted(_KERNELS))
def test_kernels_are_unchanged(src, tmp_path):
    _assert_kernels_pinned(src, _KERNELS[src], tmp_path)


_WG = dict(n_mel=80, n_flows=12, n_group=8, n_early_every=4, n_early_size=2, n_layers=8, n_channels=256, kernel_size=3)
_AR_REGIONS = ("mel_in16", "mel_flow", "d16", "gatesA", "cA", "text16", "Kp", "Vp", "Q", "p_save", "h0_16", "gates0", "c0",
               "h1_16", "gates1", "c1", "y1_16", "y2_16", "o32")


def workspace_bytes():
    """{query: bytes} for every caller-allocated workspace size the library reports, over shapes on both sides of each
    branch of the layouts (the attention overlap at T = 320, texts past the attention's shared-memory rows, every flag)."""
    from flowtron_b200 import _lib
    L = _lib.lib()
    out = {}
    for T in (200, 400):
        for B in (1, 7, 32):
            for Lt in (1, 256, 700, 1024):
                for rev in (0, 1):
                    for gate in (0, 1):
                        for prior in (0, 1):
                            d = _lib.FtArStepDesc(T=T, B=B, L=Lt, n_mel=80, n_hidden=1024, n_attn=640, n_text=512, reversed=rev,
                                                  has_gate=gate, has_prior=prior, temperature=1.0)
                            key = f"ar_step T={T} B={B} L={Lt} rev={rev} gate={gate} prior={prior}"
                            out[key] = [L.ft_ar_step_saved_bytes(d), L.ft_ar_step_scratch_bytes(d),
                                        L.ft_ar_step_bwd_carry_bytes(d)]
                            if B != 7 and Lt in (1, 700) and not gate:      # the gate flag adds no saved region
                                regions = []                                  # (offset, bytes) in _AR_REGIONS order, None: absent
                                for name in _AR_REGIONS:
                                    off, nb = c_size_t(), c_size_t()
                                    rc = L.ft_ar_step_saved_lookup(byref(d), name.encode(), byref(off), byref(nb))
                                    regions.append([off.value, nb.value] if rc == 0 else None)
                                out["ar_step lookup " + key[8:]] = regions
                            if B <= 16:
                                out["ar_step infer " + key[8:]] = L.ft_ar_step_infer_scratch_bytes(d)
    for T in (1, 200, 1000):
        for B in (1, 7, 40):
            for Lt in (1, 256, 1024):
                for given in (0, 1):
                    for prior in (0, 1):
                        d = _lib.FtAttentionDesc(T=T, B=B, L=Lt, Dq=1024, E=512, A=128, has_prior=prior, attn_given=given,
                                                 temperature=1.0)
                        out[f"attention T={T} B={B} L={Lt} given={given} prior={prior}"] = [
                            L.ft_attention_saved_bytes(d), L.ft_attention_scratch_bytes(d)]
    for frames, F_max in (([5], 5), ([10, 37, 64], 64), ([1] * 128, 1), (None, 100), (None, 1)):
        B = 4 if frames is None else len(frames)
        arr = None if frames is None else (c_int * B)(*frames)
        d = _lib.FtWaveGlowDesc(**_WG, B=B, F_max=F_max, frames=arr)
        out[f"waveglow frames={frames} F_max={F_max}"] = L.ft_waveglow_scratch_bytes(d)
    for B, F, N in ((1, 20, 5120), (4, 20, 4000), (4, 64, 16384), (128, 2, 8)):
        for nf, nl in ((12, 8), (3, 2)):
            d = _lib.FtWaveGlowTrainDesc(**dict(_WG, n_flows=nf, n_layers=nl), B=B, F=F, N=N)
            out[f"waveglow train B={B} F={F} N={N} flows={nf} layers={nl}"] = [
                L.ft_waveglow_train_saved_bytes(d), L.ft_waveglow_train_scratch_bytes(d)]
    for n_fft in (1024, 2048):
        for chunk in (1, 333, 4096):
            out[f"mel n_fft={n_fft} chunk={chunk}"] = L.ft_mel_scratch_bytes(n_fft, chunk)
    # rejected descriptors report 0
    out["rejected attention L"] = L.ft_attention_saved_bytes(_lib.FtAttentionDesc(T=8, B=2, L=1025, Dq=1024, E=512, A=128,
                                                                                  temperature=1.0))
    out["rejected attention Dq"] = L.ft_attention_scratch_bytes(_lib.FtAttentionDesc(T=8, B=2, L=8, Dq=1020, E=512, A=128,
                                                                                    temperature=1.0))
    out["rejected waveglow n_mel"] = L.ft_waveglow_scratch_bytes(_lib.FtWaveGlowDesc(**dict(_WG, n_mel=81), B=1, F_max=4))
    out["rejected waveglow frames"] = L.ft_waveglow_scratch_bytes(_lib.FtWaveGlowDesc(**_WG, B=1, F_max=4, frames=(c_int * 1)(5)))
    out["rejected waveglow train N"] = L.ft_waveglow_train_saved_bytes(_lib.FtWaveGlowTrainDesc(**_WG, B=1, F=2, N=1000))
    out["rejected waveglow train B"] = L.ft_waveglow_train_scratch_bytes(_lib.FtWaveGlowTrainDesc(**_WG, B=129, F=2, N=256))
    return out


def test_workspace_bytes_are_pinned():
    """Callers allocate these buffers, so each region's order, size and alignment is part of what the planner keeps."""
    want = json.load(open(os.path.join(GOLDEN, "workspace_bytes.json")))
    got = json.loads(json.dumps(workspace_bytes()))
    assert set(got) == set(want)
    assert [k for k in want if got[k] != want[k]] == []
    assert all(v == 0 for k, v in want.items() if k.startswith("rejected"))


_ORDERING_CALLS = ("cudaEventRecord", "cudaStreamWaitEvent", "cudaMemsetAsync", "cudaMemcpyAsync")


def _unchecked_calls(text):
    """(line, call) of every ordering / memset / memcpy call whose cudaError_t is dropped: checked means the call is the
    first argument of FT_CU or is compared with cudaSuccess; a line marked `// unchecked:` gives its reason instead."""
    text = re.sub(r'"(?:[^"\\\n]|\\.)*"', lambda q: '"' + " " * (len(q.group()) - 2) + '"', text)   # not in string literals
    found = []
    for m in re.finditer(r"\b(" + "|".join(_ORDERING_CALLS) + r")\s*\(", text):
        line_start = text.rfind("\n", 0, m.start()) + 1
        line_end = text.find("\n", m.end())
        if "// unchecked:" in text[line_start:line_end]:
            continue
        if re.search(r"FT_CU\(\s*$", text[:m.start()]):
            continue
        depth, i = 1, m.end()
        while depth:
            depth += {"(": 1, ")": -1}.get(text[i], 0)
            i += 1
        if re.match(r"\s*[!=]=\s*cudaSuccess", text[i:]):
            continue
        found.append((text.count("\n", 0, m.start()) + 1, m.group(1)))
    return found


def test_runtime_call_results_are_checked():
    bad = {}
    for f in sorted(os.listdir(CSRC)):
        if f.endswith(".cu"):
            calls = _unchecked_calls(open(os.path.join(CSRC, f)).read())
            if calls:
                bad[f] = calls
    assert bad == {}
    # the rule itself
    assert _unchecked_calls("cudaEventRecord(e, s);\nFT_CU(cudaEventRecord(e, s), who);") == [(1, "cudaEventRecord")]
    assert _unchecked_calls("if (cudaMemsetAsync(p, 0, f(n), st) != cudaSuccess) return -1;") == []
    assert _unchecked_calls("cudaEventRecord(e, s);   // unchecked: a timing event") == []
    assert _unchecked_calls('return ft_set_error("x: cudaMemsetAsync(p) failed");') == []
