"""CPU: the fp64 inverse-STFT / Denoiser restatement (tests/istft_oracle.py) against the reference-generated fixtures
(tests/make_golden_istft.py), the inverse-FFT lane code of csrc/mel_fft.cuh against a direct inverse DFT, the kernel's
register budget, and the argument checks of STFT.inverse / griffin_lim / Denoiser that need no device."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT
from flowtron_b200 import synth
from oracle import stft_oracle as S

import istft_oracle as IO
import make_golden_istft as MG

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
HAVE_NVCC = shutil.which(NVCC) is not None or os.path.isfile(NVCC)


def istft_case_input(tag):
    """(magnitude, phase, hop, win) of an istft.npz case, with the spectrum of audio cases from the fp32 transform oracle."""
    kind, seed, B, n, hop, win = MG.ISTFT_CASES[tag]
    if kind == "audio":
        mag, phase = S.stft_transform(synth.synth_istft_audio(B, n, seed), 1024, hop, win)
    else:
        mag, phase = synth.synth_istft_spectrum(B, n, seed)
    return mag, phase, hop, win


def _rel(a, ref):
    a, ref = torch.as_tensor(np.asarray(a, dtype=np.float64)), torch.as_tensor(np.asarray(ref, dtype=np.float64))
    return (a - ref).abs().max().item() / ref.abs().max().item()


@pytest.mark.parametrize("tag", list(MG.ISTFT_CASES))
def test_inverse_oracle_matches_reference_fixture(tag):
    g = np.load(os.path.join(GOLDEN, "istft.npz"))
    mag, phase, hop, win = istft_case_input(tag)
    out = IO.stft_inverse(mag, phase, 1024, hop, win)
    ref = g[f"{tag}_out"]
    assert tuple(out.shape) == ref.shape == (mag.shape[0], 1, (mag.shape[2] - 1) * hop)
    assert _rel(out, ref) <= 1e-6


def test_denoise_oracle_matches_reference_fixture():
    g = np.load(os.path.join(GOLDEN, "denoiser.npz"))
    audio = torch.from_numpy(np.load(os.path.join(GOLDEN, MG.DENOISER["input"]))["audio"])
    assert g["bias_spec"].shape == (1, 513, 1)
    for s in MG.DENOISER["strengths"]:
        out = IO.denoise(audio, g["bias_spec"], s)
        ref = g[f"out_{s}"]
        assert tuple(out.shape) == ref.shape == (audio.shape[0], 1, (audio.shape[1] // 256) * 256)
        assert _rel(out, ref) <= 1e-6, s


def test_denoiser_fixture_state_layout():
    """The reference Denoiser's state_dict: bias_spec [1, 513, 1] and the STFT's two bases."""
    g = np.load(os.path.join(GOLDEN, "denoiser.npz"))
    shapes = {k: tuple(int(d) for d in s if d) for k, s in zip(g["state_keys"].tolist(), g["state_shapes"])}
    assert shapes == {"stft.forward_basis": (1026, 1, 1024), "stft.inverse_basis": (1026, 1, 1024), "bias_spec": (1, 513, 1)}
    from flowtron_b200.audio_processing import STFT
    ours = {f"stft.{k}": tuple(v.shape) for k, v in STFT(1024, 256, 1024).state_dict().items()}
    assert ours == {k: v for k, v in shapes.items() if k.startswith("stft.")}


@pytest.mark.skipif(not HAVE_NVCC, reason="nvcc not available")
def test_inverse_fft_lane_code_on_host(tmp_path):
    exe = str(tmp_path / "test_istft_fft")
    subprocess.run([NVCC, "-std=c++17", "-I", os.path.join(ROOT, "flowtron_b200", "csrc"),
                    os.path.join(ROOT, "tests", "host", "test_istft_fft.cu"), "-o", exe], check=True, capture_output=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    worst = float(re.search(r"worst relative error ([0-9.e+-]+)", r.stdout).group(1))
    assert worst <= 1e-6, worst


@pytest.mark.skipif(not HAVE_NVCC, reason="nvcc not available")
def test_inverse_kernel_does_not_spill(tmp_path):
    r = subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr",
                        "-Xptxas", "-v", "-c", os.path.join(ROOT, "flowtron_b200", "csrc", "istft.cu"), "-o",
                        str(tmp_path / "istft.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    log = r.stderr.split("istft_kernel")[-1]
    m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert m and m.groups() == ("0", "0"), log


def test_inverse_argument_checks():
    from flowtron_b200._lib import FlowtronB200Error
    from flowtron_b200.audio_processing import STFT, griffin_lim
    mag, phase = synth.synth_istft_spectrum(1, 6, 0)
    with pytest.raises(FlowtronB200Error):
        STFT(1024, 256, 1024).inverse(mag, phase)
    with pytest.raises(FlowtronB200Error):
        griffin_lim(mag, STFT(1024, 256, 1024), 2, angles=phase)
    with pytest.raises(NotImplementedError):
        STFT(800, 200, 800).inverse(mag[:, :401], phase[:, :401])
    for hop in (200, 64, 1024):
        with pytest.raises(NotImplementedError):
            STFT(1024, hop, 1024).inverse(mag, phase)
    with pytest.raises(ValueError):
        STFT(1024, 256, 1024).inverse(mag, phase[:, :, :5])
    with pytest.raises(ValueError):
        STFT(1024, 256, 1024).inverse(mag[:, :512], phase[:, :512])
    with pytest.raises(ValueError):
        STFT(1024, 256, 1024).inverse(mag[0], phase[0])
    from flowtron_b200 import _lib
    with pytest.raises(NotImplementedError):
        _lib.stft_inverse(mag, phase, None, None, 1, 6, None, 1024, 300, None)
