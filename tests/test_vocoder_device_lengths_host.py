"""CPU: the C ABI of the vocoder with per-row lengths in device memory -- the worst-case scratch of ft_waveglow_infer_dev
and the argument checks of ft_waveglow_infer_dev, ft_waveglow_infer and ft_stft_pack_rows, all made before any device
work."""
from ctypes import byref, c_int

from flowtron_b200 import _lib


def _desc(B, F_max, frames):
    fr = None if frames is None else (c_int * B)(*frames)
    return _lib.FtWaveGlowDesc(n_mel=80, n_flows=12, n_group=8, n_early_every=4, n_early_size=2, n_layers=8, n_channels=256,
                               kernel_size=3, B=B, F_max=F_max, frames=fr)


def test_device_frames_scratch_is_the_all_rows_at_f_max_size():
    L = _lib.lib()
    worst = L.ft_waveglow_scratch_bytes(byref(_desc(16, 860, None)))
    assert worst == L.ft_waveglow_scratch_bytes(byref(_desc(16, 860, [860] * 16)))
    assert worst > L.ft_waveglow_scratch_bytes(byref(_desc(16, 860, [150 + 40 * b for b in range(16)])))
    assert L.ft_waveglow_scratch_bytes(byref(_desc(129, 8, None))) == 0
    assert L.ft_waveglow_scratch_bytes(byref(_desc(2, 0, None))) == 0


def test_entry_points_refuse_the_other_frames_form():
    L = _lib.lib()
    w = _lib.FtWaveGlowWeights()
    p = 0x1000                                                 # never dereferenced: the calls fail their checks first
    assert L.ft_waveglow_infer_dev(byref(_desc(2, 8, [8, 8])), byref(w), p, p, 1.0, p, p, p, None) != 0
    assert "NULL" in L.ft_last_error().decode()
    assert L.ft_waveglow_infer_dev(byref(_desc(2, 8, None)), byref(w), p, p, 1.0, None, p, p, None) != 0
    assert "frames_dev" in L.ft_last_error().decode()
    assert L.ft_waveglow_infer(byref(_desc(2, 8, None)), byref(w), p, p, 1.0, p, p, None) != 0
    assert "ft_waveglow_infer_dev" in L.ft_last_error().decode()


def test_stft_pack_rows_argument_checks():
    L = _lib.lib()
    p = 0x1000
    assert L.ft_stft_pack_rows(None, 2, 4096, p, 1024, 256, p, p, p, None) != 0
    assert L.ft_stft_pack_rows(p, 2, 4096, p, 800, 256, p, p, p, None) != 0
    assert L.ft_stft_pack_rows(p, 0, 4096, p, 1024, 256, p, p, p, None) != 0
    assert L.ft_stft_pack_rows(p, 2, 0, p, 1024, 256, p, p, p, None) != 0
