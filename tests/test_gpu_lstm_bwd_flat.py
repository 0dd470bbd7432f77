"""GPU: the layer pipeline's flat split-K BPTT (lstm_bwd_flat_kernel, partial sums exchanged through L2) against the 4-CTA
cluster kernel (DSMEM exchange) on the same chunked inputs: dG and the dc*f carried between chunks must be bit-identical."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

H = 1024
CHUNK = 100           # the layer pipeline's chunk (csrc/ar_step.cu kLayerChunk)


def _bwd_chunk(L, T, B, t0, t1, dh, whhT, gates, cst, lens, dG, carry, flags, xchg):
    rc = L.ft_debug_lstm_bwd_chunk(T, B, t0, t1, dh.data_ptr(), H, whhT.data_ptr(), gates.data_ptr(), cst.data_ptr(),
                                   lens.data_ptr(), dG.data_ptr(), carry.data_ptr(), flags.data_ptr(),
                                   None if xchg is None else xchg.data_ptr(), torch.cuda.current_stream().cuda_stream)
    assert rc == 0, L.ft_last_error()


@pytest.mark.parametrize("B", [32, 17, 8])
@pytest.mark.parametrize("T", [100, 250, 1000])
def test_flat_bptt_bit_identical_to_cluster(T, B):
    from flowtron_b200 import _lib
    L = _lib.lib()
    L.ft_debug_lstm_bwd_chunk.argtypes = [ctypes.c_int] * 4 + [ctypes.c_void_p, ctypes.c_longlong] + [ctypes.c_void_p] * 9
    L.ft_debug_lstm_bwd_chunk.restype = ctypes.c_int
    dev = "cuda"
    g = torch.Generator().manual_seed(T * 100 + B)
    whh = torch.randn(4 * H, H, generator=g) * (2.0 / (3 * H) ** 0.5)
    xproj = torch.randn(T, B, 4 * H, generator=g) * 0.8
    lens = torch.randint(T // 2, T + 1, (B,), generator=g)
    lens[0] = T
    lens_d = lens.to(dev, torch.int32)
    # saved gates / cell states from the forward recurrence, as the training step has them
    hseq = torch.zeros(T, B, H, device=dev, dtype=torch.float16)
    gates = torch.zeros(T, B, 4 * H, device=dev, dtype=torch.float16)
    cst = torch.zeros(T, B, H, device=dev)
    _lib.lstm_fwd(xproj.to(dev), whh.to(dev).half(), lens_d, hseq, gates, cst)
    whhT = whh.t().contiguous().to(dev).half()
    dh = (torch.randn(T, B, H, generator=g) * 8.0).to(dev)          # loss-scaled incoming gradient

    def run(flat):
        dG = torch.full((T, B, 4 * H), float("nan"), device=dev, dtype=torch.float16)
        carry = torch.zeros(B, H, device=dev)
        flags = torch.empty(CHUNK * 128, device=dev, dtype=torch.int32)
        xchg = torch.full((2 * 16 * 4 * B * 64,), float("nan"), device=dev) if flat else None
        carries = []
        for c in range((T + CHUNK - 1) // CHUNK - 1, -1, -1):
            t0, t1 = c * CHUNK, min(T, (c + 1) * CHUNK)
            _bwd_chunk(L, T, B, t0, t1, dh, whhT, gates, cst, lens_d, dG, carry, flags, xchg)
            carries.append(carry.clone())
        torch.cuda.synchronize()
        return dG, carries

    dG_c, car_c = run(False)
    assert _lib.device_status() == 0
    dG_f, car_f = run(True)
    assert _lib.device_status() == 0
    assert torch.isfinite(dG_c.float()).all()
    assert dG_c.abs().max().item() > 0
    assert torch.equal(dG_f.view(torch.int16), dG_c.view(torch.int16))
    for a, b in zip(car_f, car_c):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
