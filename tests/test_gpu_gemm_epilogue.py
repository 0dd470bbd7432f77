"""GPU: the staged TMA-store epilogue gives bit-identical outputs to the fragment-store epilogue it replaced, in every
epilogue mode (bias / bias2, alpha, tanh, beta with and without a 16-bit output, saturating fp16 and bf16, dual outputs,
CTA pairs, strided and unaligned outputs); split-K partial tiles, now added by TMA reduce-add, match fp64."""
import json
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import gemm_epilogue_cases as C  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("case", C.CASES, ids=[c[0] for c in C.CASES])
def test_epilogue_bit_identical_to_fragment_stores(case):
    from flowtron_b200 import _lib
    with open(os.path.join(HERE, "golden", "gemm_epilogue.json")) as f:
        golden = json.load(f)[case[0]]
    outs = C.run_case(_lib, case)
    assert _lib.device_status() == 0
    assert {k: C.digest(v) for k, v in outs.items()} == golden


# weight-gradient shapes with few output tiles, which launch_gemm splits over K: dense (1024 x 1024), attention query
# (640 x 1024), attention-LSTM input (4096 x 80), and a K that is not a multiple of the split
@pytest.mark.parametrize("M,N,K", [(1024, 1024, 32000), (640, 1024, 32000), (4096, 80, 32000), (640, 1024, 9000 + 40)])
def test_split_k_reduce_add_matches_fp64(M, N, K):
    from flowtron_b200 import _lib
    g = torch.Generator().manual_seed(M + N + K)
    A = (torch.randn(K, M, generator=g) * 0.3).half().cuda()
    B = (torch.randn(K, N, generator=g) * 0.3).half().cuda()
    out = torch.full((M, N), float("nan"), device="cuda")      # split-K zeroes C32 itself before adding partial tiles
    _lib.gemm(A, B, a_mn=True, b_mn=True, alpha=0.25, out32=out)
    torch.cuda.synchronize()
    assert _lib.device_status() == 0
    ref = 0.25 * (A.double().t() @ B.double())
    err = ((out.double() - ref).abs().max() / ref.abs().max()).item()
    assert err <= 1e-4, err
