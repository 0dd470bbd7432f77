"""GPU: the ping-pong GEMM schedule (each consumer warpgroup on its own 128 x 128 tile, per-warp TMA stores) gives
bit-identical outputs to the cooperative schedule, in every epilogue mode it serves (bias / bias2, alpha, tanh,
saturating fp16, bf16, dual outputs, beta by TMA reduce-add into a strided C32, MN-major A, tf32, M and N tails), against
SHA-256 digests that the cooperative build wrote (tests/make_golden_gemm_pingpong.py)."""
import json
import os
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import gemm_pingpong_cases as C  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("case", C.CASES, ids=[c[0] for c in C.CASES])
def test_pingpong_bit_identical_to_cooperative(case):
    from flowtron_b200 import _lib
    with open(os.path.join(HERE, "golden", "gemm_pingpong.json")) as f:
        golden = json.load(f)[case[0]]
    outs = C.run_case(_lib, case)
    assert _lib.device_status() == 0
    assert {k: C.digest(v) for k, v in outs.items()} == golden
