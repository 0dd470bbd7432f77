"""Seeded GEMM launches large enough for launch_gemm to run them on the ping-pong schedule (at least 3 tiles of 128 x 128
per SM, K <= 4096), one per epilogue mode that schedule serves, shared by tests/make_golden_gemm_pingpong.py (which records
the SHA-256 of each output with a build that runs them on the cooperative schedule) and tests/test_gpu_gemm_pingpong.py
(which requires the ping-pong build to reproduce them bit for bit).  Case tuples and run_case / digest are those of
gemm_epilogue_cases."""
import torch

from gemm_epilogue_cases import digest, run_case  # noqa: F401

# name, M, N, K, operand dtype, a_mn, b_mn, pair mode, epilogue options; 8020 rows end inside a tile's second 64-row half
CASES = [
    ("pp f32 two biases, M tail", 8020, 1024, 320, torch.float16, False, False, 0, dict(nb=2, out32=True)),
    ("pp f32 N = 160", 32000, 160, 256, torch.float16, False, False, 0, dict(nb=1, out32=True)),
    ("pp f16 tanh", 8000, 1024, 256, torch.float16, False, False, 0, dict(nb=1, act=1, out16=True)),
    ("pp f16 saturating", 8000, 1024, 128, torch.float16, False, False, 0, dict(out16=True, alpha=3000.0)),
    ("pp bf16 out", 8000, 1024, 192, torch.bfloat16, False, False, 0, dict(nb=2, out16=True)),
    ("pp dual f32 + f16", 8000, 1024, 256, torch.float16, False, True, 0, dict(nb=1, act=1, out32=True, out16=True)),
    ("pp beta f32 strided", 8000, 1024, 640, torch.float16, False, True, 0, dict(beta=1, out32=True, ldc=1664)),
    ("pp A MN-major", 8000, 1024, 256, torch.bfloat16, True, False, 0, dict(out32=True)),
    ("pp tf32", 8000, 1024, 160, torch.float32, False, False, 0, dict(nb=1, out32=True)),
    ("pp long K", 8000, 1024, 4096, torch.float16, False, True, 0, dict(out32=True)),
]
