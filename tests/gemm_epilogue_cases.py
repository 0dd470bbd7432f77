"""Seeded GEMM launches covering every epilogue mode reachable through ft_gemm, shared by tests/make_golden_gemm_epilogue.py
(which records the SHA-256 of each output with one build) and tests/test_gpu_gemm_epilogue.py (which requires another build
to reproduce them bit for bit).  No case splits K, so each output element is one fixed-order wgmma accumulation followed by
the same epilogue arithmetic.  Inputs come from a CPU generator, so every machine builds the same operands."""
import hashlib

import torch

# name, M, N, K, operand dtype, a_mn, b_mn, pair mode, epilogue options
CASES = [
    ("wide f32 two biases", 1100, 1024, 320, torch.float16, False, False, 0, dict(nb=2, out32=True)),
    ("wide f32 pairs", 128 * 40 + 70, 1280, 192, torch.float16, False, True, 2, dict(nb=1, out32=True)),
    ("narrow f32 N tail", 700, 160, 1024, torch.float16, False, False, 0, dict(nb=1, out32=True)),
    ("narrow f32 N = 80", 900, 80, 512, torch.float16, False, True, 0, dict(out32=True)),
    ("f16 tanh", 1000, 1024, 256, torch.float16, False, False, 0, dict(nb=1, act=1, out16=True)),
    ("f16 saturating", 600, 512, 128, torch.float16, False, False, 0, dict(out16=True, alpha=3000.0)),
    ("bf16 out", 520, 640, 192, torch.bfloat16, False, False, 0, dict(nb=2, out16=True)),
    ("dual f32 + f16", 650, 768, 256, torch.float16, False, True, 0, dict(nb=1, act=1, out32=True, out16=True)),
    ("beta f32 strided", 1000, 1024, 640, torch.float16, False, True, 0, dict(beta=1, out32=True, ldc=1664)),
    ("beta dual", 400, 512, 256, torch.float16, False, True, 0, dict(beta=1, out32=True, out16=True, alpha=0.5)),
    ("A MN-major", 1032, 512, 256, torch.bfloat16, True, False, 0, dict(out32=True)),
    ("tf32", 500, 384, 160, torch.float32, False, False, 0, dict(nb=1, out32=True)),
    ("odd ldc fallback", 300, 250, 128, torch.float16, False, False, 0, dict(nb=1, out32=True, ldc=251)),
]


def run_case(lib, case, seed=1234):
    """Run one case on cuda:0 and return its outputs (dict name -> tensor, on the device)."""
    name, M, N, K, dt, a_mn, b_mn, pair_mode, e = case
    g = torch.Generator().manual_seed(seed + sum(map(ord, name)))
    A = (torch.randn((K, M) if a_mn else (M, K), generator=g) * 0.3).to(dt).cuda()
    B = (torch.randn((K, N) if b_mn else (N, K), generator=g) * 0.3).to(dt).cuda()
    nb = e.get("nb", 0)
    bias = torch.randn(N, generator=g).cuda() if nb >= 1 else None
    bias2 = torch.randn(N, generator=g).cuda() if nb >= 2 else None
    out32 = out16 = None
    if e.get("out32"):
        ldc = e.get("ldc", N)
        out32 = torch.randn(M, ldc, generator=g).cuda()[:, :N]       # beta adds into these values
    if e.get("out16"):
        out16 = torch.zeros(M, N, dtype=torch.bfloat16 if dt == torch.bfloat16 else torch.float16, device="cuda")
    lib.set_gemm_pair_mode(pair_mode)
    try:
        lib.gemm(A, B, a_mn=a_mn, b_mn=b_mn, bias=bias, bias2=bias2, act=e.get("act", 0), beta=e.get("beta", 0),
                 alpha=e.get("alpha", 1.0), out32=out32, out16=out16)
        torch.cuda.synchronize()
    finally:
        lib.set_gemm_pair_mode(0)
    outs = {}
    if out32 is not None:
        outs["out32"] = out32.contiguous()
    if out16 is not None:
        outs["out16"] = out16
    return outs


def digest(t):
    return hashlib.sha256(t.detach().cpu().contiguous().view(torch.uint8).numpy().tobytes()).hexdigest()
