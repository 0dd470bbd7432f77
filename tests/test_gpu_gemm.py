"""GPU: wgmma/TMA GEMM primitive vs torch fp64 matmul (through the C ABI)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _ref(A, B, a_mn, b_mn, bias, bias2, act, alpha):
    a = A.double().t() if a_mn else A.double()
    b = B.double().t() if b_mn else B.double()
    c = alpha * (a @ b.t())
    if bias is not None:
        c = c + bias.double()
    if bias2 is not None:
        c = c + bias2.double()
    if act == 1:
        c = torch.tanh(c)
    return c


CASES = [
    # M, N, K, dtype, a_mn, b_mn
    (128, 128, 64, torch.float16, False, False),
    (256, 256, 256, torch.float16, False, False),
    (200, 160, 80, torch.float16, False, False),      # ragged M/N/K tails (K=80 like the mel projection)
    (512, 4096, 1664, torch.float16, False, False),
    (384, 640, 1024, torch.bfloat16, False, False),
    (256, 128, 128, torch.float32, False, False),     # tf32
    (300, 160, 1024, torch.float32, False, False),
    (256, 256, 256, torch.bfloat16, True, False),     # A given as [K, M]
    (256, 256, 256, torch.bfloat16, False, True),     # B given as [K, N]
    (1024, 1664, 2000, torch.bfloat16, True, True),   # wgrad shape: dW = dY^T X
    (500, 1664, 4096, torch.bfloat16, False, True),   # dgrad shape: dX = dY W
    # persistent kernel: more tiles than SMs (every CTA loops, all ring phases wrap)
    (128 * 37, 2048, 192, torch.float16, False, False),       # 37 x 8 = 296 wide tiles, short K: epilogue-bound
    (128 * 41 + 5, 640, 320, torch.float16, False, False),    # narrow (BN=128) path, 5 x 42 = 210 tiles, M tail
    (4096, 1664, 128 * 9, torch.float16, True, True),         # wgrad, wide N with a tail tile (1664 = 6.5 x 256)
    (128 * 20, 1280, 4096, torch.float16, False, True),       # dgrad, N > 1024 not a multiple of 256
    (128 * 13, 4096, 80, torch.float16, False, False),        # the K = 80 mel projection at many tiles
    (1300, 2304, 160, torch.float32, False, False),           # tf32, wide
    # CTA-pair path (cta_group::2, 256 x 256 tiles: taken when there are >= 74 such tiles and no split-K)
    (128 * 40, 1280, 1024, torch.float16, False, True),       # dgrad, N tail tile (1280 = 5 x 256), B MN-major halves
    (5000, 1024, 256, torch.bfloat16, True, False),           # A MN-major, M tail inside a pair tile
    (2600, 2304, 160, torch.float32, False, False),           # tf32 pair, K tail
    (128 * 64 + 130, 4096, 1664, torch.float16, False, False),   # the layer-0 input projection shape class, peer half partly out of range
]


@pytest.mark.parametrize("pair_mode", [1, 2])
@pytest.mark.parametrize("M,N,K,dt,a_mn,b_mn", CASES)
def test_gemm_matches_fp64(M, N, K, dt, a_mn, b_mn, pair_mode):
    from flowtron_b200 import _lib
    if pair_mode == 2 and (N <= 1024 and N % 256) :
        pytest.skip("narrow output: never a CTA-pair tile")
    _lib.set_gemm_pair_mode(pair_mode)      # 2: CTA pairs (cta_group::2) whenever eligible, 1: the default policy
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N * 3 + K)
    A = (torch.randn((K, M) if a_mn else (M, K), device="cuda", generator=g) * 0.5).to(dt)
    B = (torch.randn((K, N) if b_mn else (N, K), device="cuda", generator=g) * 0.5).to(dt)
    bias = torch.randn(N, device="cuda", generator=g)
    out32 = torch.full((M, N), float("nan"), device="cuda")
    out16 = torch.zeros((M, N), device="cuda", dtype=torch.float16)
    _lib.gemm(A, B, a_mn=a_mn, b_mn=b_mn, bias=bias, out32=out32, out16=out16)
    torch.cuda.synchronize()
    assert _lib.device_status() == 0
    ref = _ref(A, B, a_mn, b_mn, bias, None, 0, 1.0)
    scale = ref.abs().max().item()
    err = (out32.double() - ref).abs().max().item()
    tol = 2e-3 if dt == torch.float32 else 1e-4      # tf32 truncates fp32 inputs; 16-bit inputs are exact
    assert err <= tol * scale, (err, scale)
    assert (out16.double() - ref).abs().max().item() <= 2e-3 * scale
    # a single output tensor leaves through TMA stores of staged tiles (the two-output call above uses per-lane stores)
    only32 = torch.full((M, N), float("nan"), device="cuda")
    only16 = torch.full((M, N), float("nan"), device="cuda", dtype=torch.float16)
    _lib.gemm(A, B, a_mn=a_mn, b_mn=b_mn, bias=bias, out32=only32)
    _lib.gemm(A, B, a_mn=a_mn, b_mn=b_mn, bias=bias, out16=only16)
    torch.cuda.synchronize()
    assert _lib.device_status() == 0
    assert torch.equal(only32, out32) and torch.equal(only16, out16)
    _lib.set_gemm_pair_mode(1)


def test_gemm_epilogue_tanh_beta_alpha_strided():
    from flowtron_b200 import _lib
    g = torch.Generator(device="cuda").manual_seed(1)
    M, N, K = 320, 192, 512
    Abig = (torch.randn(M, K + 64, device="cuda", generator=g) * 0.3).half()
    A = Abig[:, 32:32 + K]                                  # strided view (row pitch K+64, 64-byte offset)
    B = (torch.randn(N, K, device="cuda", generator=g) * 0.3).half()
    b1, b2 = torch.randn(N, device="cuda", generator=g), torch.randn(N, device="cuda", generator=g)
    Cbig = torch.randn(M, N + 32, device="cuda", generator=g)
    C = Cbig[:, 16:16 + N]
    c0 = C.clone()
    out16 = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
    _lib.gemm(A, B, bias=b1, bias2=b2, act=1, beta=1, alpha=0.5, out32=C, out16=out16)
    torch.cuda.synchronize()
    ref = _ref(A, B, False, False, b1, b2, 1, 0.5) + c0.double()
    assert (C.double() - ref).abs().max().item() < 1e-4
    assert (out16.double() - ref).abs().max().item() < 2e-2
    assert _lib.device_status() == 0


@pytest.mark.parametrize("M,N,K", [(1024, 1024, 8192), (640, 1024, 128 * 70 + 24), (128, 80, 4096 * 3)])
def test_gemm_split_k_weight_gradient_shapes(M, N, K):
    """dW = dY^T X with few output tiles and a long reduction: the persistent kernel splits K over the idle SMs and adds
    the partial tiles atomically into a zeroed fp32 output (alpha is applied per partial: the result stays alpha * sum)."""
    from flowtron_b200 import _lib
    g = torch.Generator(device="cuda").manual_seed(K)
    A = (torch.randn(K, M, device="cuda", generator=g) * 0.5).half()
    B = (torch.randn(K, N, device="cuda", generator=g) * 0.5).half()
    out = torch.full((M, N), float("nan"), device="cuda")
    _lib.gemm(A, B, a_mn=True, b_mn=True, alpha=0.25, out32=out)
    torch.cuda.synchronize()
    assert _lib.device_status() == 0
    ref = 0.25 * (A.double().t() @ B.double())
    assert (out.double() - ref).abs().max().item() <= 1e-4 * ref.abs().max().item()
