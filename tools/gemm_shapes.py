#!/usr/bin/env python
"""Isolated timing of every GEMM shape and epilogue the configs[1] training step (B = 32, T <= 1000) issues.

CUDA events over repeated launches, with three rotating operand sets so a launch does not find its operands in L2.
Per shape: ms and TFLOP/s with single-CTA tiles (pair mode 0, the default schedule by shape) and with CTA pairs wherever
eligible (pair mode 2), the epilogue's HBM floor (bytes the epilogue writes and reads over the copy bandwidth measured in
the same run) and, with --mainloop, the same kernels with their output stores compiled out (FT_GEMM_NO_STORE).  With
--schedules, also the cooperative schedule alone and the ping-pong schedule wherever it is eligible (FT_GEMM_SCHEDULE=1
/ 2).  Each variant is a private build of the GEMM translation units, in a
temporary directory or --builddir (reused when present there); the library the package loads is never touched.

    python tools/gemm_shapes.py [--tree DIR] [--mainloop] [--schedules] [--builddir DIR] [--only SUBSTR] [--json FILE]

--tree runs the library built in another checkout of this project (DIR/flowtron_b200), so two builds can be timed in
one session."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ap = argparse.ArgumentParser()
ap.add_argument("--tree", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
ap.add_argument("--mainloop", action="store_true", help="also time the main loop alone (stores compiled out)")
ap.add_argument("--schedules", action="store_true", help="also time the cooperative and the ping-pong schedule alone")
ap.add_argument("--builddir", default=None, help="directory for the private builds, reused when already there")
ap.add_argument("--only", default=None)
ap.add_argument("--json", default=None)
ap.add_argument("--reps", type=int, default=20)
args = ap.parse_args()
TREE = os.path.abspath(args.tree)
sys.path.insert(0, TREE)
import torch  # noqa: E402
from flowtron_b200 import _lib  # noqa: E402

R, L = 32000, 160          # B * T rows; B * L text rows below use RL = 5120
# name, M, N, K, a_mn, b_mn, out, epilogue: bias count, act, beta, aux (f16 [M, N] read), ldc (None: N)
SHAPES = [
    ("fwd xproj0", R, 4096, 1664, 0, 0, "f32", dict(nb=2)),
    ("fwd xproj0 last chunk", 7424, 4096, 1664, 0, 0, "f32", dict(nb=2)),
    ("fwd attn-lstm proj chunk", 8192, 4096, 80, 0, 0, "f32", dict(nb=2)),
    ("fwd xproj1 chunk", 3200, 4096, 1024, 0, 0, "f32", dict(nb=2)),
    ("fwd Q chunk", 8192, 640, 1024, 0, 0, "f32", dict()),
    ("fwd K/V", 5120, 640, 640, 0, 0, "f32", dict()),
    ("fwd dense tanh", R, 1024, 1024, 0, 0, "f16", dict(nb=1, act=1)),
    ("fwd conv", R, 160, 1024, 0, 0, "f32", dict(nb=1)),
    ("dgrad conv (f16 out)", R, 1024, 160, 0, 1, "f16", dict(aux=1)),
    ("dgrad dense (f16 out)", R, 1024, 1024, 0, 1, "f16", dict(aux=1)),
    ("dgrad dense -> dh", R, 1024, 1024, 0, 1, "f32", dict()),
    ("dgrad xproj1 chunk", 3200, 1024, 4096, 0, 1, "f32", dict()),
    ("dgrad ih0", R, 1664, 4096, 0, 1, "f32", dict()),
    ("dgrad dQ beta=1", R, 1024, 640, 0, 1, "f32", dict(beta=1, ldc=1664)),
    ("dgrad d_mel", R, 80, 4096, 0, 1, "f32", dict()),
    ("wgrad hh", 4096, 1024, R - 32, 1, 1, "f32", dict()),
    ("wgrad ih0", 4096, 1664, R, 1, 1, "f32", dict()),
    ("wgrad dense (split-K)", 1024, 1024, R, 1, 1, "f32", dict()),
    ("wgrad query (split-K)", 640, 1024, R, 1, 1, "f32", dict()),
    ("wgrad attn-lstm ih (split-K)", 4096, 80, R, 1, 1, "f32", dict()),
]


def gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:          # the card name from torch still identifies the device
        q = f"nvidia-smi unavailable: {type(e).__name__}"
    return name, q


def copy_bandwidth():
    """Device-to-device copy of 1 GiB: (read + write bytes) / time, GB/s."""
    n = 1 << 28
    a = torch.empty(n, device="cuda")
    b = torch.empty_like(a)
    for _ in range(3):
        b.copy_(a)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(10):
        b.copy_(a)
    e1.record()
    torch.cuda.synchronize()
    return 2 * 4 * n * 10 / (e0.elapsed_time(e1) / 1e3) / 1e9


VARIANTS = {"mainloop": "-DFT_GEMM_NO_STORE", "coop": "-DFT_GEMM_SCHEDULE=1", "pp": "-DFT_GEMM_SCHEDULE=2"}


def variant_lib(tree, name):
    """The GEMM translation units of `tree` rebuilt with VARIANTS[name], linked with the tree's other objects."""
    from flowtron_b200 import build as fb
    csrc, objdir = fb.CSRC, os.path.join(fb.HERE, "build")
    tmp = os.path.join(args.builddir, name) if args.builddir else tempfile.mkdtemp(prefix=f"gemm_{name}_")
    lib = os.path.join(tmp, "libflowtron_b200.so")
    if os.path.exists(lib):
        return lib
    os.makedirs(tmp, exist_ok=True)
    gemm_srcs = [s for s in fb.sources() if s.startswith("gemm")]
    procs = [subprocess.Popen([fb.NVCC, *fb.FLAGS, VARIANTS[name], "-c", os.path.join(csrc, s), "-o",
                               os.path.join(tmp, s[:-3] + ".o")], stdout=subprocess.DEVNULL, stderr=subprocess.PIPE)
             for s in gemm_srcs]
    for p in procs:
        if p.wait() != 0:
            raise RuntimeError(p.stderr.read().decode())
    objs = [os.path.join(tmp, s[:-3] + ".o") if s in gemm_srcs else os.path.join(objdir, s[:-3] + ".o") for s in fb.sources()]
    subprocess.run([fb.NVCC, "-shared", "-o", lib, *objs, "-gencode", "arch=compute_90a,code=sm_90a", "-cudart", "shared",
                    "-lcufft", "-Xlinker", "-rpath,/usr/local/cuda/lib64"], check=True, capture_output=True)
    return lib


def run_shape(shape, modes):
    name, M, N, K, a_mn, b_mn, out, e = shape
    nb, act, beta, aux, ldc = e.get("nb", 0), e.get("act", 0), e.get("beta", 0), e.get("aux", 0), e.get("ldc", N)
    nbuf = 3
    g = torch.Generator(device="cuda").manual_seed(0)
    As = [(torch.randn((K, M) if a_mn else (M, K), device="cuda", generator=g) * 0.3).half() for _ in range(nbuf)]
    Bs = [(torch.randn((K, N) if b_mn else (N, K), device="cuda", generator=g) * 0.3).half() for _ in range(nbuf)]
    bias = torch.randn(N, device="cuda", generator=g) if nb >= 1 else None
    bias2 = torch.randn(N, device="cuda", generator=g) if nb >= 2 else None
    o32 = torch.zeros(M, ldc, device="cuda")[:, :N] if out == "f32" else None
    o16 = torch.empty(M, N, device="cuda", dtype=torch.float16) if out == "f16" else None
    res = {}
    for mode in modes:
        _lib.set_gemm_pair_mode(mode)

        def call(i):
            _lib.gemm(As[i % nbuf], Bs[i % nbuf], a_mn=bool(a_mn), b_mn=bool(b_mn), bias=bias, bias2=bias2, act=act,
                      beta=beta, out32=o32, out16=o16)
        for i in range(3):
            call(i)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(args.reps):
            call(i)
        e1.record()
        torch.cuda.synchronize()
        assert _lib.device_status() == 0
        res[mode] = e0.elapsed_time(e1) / args.reps
    _lib.set_gemm_pair_mode(0)          # the default policy
    # what the epilogue itself moves through HBM (the aux read of act = 2 is not reachable through ft_gemm; counted)
    esz = 4 if out == "f32" else 2
    epi_bytes = M * N * esz + (M * N * 4 if beta else 0) + (M * N * 2 if aux else 0)
    return res, epi_bytes


def main():
    child = os.environ.get("FT_GEMM_SHAPES_CHILD") == "1"
    if child:                       # one variant library: its single-CTA times only
        _lib.LIB_PATH = os.environ["FT_GEMM_SHAPES_LIB"]
        ms = {s[0]: run_shape(s, (0,))[0][0] for s in SHAPES if not args.only or args.only in s[0]}
        print(json.dumps({"ms": ms}))
        return
    # two libraries cannot share the process: each variant runs in a child
    names = (["mainloop"] if args.mainloop else []) + (["coop", "pp"] if args.schedules else [])
    libs = {n: variant_lib(TREE, n) for n in names}
    var = {}
    for n in names:
        env = dict(os.environ, FT_GEMM_SHAPES_CHILD="1", FT_GEMM_SHAPES_LIB=libs[n])
        out = subprocess.run([sys.executable, __file__, "--tree", TREE, "--reps", str(args.reps)] +
                             (["--only", args.only] if args.only else []), env=env, capture_output=True, text=True)
        if out.returncode != 0:
            raise RuntimeError(out.stderr)
        var[n] = json.loads(out.stdout.strip().splitlines()[-1])["ms"]
    name, smi = gpu_info()
    bw = copy_bandwidth()
    rows = []
    print(f"# {name} | {smi} | copy bandwidth {bw:.0f} GB/s | tree {TREE}")
    cols = "".join(f" | {n:>8s} ms" for n in ("coop", "pp") if n in var)
    print(f"{'shape':30s} {'M x N x K':>22s} | {'single ms':>9s} {'TF/s':>6s} | {'pair ms':>8s} {'TF/s':>6s}{cols} | "
          f"{'epi floor':>9s} | {'main loop':>9s} {'share':>6s}")
    for s in SHAPES:
        if args.only and args.only not in s[0]:
            continue
        nm, M, N, K = s[:4]
        res, eb = run_shape(s, (0, 2))
        tf = lambda ms: 2.0 * M * N * K / ms / 1e9
        floor = eb / (bw * 1e9) * 1e3
        ml = var.get("mainloop", {}).get(nm)
        mls = f"{ml:9.3f} {ml / res[0] * 100:5.0f}%" if ml else f"{'-':>9s} {'':>6s}"
        sch = "".join(f" | {var[n][nm]:11.3f}" for n in ("coop", "pp") if n in var)
        print(f"{nm:30s} {M:6d} x {N:5d} x {K:6d} | {res[0]:9.3f} {tf(res[0]):6.1f} | {res[2]:8.3f} {tf(res[2]):6.1f}{sch} | "
              f"{floor:9.3f} | {mls}")
        rows.append(dict(shape=nm, M=M, N=N, K=K, single_ms=res[0], pair_ms=res[2], epi_bytes=eb, epi_floor_ms=floor,
                         mainloop_ms=ml, coop_ms=var.get("coop", {}).get(nm), pp_ms=var.get("pp", {}).get(nm)))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(gpu=name, nvidia_smi=smi, copy_gbps=bw, tree=TREE, rows=rows), f, indent=1)

main()
