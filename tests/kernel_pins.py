"""Pin what nvcc makes of a CUDA source: each kernel's registers and spills (-Xptxas -v) and a hash of its SASS instructions
(cuobjdump -sass, addresses and encodings stripped).  A host-side refactor that moves device code between files compares
these against a table recorded before the move, so the kernels themselves are shown not to change."""
import hashlib
import os
import re
import shutil
import subprocess

from conftest import ROOT

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
HAVE_NVCC = os.path.exists(NVCC) or shutil.which("nvcc") is not None


def _compile(src, tmp_path):
    obj = str(tmp_path / (src + ".o"))
    r = subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                        "--expt-relaxed-constexpr", "-Xptxas", "-v", "-c", os.path.join(ROOT, "flowtron_b200", "csrc", src),
                        "-o", obj], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    regs = {}
    for part in r.stderr.split("Compiling entry function")[1:]:
        name = re.match(r"\s*'(\S+)'", part).group(1)
        spill = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", part).groups()
        regs[name] = (int(re.search(r"Used (\d+) registers", part).group(1)), spill)
    return obj, regs


def _sass_hashes(obj):
    cuobjdump = os.path.join(os.path.dirname(NVCC), "cuobjdump") if os.path.exists(NVCC) else shutil.which("cuobjdump")
    text = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    out, cur = {}, None
    for line in text.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            out[cur] = []
        elif cur and line.strip().startswith("/*") and "*/" in line:
            ins = re.sub(r"/\*[0-9a-f]{4,}\*/", "", line.split("/* 0x")[0]).strip()
            if ins:
                out[cur].append(ins)
    return {k: hashlib.sha256("\n".join(v).encode()).hexdigest()[:16] for k, v in out.items()}


def _stable_name(name):
    """The mangled name with an anonymous namespace's per-build identifier (<len>_GLOBAL__N__<hashes of the path>) replaced."""
    m = re.search(r"(\d+)_GLOBAL__N_", name)
    if not m:
        return name
    return name[:m.start()] + "_GLOBAL__N_" + name[m.start(1) + len(m.group(1)) + int(m.group(1)):]


def kernel_table(src, tmp_path):
    """{kernel: (registers, (spill stores, spill loads), SASS hash)} of one source under flowtron_b200/csrc."""
    obj, regs = _compile(src, tmp_path)
    sass = _sass_hashes(obj)
    assert set(regs) == set(sass)
    return {_stable_name(name): (r, spill, sass[name]) for name, (r, spill) in regs.items()}


def _assert_kernels_pinned(src, table, tmp_path):
    got = kernel_table(src, tmp_path)
    assert set(got) == set(table)
    for name, want in table.items():
        assert got[name][:2] == want[:2], name
        assert got[name][2] == want[2], name
