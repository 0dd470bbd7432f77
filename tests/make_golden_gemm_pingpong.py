"""Write tests/golden/gemm_pingpong.json: the SHA-256 of every output of gemm_pingpong_cases.CASES, computed with the
library of TREE (default: this checkout).  The digests were written with the build before the ping-pong schedule existed,
which runs every case on the cooperative schedule, so the test checks that the two schedules agree bit for bit.

    python tests/make_golden_gemm_pingpong.py [TREE] [OUT]"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
TREE = os.path.abspath(sys.argv[1]) if len(sys.argv) > 1 else os.path.dirname(HERE)
OUT = sys.argv[2] if len(sys.argv) > 2 else os.path.join(HERE, "golden", "gemm_pingpong.json")
sys.path.insert(0, HERE)
sys.path.insert(0, TREE)
import gemm_pingpong_cases as C  # noqa: E402
from flowtron_b200 import _lib  # noqa: E402

out = {}
for case in C.CASES:
    outs = C.run_case(_lib, case)
    assert _lib.device_status() == 0
    out[case[0]] = {k: C.digest(v) for k, v in outs.items()}
with open(OUT, "w") as f:
    json.dump(out, f, indent=1)
print(f"wrote {len(out)} cases to {OUT}")
