#!/usr/bin/env python
"""Write tests/golden/gemm_epilogue.json: the SHA-256 of every output of tests/gemm_epilogue_cases.py, computed with the
library of one checkout of this project (needs a GPU).  The recorded digests come from the build with fragment stores,
the commit before the staged TMA-store epilogue; tests/test_gpu_gemm_epilogue.py requires the current build to reproduce
them bit for bit.

    python tests/make_golden_gemm_epilogue.py [--tree DIR] [--out FILE]
"""
import argparse
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ap = argparse.ArgumentParser()
ap.add_argument("--tree", default=os.path.dirname(HERE), help="checkout whose flowtron_b200 library computes the outputs")
ap.add_argument("--out", default=os.path.join(HERE, "golden", "gemm_epilogue.json"))
args = ap.parse_args()
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.abspath(args.tree))
from flowtron_b200 import _lib  # noqa: E402
import gemm_epilogue_cases as C  # noqa: E402

res = {}
for case in C.CASES:
    outs = C.run_case(_lib, case)
    res[case[0]] = {k: C.digest(v) for k, v in outs.items()}
assert _lib.device_status() == 0
with open(args.out, "w") as f:
    json.dump(res, f, indent=1, sort_keys=True)
print(f"wrote {len(res)} cases to {args.out}")
