import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device")
    config.addinivalue_line("markers", "needs_reference: needs /root/reference (build container only)")


def pytest_collection_modifyitems(config, items):
    import torch
    has_gpu = torch.cuda.is_available()
    for item in items:
        if "gpu" in item.keywords and not has_gpu:
            item.add_marker(pytest.mark.skip(reason="no CUDA device"))


def record_parity(test: str, values: dict) -> None:
    """Append the measured parity errors of a GPU test to gpurun_out/parity.jsonl (scratch, merged back by gpurun) so the
    numbers behind a green run can be committed under profiles/."""
    import json
    d = os.path.join(ROOT, "gpurun_out")
    try:
        os.makedirs(d, exist_ok=True)
        with open(os.path.join(d, os.environ.get("FT_PARITY_LOG", "parity.jsonl")), "a") as f:
            f.write(json.dumps({"test": test, **{k: (float(v) if isinstance(v, (int, float)) else v) for k, v in values.items()}}) + "\n")
    except OSError:
        pass
