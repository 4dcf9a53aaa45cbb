import json
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100: pytest -m gpu)")


def pytest_collection_modifyitems(config, items):
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


def pytest_sessionfinish(session, exitstatus):
    """On a GPU box: dump the worst err/tol ratio every parity test observed (to $B2Q_PARITY_JSON)."""
    if not torch.cuda.is_available():
        return
    try:
        import helpers
        if helpers.PARITY_LOG:
            out = os.environ.get("B2Q_PARITY_JSON", os.path.join(ROOT, "gpurun_out", "parity.json"))
            os.makedirs(os.path.dirname(out), exist_ok=True)
            with open(out, "w") as f:
                json.dump({"tolerance": "|out-ref| <= rel*|ref| + rel*rms(ref)", "exitstatus": int(exitstatus),
                           "tests": helpers.PARITY_LOG}, f, indent=1, sort_keys=True)
    except Exception as e:  # never let bookkeeping fail the run
        print("parity log not written:", e)


class RefCases:
    """tests/golden/ref_cases.npz — outputs of the reference's TorchLinear/TorchAtenLinear (make_golden.py)."""

    def __init__(self):
        z = np.load(os.path.join(GOLDEN, "ref_cases.npz"))
        self.z = z
        self.meta = json.loads(bytes(z["__meta__"]).decode())

    def names(self):
        return list(self.meta.keys())

    def get(self, name, key, dtype=None):
        k = f"{name}.{key}"
        if k not in self.z.files:
            return None
        t = torch.from_numpy(self.z[k])
        return t.to(dtype) if dtype is not None else t


@pytest.fixture(scope="session")
def ref_cases():
    return RefCases()


@pytest.fixture(scope="session")
def q4_golden():
    with open(os.path.join(GOLDEN, "q4_reference.json")) as f:
        return json.load(f)
