"""pytest configuration: `gpu` marker + shared fixtures (goldens, oracle, seeded graphs)."""
import json
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
GOLDEN = ROOT / "tests" / "golden"
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def pytest_collection_modifyitems(config, items):
    # GPU tests are selected with `-m gpu`; when a GPU is absent they are skipped, never faked.
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:  # pragma: no cover
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def goldens():
    return json.loads((GOLDEN / "reference_goldens.json").read_text())


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


@pytest.fixture(scope="session")
def scale8_edges():
    import oracle
    src, dst, n = oracle.graph500_decode((GOLDEN / "scale_8.graph500").read_bytes())
    return src, dst, n


LAYOUTS = {"Unsorted": 0, "Sorted": 1, "Deduplicated": 2}


def edges_to_arrays(edges):
    e = np.asarray(edges)
    src = np.ascontiguousarray(e[:, 0]).astype(np.uint32)
    dst = np.ascontiguousarray(e[:, 1]).astype(np.uint32)
    w = np.ascontiguousarray(e[:, 2]).astype(np.float32) if e.shape[1] > 2 else None
    return src, dst, w
