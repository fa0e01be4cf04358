import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100, sm_90a)")


@pytest.fixture(scope="session", autouse=True)
def _fresh_library():
    """Rebuild libgraphsage_b200.so if any source is newer than it (no-op otherwise)."""
    from graphsage_b200.build import build_library
    build_library()


def load_golden(name):
    return np.load(os.path.join(GOLDEN, name + ".npz"))


@pytest.fixture(scope="session")
def golden():
    return load_golden


def rel_err(y, ref, floor=1e-6):
    """max over rows of ||y - ref||_inf / max(||ref||_inf, floor) - the 1e-4 parity metric (SURVEY 8c)."""
    y = np.asarray(y, dtype=np.float64)
    ref = np.asarray(ref, dtype=np.float64)
    num = np.abs(y - ref).reshape(len(ref), -1).max(axis=1)
    den = np.maximum(np.abs(ref).reshape(len(ref), -1).max(axis=1), floor)
    return float((num / den).max()) if len(ref) else 0.0


def elem_err(y, ref, atol=1e-6):
    """Elementwise companion of rel_err (SURVEY 8c): max |y - ref| / (|ref| + atol-floor scaled by the row's magnitude).
    An element counts relative to max(|ref_ij|, 1e-2 * ||ref_i||_inf, atol): small entries of a row are judged against
    the row's scale (they are sums of O(row scale) terms), large ones against themselves."""
    y = np.asarray(y, dtype=np.float64)
    ref = np.asarray(ref, dtype=np.float64)
    if not len(ref):
        return 0.0
    rows = np.abs(ref).reshape(len(ref), -1).max(axis=1, keepdims=True)
    den = np.maximum(np.maximum(np.abs(ref).reshape(len(ref), -1), 1e-2 * rows), atol)
    return float((np.abs(y - ref).reshape(len(ref), -1) / den).max())


def bf16_round(x):
    """float32 -> nearest-even bfloat16 -> float32 (numpy), the rounding the CUDA bf16 operands get."""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16
    return r.astype(np.uint32).view(np.float32).reshape(np.shape(x))
