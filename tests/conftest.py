import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def oracle():
    """The CPU oracle (test infrastructure).  Built on demand with gcc."""
    from oracle import oracle as O
    O.build()
    return O


@pytest.fixture(scope="session")
def golden():
    class G:
        dir = GOLDEN
        model_path = os.path.join(GOLDEN, "face_landmarks_model_rcr_22.bin")
        examples = np.load(os.path.join(GOLDEN, "examples.npz"))
        resize = np.load(os.path.join(GOLDEN, "resize_cv2.npz"))
        hog = np.load(os.path.join(GOLDEN, "hog_ref.npz"))
        detect = np.load(os.path.join(GOLDEN, "detect_ref.npz"))
        mean68 = np.load(os.path.join(GOLDEN, "mean_ibug_lfpw_68.npy"))
    return G


@pytest.fixture(scope="session")
def sd():
    """The product API bound to cuda:0 (GPU tests only)."""
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from superviseddescent_b200 import api
    return api


def rel_err(a, b):
    """max-norm error relative to the max-abs of the reference tensor (SURVEY 8d parity gate)."""
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-30))
