"""CPU-side checks of the drop-in boundary: the library loads and exports every declared symbol."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def built_lib():
    from superviseddescent_b200 import build
    return build.build()


def test_header_symbols_are_exported(built_lib):
    header = open(os.path.join(ROOT, "include", "sd_b200.h")).read()
    declared = set(re.findall(r"SD_API\s+[\w\s\*]+?\b(sd_\w+)\s*\(", header))
    assert len(declared) >= 40
    lib = ctypes.CDLL(built_lib)
    missing = [s for s in sorted(declared) if not hasattr(lib, s)]
    assert not missing, f"declared in include/sd_b200.h but not exported: {missing}"
    from superviseddescent_b200 import _capi
    assert set(_capi.EXPORTS) == declared


def test_no_oracle_in_product():
    """The product package and the public header must not import, link or reference anything under oracle/ (only tests/,
    smoke() and bench.py's CPU baseline may)."""
    for top in ("superviseddescent_b200", "include"):
        for dirpath, _, files in os.walk(os.path.join(ROOT, top)):
            for f in files:
                if f.endswith((".py", ".cu", ".cuh", ".hpp", ".h", ".cpp", ".sh")):
                    text = open(os.path.join(dirpath, f), errors="ignore").read()
                    assert "sd_oracle" not in text and "from oracle" not in text and "import oracle" not in text, os.path.join(dirpath, f)


def test_fails_loudly_without_gpu(built_lib):
    """No CPU fallback: creating a context without a usable device is an error."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    lib = ctypes.CDLL(built_lib)
    h = ctypes.c_void_p()
    assert lib.sd_ctx_create(0, None, ctypes.byref(h)) != 0
    from superviseddescent_b200 import api
    with pytest.raises(Exception):
        api.Context(0)


def test_align_mean_host_function(built_lib):
    """sd_align_mean is pure host code: check it against the formula of model.hpp:72-73."""
    import numpy as np
    from superviseddescent_b200 import api
    mean = np.linspace(-0.4, 0.4, 44).astype(np.float32)
    out = api.align_mean(mean, (100, 50, 240, 260))
    exp_x = (mean[:22] * 1.0 + 0.5) * 240 + 100
    exp_y = (mean[22:] * 1.0 + 0.5) * 260 + 50
    assert np.allclose(out[:22], exp_x, rtol=0, atol=1e-3) and np.allclose(out[22:], exp_y, rtol=0, atol=1e-3)


def test_host_side_functions_match_the_oracle(built_lib):
    """sd_align_mean and sd_perturb_box are pure host code (no device needed): bit-exact against the oracle's restatement
    of model.hpp:64-76 and apps/rcr/rcr-train.cpp:130-146 on random inputs."""
    import numpy as np
    from oracle import oracle as O
    from superviseddescent_b200 import api
    O.build()
    rng = np.random.default_rng(11)
    mean = rng.uniform(-0.5, 0.5, 44).astype(np.float32)
    for _ in range(300):
        box = (int(rng.integers(-50, 600)), int(rng.integers(-50, 400)), int(rng.integers(10, 400)), int(rng.integers(10, 400)))
        sx, sy = float(rng.normal(1, 0.05)), float(rng.normal(1, 0.05))
        tx, ty = float(rng.normal(0, 0.05)), float(rng.normal(0, 0.05))
        assert np.array_equal(api.align_mean(mean, box, sx, sy, tx, ty), O.align_mean(mean, box, sx, sy, tx, ty))
        assert api.perturb(box, tx, ty, sx) == O.perturb_box(box, tx, ty, sx)
