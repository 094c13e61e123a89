"""The C++14 shell's dense HOG of whole frames, rcr::hog_dense (tests/cpp/test_hog_dense.cpp).

CPU: the translation unit compiles.  GPU: on grey and colour frames of different sizes (row steps wider than the pixels) the
shell returns, frame by frame, the Python hog_dense result bit for bit, as dd * hogH rows of hogW columns."""
import os
import subprocess

import numpy as np
import pytest

import synth
from colour_examples import bgr_with_gray

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def dense_binary(tmp_path_factory):
    from superviseddescent_b200 import build
    lib = build.build()
    out = str(tmp_path_factory.mktemp("cpp") / "test_hog_dense")
    cmd = ["g++", "-std=c++14", "-O1", "-Wall", "-Werror=return-type", "-I", os.path.join(ROOT, "include"),
           "-I", os.path.join(ROOT, "superviseddescent_b200", "include"), os.path.join(ROOT, "tests", "cpp", "test_hog_dense.cpp"),
           "-L", os.path.dirname(lib), "-lsd_b200", f"-Wl,-rpath,{os.path.dirname(lib)}", "-lpthread", "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return out


def test_hog_dense_shell_compiles_as_cxx14(dense_binary):
    assert os.path.exists(dense_binary)


@pytest.mark.gpu
@pytest.mark.parametrize("cs,K,variant", [(8, 9, 1), (6, 4, 0)])
def test_shell_hog_dense_matches_python(dense_binary, sd, tmp_path, cs, K, variant):
    rng = np.random.default_rng(cs * 10 + K)
    sizes = [(120, 160), (97, 131), (37, 29)]
    grey = [synth.smooth_images(1, h, w, seed=60 + i)[0] for i, (h, w) in enumerate(sizes)]
    frames = [grey[0], bgr_with_gray(grey[1], rng.integers(-40, 41, grey[1].shape), rng.integers(-40, 41, grey[1].shape)), grey[2]]
    blob = [np.int32(len(frames)).tobytes()]
    for f in frames:
        ch = 1 if f.ndim == 2 else 3
        blob += [np.array([f.shape[1], f.shape[0], ch], dtype=np.int32).tobytes(), np.ascontiguousarray(f).tobytes()]
    (tmp_path / "in.bin").write_bytes(b"".join(blob))
    r = subprocess.run([dense_binary, str(tmp_path / "in.bin"), str(tmp_path / "out.bin"), str(cs), str(K), str(variant)],
                       capture_output=True, text=True, timeout=300)
    print(r.stdout[-3000:])
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
    raw = (tmp_path / "out.bin").read_bytes()
    want = sd.hog_dense(frames, cs, K, variant)
    pos = 0
    for w in want:
        rows, cols = np.frombuffer(raw, dtype=np.int32, count=2, offset=pos)
        pos += 8
        got = np.frombuffer(raw, dtype=np.float32, count=rows * cols, offset=pos).reshape(rows, cols)
        pos += 4 * rows * cols
        w = w.cpu().numpy()
        assert (rows, cols) == (w.shape[0] * w.shape[1], w.shape[2])
        assert np.array_equal(got, w.reshape(rows, cols))
    assert pos == len(raw)
