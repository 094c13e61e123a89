"""The C++14 shell's dense HOG of multi-channel frames, rcr::vl_hog (tests/cpp/test_vl_hog.cpp).

CPU: the translation unit compiles.  GPU: on 8-bit and float frames of three planes and different sizes (row steps wider than the
pixels), nearest-bin and bilinear, the shell returns, frame by frame, the Python vl_hog result bit for bit, as dd * hogH rows of
hogW columns."""
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def vl_hog_binary(tmp_path_factory):
    from superviseddescent_b200 import build
    lib = build.build()
    out = str(tmp_path_factory.mktemp("cpp") / "test_vl_hog")
    cmd = ["g++", "-std=c++14", "-O1", "-Wall", "-Werror=return-type", "-I", os.path.join(ROOT, "include"),
           "-I", os.path.join(ROOT, "superviseddescent_b200", "include"), os.path.join(ROOT, "tests", "cpp", "test_vl_hog.cpp"),
           "-L", os.path.dirname(lib), "-lsd_b200", f"-Wl,-rpath,{os.path.dirname(lib)}", "-lpthread", "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return out


def test_vl_hog_shell_compiles_as_cxx14(vl_hog_binary):
    assert os.path.exists(vl_hog_binary)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.uint8, np.float32])
@pytest.mark.parametrize("cs,K,variant,bilinear", [(8, 9, 1, 0), (6, 4, 0, 1)])
def test_shell_vl_hog_matches_python(vl_hog_binary, sd, tmp_path, dtype, cs, K, variant, bilinear):
    rng = np.random.default_rng(cs * 10 + K)
    sizes = [(120, 160), (97, 131), (37, 29)]
    frames = []
    for h, w in sizes:
        f = rng.integers(0, 256, (3, h, w)).astype(dtype)
        frames.append(f / np.float32(255) if dtype == np.float32 else f)
    frames = [np.ascontiguousarray(f, dtype=dtype) for f in frames]
    blob = [np.array([len(frames), 3, 0 if dtype == np.uint8 else 1], dtype=np.int32).tobytes()]
    for f in frames:
        blob += [np.array([f.shape[2], f.shape[1]], dtype=np.int32).tobytes(), f.tobytes()]
    (tmp_path / "in.bin").write_bytes(b"".join(blob))
    r = subprocess.run([vl_hog_binary, str(tmp_path / "in.bin"), str(tmp_path / "out.bin"), str(cs), str(K), str(variant), str(bilinear)],
                       capture_output=True, text=True, timeout=300)
    print(r.stdout[-3000:])
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
    raw = (tmp_path / "out.bin").read_bytes()
    want = sd.vl_hog(frames, cs, K, variant, bilinear_orientations=bool(bilinear))
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
