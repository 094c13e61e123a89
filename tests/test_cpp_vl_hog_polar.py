"""The C++14 shell's dense HOG of gradient fields, rcr::vl_hog_polar (tests/cpp/test_vl_hog_polar.cpp).

CPU: the translation unit compiles.  GPU: on fields of different sizes held with row steps wider than their pixels, nearest-bin
and bilinear, directed and undirected, the shell returns, field by field, the Python vl_hog_polar result bit for bit, as
dd * hogH rows of hogW columns; pairs of different sizes, other types and refused configurations throw."""
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def vl_hog_polar_binary(tmp_path_factory):
    from superviseddescent_b200 import build
    lib = build.build()
    out = str(tmp_path_factory.mktemp("cpp") / "test_vl_hog_polar")
    cmd = ["g++", "-std=c++14", "-O1", "-Wall", "-Werror=return-type", "-I", os.path.join(ROOT, "include"),
           "-I", os.path.join(ROOT, "superviseddescent_b200", "include"), os.path.join(ROOT, "tests", "cpp", "test_vl_hog_polar.cpp"),
           "-L", os.path.dirname(lib), "-lsd_b200", f"-Wl,-rpath,{os.path.dirname(lib)}", "-lpthread", "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return out


def test_vl_hog_polar_shell_compiles_as_cxx14(vl_hog_polar_binary):
    assert os.path.exists(vl_hog_polar_binary)


@pytest.mark.gpu
@pytest.mark.parametrize("cs,K,variant,directed,bilinear", [(8, 9, 1, 1, 0), (6, 4, 0, 0, 1), (4, 9, 1, 0, 0), (11, 16, 0, 1, 1)])
def test_shell_vl_hog_polar_matches_python(vl_hog_polar_binary, sd, tmp_path, cs, K, variant, directed, bilinear):
    rng = np.random.default_rng(cs * 10 + K)
    sizes = [(120, 160), (97, 131), (37, 29)]
    mods, angs = [], []
    for h, w in sizes:
        mods.append(np.where(rng.random((h, w)) < 0.1, 0, rng.normal(1, 1, (h, w))).astype(np.float32))
        angs.append(rng.uniform(-4 * np.pi, 4 * np.pi, (h, w)).astype(np.float32))
    blob = [np.array([len(sizes)], dtype=np.int32).tobytes()]
    for m, a in zip(mods, angs):
        blob += [np.array([m.shape[1], m.shape[0]], dtype=np.int32).tobytes(), m.tobytes(), a.tobytes()]
    (tmp_path / "in.bin").write_bytes(b"".join(blob))
    r = subprocess.run([vl_hog_polar_binary, str(tmp_path / "in.bin"), str(tmp_path / "out.bin"), str(cs), str(K), str(variant),
                        str(directed), str(bilinear)], capture_output=True, text=True, timeout=300)
    print(r.stdout[-3000:])
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
    raw = (tmp_path / "out.bin").read_bytes()
    want = sd.vl_hog_polar(mods, angs, cs, K, variant, directed=bool(directed), bilinear_orientations=bool(bilinear))
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
