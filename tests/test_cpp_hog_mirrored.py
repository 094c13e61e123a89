"""Mirrored entries in the C++14 shells (tests/cpp/test_hog_mirrored.cpp).

CPU: the translation unit compiles as C++14.  GPU: training and testing on shallow copies marked mirrored in rcr::HogTransform give
bit for bit the results of hand-flipped deep copies, on the device route and on the host route, with each photo held once;
rcr::mirror_permutation of the rcr_22 list is the known answer of the Python helper."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def mirrored_binary(tmp_path_factory):
    from superviseddescent_b200 import build
    lib = build.build()
    out = str(tmp_path_factory.mktemp("cpp") / "test_hog_mirrored")
    cmd = ["g++", "-std=c++14", "-O1", "-Wall", "-Werror=return-type", "-I", os.path.join(ROOT, "include"),
           "-I", os.path.join(ROOT, "superviseddescent_b200", "include"), os.path.join(ROOT, "tests", "cpp", "test_hog_mirrored.cpp"),
           "-L", os.path.dirname(lib), "-lsd_b200", f"-Wl,-rpath,{os.path.dirname(lib)}", "-lpthread", "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return out


def test_hog_mirrored_compiles_as_cxx14(mirrored_binary):
    assert os.path.exists(mirrored_binary)


@pytest.mark.gpu
def test_shell_mirrored_entries_equal_flipped_copies(mirrored_binary, golden):
    r = subprocess.run([mirrored_binary, golden.model_path], capture_output=True, text=True, timeout=600)
    print(r.stdout[-3000:])
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
    assert "PERM 0 1 3 2 13 12 11 10 15 14 7 6 5 4 9 8 18 17 16 19 20 21\n" in r.stdout
    assert "FRAMES mirrored 12 copies 24" in r.stdout
    for line in ("TEST: 0.000e+00", "HOST TEST: 0.000e+00", "FUNCTOR: 0.000e+00"):
        assert "\n" + line in r.stdout, line
