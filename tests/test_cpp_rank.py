"""The C++14 shells' rank diagnostic on the optimiser's device route (tests/cpp/test_rank.cpp).

CPU: the translation unit compiles.  GPU: a QR-solver cascade reports full rank on MatrixNorm-regularised levels, and an
unregularised level with fewer samples than features prints the reference's message and throws with the same rank."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def rank_binary(tmp_path_factory):
    from superviseddescent_b200 import build
    lib = build.build()
    out = str(tmp_path_factory.mktemp("cpp") / "test_rank")
    cmd = ["g++", "-std=c++14", "-O1", "-Wall", "-Werror=return-type", "-I", os.path.join(ROOT, "include"),
           "-I", os.path.join(ROOT, "superviseddescent_b200", "include"), os.path.join(ROOT, "tests", "cpp", "test_rank.cpp"),
           "-L", os.path.dirname(lib), "-lsd_b200", f"-Wl,-rpath,{os.path.dirname(lib)}", "-lpthread", "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return out


def test_rank_compiles_as_cxx14(rank_binary):
    assert os.path.exists(rank_binary)


@pytest.mark.gpu
def test_shell_optimiser_reports_rank(rank_binary, golden):
    r = subprocess.run([rank_binary, golden.model_path], capture_output=True, text=True, timeout=600)
    print(r.stdout[-3000:])
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
    assert "RANK level 0: 3169 of 3169" in r.stdout and "RANK level 1: 3169 of 3169" in r.stdout
    m = re.search(r"DEFICIENT level 0: (\d+) of 3169", r.stdout)
    assert m and 0 < int(m.group(1)) < 3169
    assert f"(The rank is {m.group(1)}, full rank would be 3169). Increase lambda." in r.stdout   # regressors.hpp:290-293
