"""The C++14 shells' chunked training and testing on the optimiser's device route (tests/cpp/test_train_chunks.cpp).

CPU: the translation unit compiles.  GPU: set_rows_per_chunk(300) trains within 1e-5 of one chunk, and the chunked test()
equals the unchunked one."""
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def chunks_binary(tmp_path_factory):
    from superviseddescent_b200 import build
    lib = build.build()
    out = str(tmp_path_factory.mktemp("cpp") / "test_train_chunks")
    cmd = ["g++", "-std=c++14", "-O1", "-Wall", "-Werror=return-type", "-I", os.path.join(ROOT, "include"),
           "-I", os.path.join(ROOT, "superviseddescent_b200", "include"), os.path.join(ROOT, "tests", "cpp", "test_train_chunks.cpp"),
           "-L", os.path.dirname(lib), "-lsd_b200", f"-Wl,-rpath,{os.path.dirname(lib)}", "-lpthread", "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return out


def test_train_chunks_compiles_as_cxx14(chunks_binary):
    assert os.path.exists(chunks_binary)


@pytest.mark.gpu
def test_shell_optimiser_trains_in_chunks(chunks_binary, golden):
    r = subprocess.run([chunks_binary, golden.model_path], capture_output=True, text=True, timeout=600)
    print(r.stdout[-3000:])
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
    assert len(re.findall(r"WEIGHTS level \d: ", r.stdout)) == 2 and "TEST: 0.000e+00" in r.stdout
