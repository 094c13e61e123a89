"""The C++14 shells with rcr-train's shallow copies of each photo (tests/cpp/test_train_host_frames.cpp).

CPU: the translation unit compiles.  GPU: each photo is held on the device once, and training and testing give bit for bit the
results of the same set built from deep copies; with the route threshold lowered the frames stay in host memory and training and
testing give bit for bit the device route's results."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def host_frames_binary(tmp_path_factory):
    from superviseddescent_b200 import build
    lib = build.build()
    out = str(tmp_path_factory.mktemp("cpp") / "test_train_host_frames")
    cmd = ["g++", "-std=c++14", "-O1", "-Wall", "-Werror=return-type", "-I", os.path.join(ROOT, "include"),
           "-I", os.path.join(ROOT, "superviseddescent_b200", "include"), os.path.join(ROOT, "tests", "cpp", "test_train_host_frames.cpp"),
           "-L", os.path.dirname(lib), "-lsd_b200", f"-Wl,-rpath,{os.path.dirname(lib)}", "-lpthread", "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return out


def test_train_host_frames_compiles_as_cxx14(host_frames_binary):
    assert os.path.exists(host_frames_binary)


@pytest.mark.gpu
def test_shell_uploads_each_photo_once(host_frames_binary, golden):
    r = subprocess.run([host_frames_binary, golden.model_path], capture_output=True, text=True, timeout=600)
    print(r.stdout[-3000:])
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
    assert "FRAMES shallow 40 deep 440" in r.stdout and "\nTEST: 0.000e+00" in r.stdout
    assert "HOST ROUTE on_device 0 frames 40" in r.stdout and "HOST TEST: 0.000e+00" in r.stdout
