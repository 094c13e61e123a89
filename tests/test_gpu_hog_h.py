"""The hog.h drop-in against the reference's hog.c: one driver program (oracle/vl_hog_driver.cpp), written against the hog.h API
alone, built against the reference (oracle/_ref/vl_hog_driver_ref) and against this project's shell, runs one case list:
put_image with 1 / 3 / 16 channels, bilinear on and off, transposed on and off, both variants, K 1 / 4 / 9 / 16, cell sizes
1 / 4 / 8 / 11 / 32, frames from 4 x 4 to 1920 x 1080; one object reused across sizes; put_polar_field directed and undirected;
render into a non-zero image with a NaN pixel.

  - dims, get_dimension, the permutation and the glyph size are equal; features and renders are within the project bar;
  - bit identities: put_image + extract is vl_hog of the same frame, and in transposed mode vl_hog of the transposed view with
    its planes transposed; put_polar_field is vl_hog_polar the same way;
  - the driver overwrites each host input right after the put, and four threads with their own objects write the
    single-thread dump byte for byte."""
import os
import subprocess

import numpy as np
import pytest
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def ref():
    from oracle import vl_hog_api_ref
    vl_hog_api_ref.build()
    if not os.path.exists(vl_hog_api_ref.DRIVER):
        pytest.skip("oracle/_ref/vl_hog_driver_ref (the driver built against the reference's hog.c) is not built")
    return vl_hog_api_ref


@pytest.fixture(scope="module")
def shell_driver(tmp_path_factory):
    from superviseddescent_b200 import build
    lib = build.build()
    out = str(tmp_path_factory.mktemp("cpp") / "vl_hog_driver_shell")
    cmd = ["g++", "-std=c++14", "-O2", "-Wall", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "superviseddescent_b200", "include"),
           os.path.join(ROOT, "oracle", "vl_hog_driver.cpp"), "-L", os.path.dirname(lib), "-lsd_b200",
           f"-Wl,-rpath,{os.path.dirname(lib)}", "-lpthread", "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return out


def _run(binary, path, *args):
    r = subprocess.run([binary, str(path)] + list(args), capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    return path.read_bytes()


def _records(raw):
    out, pos = [], 0
    while pos < len(raw):
        n = int(np.frombuffer(raw, np.int32, 1, pos)[0])
        ints = np.frombuffer(raw, np.int32, n, pos + 4).tolist()
        pos += 4 + 4 * n
        m = int(np.frombuffer(raw, np.int64, 1, pos)[0])
        data = np.frombuffer(raw, np.float32, m, pos + 8)
        pos += 8 + 4 * m
        out.append((ints, data))
    return out


@pytest.fixture(scope="module")
def dumps(sd, ref, shell_driver, tmp_path_factory):
    d = tmp_path_factory.mktemp("dumps")
    return {"ref": _run(ref.DRIVER, d / "ref.bin"), "shell": _run(shell_driver, d / "shell.bin"),
            "threads": _run(shell_driver, d / "threads.bin", "threads")}


def _values(seed, n, scale, shift):
    """vl_hog_driver_value of oracle/vl_hog_driver.cpp: one LCG step of seed * 0x9E3779B97F4A7C15 + i, top 24 bits."""
    x = np.full(n, seed, np.uint64) * np.uint64(0x9E3779B97F4A7C15) + np.arange(n, dtype=np.uint64)
    x = x * np.uint64(6364136223846793005) + np.uint64(1442695040888963407)
    u = (x >> np.uint64(40)).astype(np.float32) * np.float32(1.0 / 16777216.0)
    return u * np.float32(scale) + np.float32(shift)


def test_drop_in_matches_hog_c(dumps):
    got, want = _records(dumps["shell"]), _records(dumps["ref"])
    assert len(got) == len(want) == 49
    worst = {1: 0.0, 2: 0.0}
    for (gi, gd), (wi, wd) in zip(got, want):
        assert gi == wi                                   # parameters, dims, dimension, glyph size, permutation
        assert gd.shape == wd.shape
        assert np.array_equal(np.isnan(gd), np.isnan(wd)), gi[:12]
        ok = ~np.isnan(wd)
        e = rel_err(gd[ok], wd[ok]) if ok.any() else 0.0
        worst[gi[0]] = max(worst[gi[0]], e)
        assert e <= 1e-4, (gi[:12], e)
    print(f"worst rel_err against hog.c: features {worst[1]:.2e}, renders {worst[2]:.2e}")


def test_four_threads_write_the_single_thread_dump(dumps):
    assert dumps["threads"] == dumps["shell"]


def test_put_is_the_batched_dense_hog_bit_for_bit(sd, dumps):
    dev = "cuda"
    checked = 0
    for ints, data in _records(dumps["shell"]):
        if ints[0] != 1:
            continue
        _, polar, seed, W, H, C, cs, K, variant, bil, tr, directed, w, h, dd = ints[:15]
        if polar:
            mod = torch.from_numpy(_values(seed, W * H, 4.0, -0.5).reshape(1, H, W)).to(dev)
            ang = torch.from_numpy(_values(seed + 1000, W * H, 20.0, -10.0).reshape(1, H, W)).to(dev)
            if tr:          # the buffer is column-major: the image is its transpose, read in place
                mod, ang = mod.transpose(1, 2), ang.transpose(1, 2)
            f = sd.vl_hog_polar(mod, ang, cs, K, variant, directed=bool(directed), bilinear_orientations=bool(bil))[0]
        else:
            buf = torch.from_numpy(_values(seed, W * H * C, 255.0, 0.0).reshape(1, C, H, W)).to(dev)
            f = sd.vl_hog(buf.transpose(2, 3) if tr else buf, cs, K, variant, bilinear_orientations=bool(bil))[0]
        if tr:
            f = f.transpose(1, 2)
        assert tuple(f.shape) == (dd, h, w)
        assert np.array_equal(f.contiguous().cpu().numpy().ravel().view(np.uint32), data.view(np.uint32)), ints[:12]
        checked += 1
    assert checked == 31
