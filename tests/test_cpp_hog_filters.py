"""The C++14 shell's HOG pyramid and filter scores, rcr::vl_hog_pyramid and rcr::vl_hog_correlate (tests/cpp/test_hog_filters.cpp).

CPU: the translation unit compiles.  GPU: on grey and colour frames of different sizes (row steps wider than the pixels) the
shell returns, level by level, the Python vl_hog_pyramid result bit for bit (an empty Mat for an empty level), and the scores of
a filter bank on every level bit for bit as vl_hog_correlate computes them, Q * oh rows of ow columns; refused configurations
throw."""
import os
import subprocess

import numpy as np
import pytest
import torch

import synth
from colour_examples import bgr_with_gray

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def filters_binary(tmp_path_factory):
    from superviseddescent_b200 import build
    lib = build.build()
    out = str(tmp_path_factory.mktemp("cpp") / "test_hog_filters")
    cmd = ["g++", "-std=c++14", "-O1", "-Wall", "-Werror=return-type", "-I", os.path.join(ROOT, "include"),
           "-I", os.path.join(ROOT, "superviseddescent_b200", "include"), os.path.join(ROOT, "tests", "cpp", "test_hog_filters.cpp"),
           "-L", os.path.dirname(lib), "-lsd_b200", f"-Wl,-rpath,{os.path.dirname(lib)}", "-lpthread", "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return out


def test_hog_filters_shell_compiles_as_cxx14(filters_binary):
    assert os.path.exists(filters_binary)


def _read(raw, pos):
    rows, cols = np.frombuffer(raw, dtype=np.int32, count=2, offset=pos)
    pos += 8
    m = np.frombuffer(raw, dtype=np.float32, count=rows * cols, offset=pos).reshape(rows, cols)
    return m, pos + 4 * rows * cols


@pytest.mark.gpu
@pytest.mark.parametrize("cs,K,variant,bias,pad", [(8, 9, 1, True, (0, 0)), (4, 4, 0, False, (2, 1))])
def test_shell_matches_python(filters_binary, sd, tmp_path, cs, K, variant, bias, pad):
    rng = np.random.default_rng(cs * 10 + K)
    sizes = [(120, 160), (97, 131), (37, 29)]
    grey = [synth.smooth_images(1, h, w, seed=80 + i)[0] for i, (h, w) in enumerate(sizes)]
    frames = [grey[0], bgr_with_gray(grey[1], rng.integers(-40, 41, grey[1].shape), rng.integers(-40, 41, grey[1].shape)), grey[2]]
    scales = [1.0, 0.5, 1.5, 2 ** -0.2, 0.05]
    dd = 3 * K + 4 if variant == 1 else 4 * K
    Q, fh, fw = 3, 4, 5
    filt = rng.normal(0, 1, (Q, dd, fh, fw)).astype(np.float32)
    b = rng.normal(0, 1, Q).astype(np.float32)
    blob = [np.int32(len(frames)).tobytes()]
    for f in frames:
        ch = 1 if f.ndim == 2 else 3
        blob += [np.array([f.shape[1], f.shape[0], ch], dtype=np.int32).tobytes(), np.ascontiguousarray(f).tobytes()]
    blob += [np.int32(len(scales)).tobytes(), np.array(scales, dtype=np.float64).tobytes(),
             np.array([Q, fw, fh], dtype=np.int32).tobytes(), filt.tobytes(), np.int32(int(bias)).tobytes()]
    if bias:
        blob.append(b.tobytes())
    (tmp_path / "in.bin").write_bytes(b"".join(blob))
    r = subprocess.run([filters_binary, str(tmp_path / "in.bin"), str(tmp_path / "out.bin"), str(cs), str(K), str(variant),
                        str(pad[0]), str(pad[1])], capture_output=True, text=True, timeout=300)
    print(r.stdout[-3000:])
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
    raw = (tmp_path / "out.bin").read_bytes()
    feats, _ = sd.vl_hog_pyramid(frames, scales, cs, K, variant)
    pos = 0
    for fr in feats:
        for w in fr:
            got, pos = _read(raw, pos)
            if w is None:
                assert got.size == 0
            else:
                w = w.cpu().numpy()
                assert got.shape == (w.shape[0] * w.shape[1], w.shape[2]) and np.array_equal(got, w.reshape(got.shape))
    ft = torch.from_numpy(filt).cuda()
    bt = torch.from_numpy(b).cuda() if bias else None
    n_scores = 0
    for fr in feats:
        maps = [w for w in fr if w is not None]
        for s in sd.vl_hog_correlate(maps, ft, K, variant, bias=bt, pad=pad):
            got, pos = _read(raw, pos)
            if s.numel() == 0:
                assert got.size == 0
            else:
                s = s.cpu().numpy()
                assert got.shape == (Q * s.shape[1], s.shape[2]) and np.array_equal(got, s.reshape(got.shape))
                n_scores += 1
    assert pos == len(raw) and n_scores > 0
