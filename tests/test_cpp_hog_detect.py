"""The C++14 shell's sliding-window detector, rcr::vl_hog_detect (tests/cpp/test_hog_detect.cpp).

CPU: the translation unit compiles.  GPU: on grey and colour frames of different sizes (row steps wider than the pixels) the
shell returns, frame by frame, the Python vl_hog_detect result bit for bit: every box, score, filter, level and cell; refused
arguments throw."""
import os
import subprocess

import numpy as np
import pytest
import torch

import synth
from colour_examples import bgr_with_gray

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def detect_binary(tmp_path_factory):
    from superviseddescent_b200 import build
    lib = build.build()
    out = str(tmp_path_factory.mktemp("cpp") / "test_hog_detect")
    cmd = ["g++", "-std=c++14", "-O1", "-Wall", "-Werror=return-type", "-I", os.path.join(ROOT, "include"),
           "-I", os.path.join(ROOT, "superviseddescent_b200", "include"), os.path.join(ROOT, "tests", "cpp", "test_hog_detect.cpp"),
           "-L", os.path.dirname(lib), "-lsd_b200", f"-Wl,-rpath,{os.path.dirname(lib)}", "-lpthread", "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return out


def test_hog_detect_shell_compiles_as_cxx14(detect_binary):
    assert os.path.exists(detect_binary)


@pytest.mark.gpu
@pytest.mark.parametrize("cs,K,variant,bias,pad,thr,overlap,mc,md", [(8, 9, 1, True, (0, 0), 0.0, 0.5, 500, 20),
                                                                     (4, 4, 0, False, (2, 1), -0.5, 0.3, 4096, 64)])
def test_shell_matches_python(detect_binary, sd, tmp_path, cs, K, variant, bias, pad, thr, overlap, mc, md):
    rng = np.random.default_rng(cs * 10 + K)
    sizes = [(120, 160), (97, 131), (37, 29)]
    grey = [synth.smooth_images(1, h, w, seed=90 + i)[0] for i, (h, w) in enumerate(sizes)]
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
    r = subprocess.run([detect_binary, str(tmp_path / "in.bin"), str(tmp_path / "out.bin"), str(cs), str(K), str(variant),
                        str(pad[0]), str(pad[1]), repr(thr), repr(overlap), str(mc), str(md)], capture_output=True, text=True,
                       timeout=300)
    print(r.stdout[-3000:])
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
    raw = np.frombuffer((tmp_path / "out.bin").read_bytes(), dtype=np.int32)
    d = sd.vl_hog_detect(frames, scales, torch.from_numpy(filt), cs, K, thr, variant=variant,
                         bias=torch.from_numpy(b) if bias else None, pad=pad, overlap=overlap, max_candidates=mc, max_detections=md)
    pos, total = 0, 0
    for i in range(len(frames)):
        n = int(raw[pos])
        got = raw[pos + 1:pos + 1 + 9 * n].reshape(n, 9)
        pos += 1 + 9 * n
        mine = d.frame == i
        ref = np.concatenate([d.boxes[mine], d.scores[mine].view(np.int32)[:, None], d.filter[mine][:, None], d.level[mine][:, None],
                              d.cell[mine]], axis=1)
        assert np.array_equal(got, ref), i
        total += n
    assert pos == raw.size and total > 0
    print(f"{total} detections over {len(frames)} frames, above {d.above.tolist()}")
