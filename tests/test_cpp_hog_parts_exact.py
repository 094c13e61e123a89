"""The C++14 shell's star-model detector with the exact transform: rcr::vl_hog_part_detect of a model with unbounded = true
(tests/cpp/test_hog_parts_exact.cpp).

CPU: the translation unit compiles.  GPU: on grey and colour frames of different sizes (row steps wider than the pixels) the
shell returns, frame by frame, the Python vl_hog_part_detect result of the same model with max_displacement=None bit for bit:
every box, score, component, level and cell, and every part's placement, score and box; w0 = 0 throws."""
import os
import subprocess

import numpy as np
import pytest
import torch

import synth
from colour_examples import bgr_with_gray

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def exact_binary(tmp_path_factory):
    from superviseddescent_b200 import build
    lib = build.build()
    out = str(tmp_path_factory.mktemp("cpp") / "test_hog_parts_exact")
    cmd = ["g++", "-std=c++14", "-O1", "-Wall", "-Werror=return-type", "-I", os.path.join(ROOT, "include"),
           "-I", os.path.join(ROOT, "superviseddescent_b200", "include"), os.path.join(ROOT, "tests", "cpp", "test_hog_parts_exact.cpp"),
           "-L", os.path.dirname(lib), "-lsd_b200", f"-Wl,-rpath,{os.path.dirname(lib)}", "-lpthread", "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return out


def test_hog_parts_exact_shell_compiles_as_cxx14(exact_binary):
    assert os.path.exists(exact_binary)


@pytest.mark.gpu
@pytest.mark.parametrize("cs,K,variant,R,thr,overlap,mc,md", [(8, 9, 1, 3, -0.5, 0.5, 500, 20), (4, 4, 0, 0, -1.0, 0.3, 4096, 64),
                                                               (8, 9, 1, 32, 0.0, 0.5, 300, 30)])
def test_exact_shell_matches_python(exact_binary, sd, tmp_path, cs, K, variant, R, thr, overlap, mc, md):
    rng = np.random.default_rng(cs * 10 + K + R)
    sizes = [(120, 160), (97, 131), (37, 29)]
    grey = [synth.smooth_images(1, h, w, seed=70 + i, sigma=1.0)[0] for i, (h, w) in enumerate(sizes)]
    frames = [grey[0], bgr_with_gray(grey[1], rng.integers(-40, 41, grey[1].shape), rng.integers(-40, 41, grey[1].shape)), grey[2]]
    scales = [1.0, 0.5, 0.7]
    dd = 3 * K + 4 if variant == 1 else 4 * K
    Q, P, fw, fh, pfw, pfh, pad, ppad = 2, 3, 4, 3, 3, 2, (1, 0), (0, 1)
    root = rng.normal(0, 0.3, (Q, dd, fh, fw)).astype(np.float32)
    bias = rng.normal(0, 0.3, Q).astype(np.float32)
    parts = rng.normal(0, 0.3, (Q, P, dd, pfh, pfw)).astype(np.float32)
    anchors = np.stack([rng.integers(-1, 2 * fw - pfw + 2, (Q, P)), rng.integers(-1, 2 * fh - pfh + 2, (Q, P))], -1).astype(np.int32)
    deformation = np.stack([rng.uniform(0.001, 0.2, (Q, P)), rng.normal(0, 0.3, (Q, P)), rng.uniform(0.001, 0.2, (Q, P)),
                            rng.normal(0, 0.1, (Q, P))], -1).astype(np.float32)
    blob = [np.int32(len(frames)).tobytes()]
    for f in frames:
        ch = 1 if f.ndim == 2 else 3
        blob += [np.array([f.shape[1], f.shape[0], ch], dtype=np.int32).tobytes(), np.ascontiguousarray(f).tobytes()]
    blob += [np.int32(len(scales)).tobytes(), np.array(scales, dtype=np.float64).tobytes(),
             np.array([Q, P, fw, fh, pfw, pfh, pad[0], pad[1], ppad[0], ppad[1], R], dtype=np.int32).tobytes(),
             root.tobytes(), bias.tobytes(), parts.tobytes(), anchors.tobytes(), deformation.tobytes()]
    (tmp_path / "in.bin").write_bytes(b"".join(blob))
    r = subprocess.run([exact_binary, str(tmp_path / "in.bin"), str(tmp_path / "out.bin"), str(cs), str(K), str(variant), repr(thr),
                        repr(overlap), str(mc), str(md)], capture_output=True, text=True, timeout=300)
    print(r.stdout[-3000:])
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
    raw = np.frombuffer((tmp_path / "out.bin").read_bytes(), dtype=np.int32)
    model = sd.HogPartModel(root, bias, parts, anchors, deformation, pad, ppad, None)   # R travels to the shell and is ignored
    d = sd.vl_hog_part_detect(frames, scales, model, cs, K, thr, variant=variant, overlap=overlap, max_candidates=mc,
                              max_detections=md)
    pos, total = 0, 0
    for i in range(len(frames)):
        n = int(raw[pos])
        got = raw[pos + 1:pos + 1 + (9 + 7 * P) * n].reshape(n, 9 + 7 * P)
        pos += 1 + (9 + 7 * P) * n
        mine = d.frame == i
        ref = np.concatenate([d.boxes[mine], d.scores[mine].view(np.int32)[:, None], d.filter[mine][:, None], d.level[mine][:, None],
                              d.cell[mine], np.concatenate([d.placement[mine], d.part_scores[mine].view(np.int32)[..., None],
                                                            d.parts[mine]], axis=2).reshape(-1, 7 * P)], axis=1)
        assert np.array_equal(got, ref), i
        total += n
    assert pos == raw.size and total > 0
    print(f"{total} detections over {len(frames)} frames, above {d.above.tolist()}")
