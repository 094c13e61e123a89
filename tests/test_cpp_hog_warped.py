"""Warped samples in the C++14 shells (tests/cpp/test_hog_warped.cpp).

CPU: the translation unit compiles as C++14.  GPU: training and testing through rcr::HogTransform's `warps` on shallow copies of
photos equal the same on the virtual frames materialised by cv2, on the device and the host route; rcr::detection_model::detect
with warps equals detect on those frames; and the shell's warped detect, rcr::rotation_warp, rcr::invert_warp and
rcr::warp_landmarks equal the Python API's bit for bit."""
import os
import subprocess

import numpy as np
import pytest

import sample_warp_ref as SW

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ROT = [(0, 0, 0, 1), (320.5, 240.25, 30, 1), (-17, 1000, -45, 1.7), (61.5, 40.25, 180, 0.25), (100, 80, 721, 4)]


@pytest.fixture(scope="module")
def warped_binary(tmp_path_factory):
    from superviseddescent_b200 import build
    lib = build.build()
    out = str(tmp_path_factory.mktemp("cpp") / "test_hog_warped")
    cmd = ["g++", "-std=c++14", "-O1", "-Wall", "-Werror=return-type", "-I", os.path.join(ROOT, "include"),
           "-I", os.path.join(ROOT, "superviseddescent_b200", "include"), os.path.join(ROOT, "tests", "cpp", "test_hog_warped.cpp"),
           "-L", os.path.dirname(lib), "-lsd_b200", f"-Wl,-rpath,{os.path.dirname(lib)}", "-lpthread", "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return out


def test_hog_warped_compiles_as_cxx14(warped_binary):
    assert os.path.exists(warped_binary)


def _image(img):
    h, w = img.shape[:2]
    ch = 1 if img.ndim == 2 else img.shape[2]
    return np.array([h, w, ch], np.int32).tobytes() + np.ascontiguousarray(img, np.uint8).tobytes()


@pytest.mark.gpu
def test_shell_warps_equal_materialised_frames_and_python(warped_binary, golden, sd, tmp_path):
    import cv2
    import synth
    m = sd.load_detection_model(golden.model_path)
    mean = m.get_mean()
    rng = np.random.default_rng(12)
    photos = []
    for i in range(6):
        w, h = (151, 140) if i % 2 else (130, 127)
        g = synth.smooth_images(3 if i % 3 == 0 else 1, h, w, seed=60 + i)
        photos.append(np.ascontiguousarray(np.moveaxis(g, 0, -1)) if i % 3 == 0 else g[0])
    photo, warps, sizes, x_gt, x0, boxes = [], [], [], [], [], []
    for i, p in enumerate(photos):
        h, w = p.shape[:2]
        for k in range(5):
            M = sd.rotation_warp((w / 2 + rng.uniform(-4, 4), h / 2 + rng.uniform(-4, 4)), float(rng.uniform(-50, 50)), float(rng.uniform(0.9, 1.1)))
            box = (int(8 + i % 7), int(9 + i % 5), 100, 100)
            photo.append(i); warps.append(M); sizes.append((w + int(rng.integers(-6, 10)), h + int(rng.integers(-6, 10))))
            boxes.append(box)
            x_gt.append(sd.align_mean(mean, box))
            x0.append(sd.align_mean(mean, box, 1 + rng.normal(0, 0.03), 1 + rng.normal(0, 0.03), rng.normal(0, 0.03), rng.normal(0, 0.03)))
    n = len(photo)
    grey = [p if p.ndim == 2 else cv2.cvtColor(p, cv2.COLOR_BGR2GRAY) for p in photos]
    vs = [SW.materialise(grey[f], M, s) for f, M, s in zip(photo, warps, sizes)]
    rec = np.zeros(n, dtype=[("m", "<f8", (6,)), ("w", "<i4"), ("h", "<i4")])
    rec["m"] = np.stack(warps).reshape(n, 6)
    rec["w"], rec["h"] = np.array(sizes)[:, 0], np.array(sizes)[:, 1]
    blob = np.int32(len(photos)).tobytes() + b"".join(_image(p) for p in photos) + np.int32(n).tobytes()
    blob += np.array(photo, np.int32).tobytes() + rec.tobytes() + np.stack(x_gt).astype(np.float32).tobytes()
    blob += np.stack(x0).astype(np.float32).tobytes() + np.array(boxes, np.int32).tobytes() + b"".join(_image(v) for v in vs)
    (tmp_path / "in.bin").write_bytes(blob)
    r = subprocess.run([warped_binary, golden.model_path, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True,
                       text=True, timeout=600)
    print(r.stdout[-3000:])
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
    for line in ("TEST: 0.000e+00", "HOST TEST: 0.000e+00", "FUNCTOR: 0.000e+00", "DETECT: 0.000e+00"):
        assert "\n" + line in r.stdout, line
    out = (tmp_path / "out.bin").read_bytes()
    P = mean.size
    det = np.frombuffer(out, np.float32, n * P).reshape(n, P)
    o = n * P * 4
    rot = np.frombuffer(out, np.float64, 6 * len(ROT), o).reshape(-1, 2, 3)
    o += rot.nbytes
    inv = np.frombuffer(out, np.float64, 6 * n, o).reshape(n, 2, 3)
    o += inv.nbytes
    back = np.frombuffer(out, np.float32, n * P, o).reshape(n, P)
    want = m.detect_faces(photos, photo, boxes=np.array(boxes), warps=np.stack(warps), warp_sizes=np.array(sizes))
    assert np.array_equal(det.view(np.uint32), want.view(np.uint32))
    for got, (cx, cy, a, s) in zip(rot, ROT):
        assert np.array_equal(got, sd.rotation_warp((cx, cy), a, s))
    assert np.array_equal(inv, sd.invert_warp(np.stack(warps)))
    assert np.array_equal(back.view(np.uint32), sd.warp_landmarks(np.stack(x0).astype(np.float32), np.stack(warps)).view(np.uint32))
