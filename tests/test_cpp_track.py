"""The C++14 shell's tracking step, rcr::detection_model::track, and rcr::hog_box_scores (tests/cpp/test_track.cpp).

CPU: the translation unit compiles.  GPU: on grey and colour golden frames of different sizes (row steps wider than the pixels)
the shell's step returns the Python track_faces result bit for bit -- landmarks, boxes, scores and alive flags, a dying track
included -- and its box scores are hog_box_scores'; refused arguments throw."""
import os
import subprocess

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODEL = os.path.join(ROOT, "tests", "golden", "face_landmarks_model_rcr_22.bin")


@pytest.fixture(scope="module")
def track_binary(tmp_path_factory):
    from superviseddescent_b200 import build
    lib = build.build()
    out = str(tmp_path_factory.mktemp("cpp") / "test_track")
    cmd = ["g++", "-std=c++14", "-O1", "-Wall", "-Werror=return-type", "-I", os.path.join(ROOT, "include"),
           "-I", os.path.join(ROOT, "superviseddescent_b200", "include"), os.path.join(ROOT, "tests", "cpp", "test_track.cpp"),
           "-L", os.path.dirname(lib), "-lsd_b200", f"-Wl,-rpath,{os.path.dirname(lib)}", "-lpthread", "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return out


def test_track_shell_compiles_as_cxx14(track_binary):
    assert os.path.exists(track_binary)


@pytest.mark.gpu
@pytest.mark.parametrize("colour", [False, True])
def test_shell_matches_python(track_binary, sd, golden, tmp_path, colour):
    from colour_examples import examples_bgr
    m = sd.load_detection_model(golden.model_path)
    grey = [golden.examples[f"gray{i}"] for i in range(5)]
    frames = examples_bgr(golden) if colour else grey
    prev = m.detect_faces(grey, np.arange(5), boxes=golden.examples["boxes"])
    prev = np.concatenate([prev, np.full((1, prev.shape[1]), 50.0, np.float32), prev[[2]] + np.float32(3)])   # one collapsed track
    face = np.array([0, 1, 2, 3, 4, 1, 2], np.int32)
    cs, K, fw, fh = 8, 9, 6, 6
    rng = np.random.default_rng(int(colour))
    filt = rng.normal(0, 0.1, (3 * K + 4, fh, fw)).astype(np.float32)
    bias = np.float32(rng.normal(0, 0.5))
    threshold = 0.0
    box_frame = np.array([0, 1, 3, 4, 4], np.int32)
    boxes = np.array([[91, 157, 209, 209], [-30, 20, 100, 90], [600, 900, 200, 200], [5, 5, 40, 60], [2000, 0, 50, 50]], np.int32)
    blob = [np.int32(len(frames)).tobytes()]
    for f in frames:
        ch = 1 if f.ndim == 2 else 3
        blob += [np.array([f.shape[1], f.shape[0], ch], dtype=np.int32).tobytes(), np.ascontiguousarray(f).tobytes()]
    blob += [np.int32(len(face)).tobytes(), face.tobytes(), prev.astype(np.float32).tobytes(), np.array([fw, fh], np.int32).tobytes(),
             filt.tobytes(), bias.tobytes(), np.int32(len(box_frame)).tobytes(), box_frame.tobytes(), boxes.tobytes()]
    (tmp_path / "in.bin").write_bytes(b"".join(blob))
    r = subprocess.run([track_binary, MODEL, str(tmp_path / "in.bin"), str(tmp_path / "out.bin"), str(cs), str(K), "1", repr(threshold)],
                       capture_output=True, text=True, timeout=300)
    print(r.stdout[-3000:])
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
    raw = (tmp_path / "out.bin").read_bytes()
    T, P, n = len(face), prev.shape[1], len(box_frame)
    lm = np.frombuffer(raw, np.float32, T * P, 0).reshape(T, P)
    bx = np.frombuffer(raw, np.int32, 4 * T, 4 * T * P).reshape(T, 4)
    sc = np.frombuffer(raw, np.uint32, T, 4 * T * (P + 4))
    alive = np.frombuffer(raw, np.int32, T, 4 * T * (P + 5))
    bsc = np.frombuffer(raw, np.uint32, n, 4 * T * (P + 6))
    assert len(raw) == 4 * (T * (P + 6) + n)
    want = m.track_faces(frames, face, prev, (torch.from_numpy(filt), float(bias)), (fw, fh), cs, K, threshold)
    assert np.array_equal(lm, want.landmarks.cpu().numpy())
    alive_want = want.alive.cpu().numpy()
    assert np.array_equal(alive.astype(bool), alive_want) and not alive_want[5]
    ok = np.arange(T) != 5                                                  # the collapsed track's box and score are unspecified
    assert np.array_equal(bx[ok], want.boxes.cpu().numpy()[ok])
    assert np.array_equal(sc[ok], want.scores.cpu().numpy().view(np.uint32)[ok])
    got = sd.hog_box_scores(frames, box_frame, boxes, torch.from_numpy(filt), float(bias), cs, K).cpu().numpy()
    assert np.array_equal(bsc, got.view(np.uint32))
