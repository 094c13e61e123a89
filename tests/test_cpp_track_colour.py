"""The C++14 shell's tracking steps and box scores on colour and float frames: rcr::detection_model::track and
track_and_detect and rcr::hog_box_scores with multichannel, bilinear_orientations, float_frames and grey_images
(tests/cpp/test_track_colour.cpp).

CPU: the translation unit compiles.  GPU: on the colour golden frames of different sizes plus a noise frame (8-bit B,G,R with
nearest and bilinear bins, and the same frames as float with their grey passed as grey_images), with tracks on faces, a
duplicated track and a listed subset of frames, every output of the shell is the Python front end's bit for bit, and refused
arguments throw."""
import os
import subprocess

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODEL = os.path.join(ROOT, "tests", "golden", "face_landmarks_model_rcr_22.bin")
SCALES = [2.0 ** (-k / 4) for k in range(2, 14)]


@pytest.fixture(scope="module")
def binary(tmp_path_factory):
    from superviseddescent_b200 import build
    lib = build.build()
    out = str(tmp_path_factory.mktemp("cpp") / "test_track_colour")
    cmd = ["g++", "-std=c++14", "-O1", "-Wall", "-Werror=return-type", "-I", os.path.join(ROOT, "include"),
           "-I", os.path.join(ROOT, "superviseddescent_b200", "include"), os.path.join(ROOT, "tests", "cpp", "test_track_colour.cpp"),
           "-L", os.path.dirname(lib), "-lsd_b200", f"-Wl,-rpath,{os.path.dirname(lib)}", "-lpthread", "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return out


def test_track_colour_shell_compiles_as_cxx14(binary):
    assert os.path.exists(binary)


def _rows(raw, o, R, P):
    lm = np.frombuffer(raw, np.float32, R * P, o).reshape(R, P)
    o += 4 * R * P
    bx = np.frombuffer(raw, np.int32, 4 * R, o).reshape(R, 4)
    o += 16 * R
    sc = np.frombuffer(raw, np.uint32, R, o)
    alive = np.frombuffer(raw, np.int32, R, o + 4 * R).astype(bool)
    return (lm, bx, sc, alive), o + 8 * R


def _check(got, want):
    lm, bx, sc, alive = got
    assert np.array_equal(lm, want.landmarks.cpu().numpy())
    assert np.array_equal(bx, want.boxes.cpu().numpy())
    assert np.array_equal(sc, want.scores.cpu().numpy().view(np.uint32))
    assert np.array_equal(alive, want.alive.cpu().numpy())


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["colour", "colour_bilinear", "float"])
def test_shell_matches_python(binary, sd, golden, tmp_path, kind):
    import synth
    from colour_examples import examples_bgr
    m = sd.load_detection_model(golden.model_path)
    grey = [golden.examples[f"gray{i}"] for i in range(5)]
    noise = synth.smooth_images(1, 360, 480, seed=7)[0]
    grey = grey + [noise]
    colour = examples_bgr(golden) + [np.ascontiguousarray(np.repeat(noise[..., None], 3, axis=2))]
    fl = kind == "float"
    bil = kind == "colour_bilinear"
    frames = [c.astype(np.float32) / np.float32(255) for c in colour] if fl else colour
    prev = m.detect_faces(grey[:5], np.arange(5), boxes=golden.examples["boxes"])
    prev = np.concatenate([prev, prev[[2]]]).astype(np.float32)
    face = np.array([0, 1, 2, 3, 4, 2], np.int32)
    cs, K, fw, fh = 8, 9, 6, 6
    rng = np.random.default_rng(len(kind))
    filt = rng.normal(0, 0.1, (3 * K + 4, fh, fw)).astype(np.float32)
    bias = np.float32(rng.normal(0, 0.5))
    listed = np.array([5, 1, 3], np.int32)
    threshold, det_threshold, t_ov, max_det = 0.0, -1.0, 0.5, 4
    blob = [np.array([int(fl), len(frames)], np.int32).tobytes()]
    for f in frames:
        blob += [np.array([f.shape[1], f.shape[0], 3], dtype=np.int32).tobytes(), np.ascontiguousarray(f).tobytes()]
    if fl:
        blob += [np.ascontiguousarray(g).tobytes() for g in grey]
    blob += [np.int32(len(face)).tobytes(), face.tobytes(), prev.tobytes(), np.array([fw, fh], np.int32).tobytes(), filt.tobytes(),
             bias.tobytes(), np.int32(len(SCALES)).tobytes(), np.array(SCALES, np.float64).tobytes(), np.int32(len(listed)).tobytes(),
             listed.tobytes()]
    (tmp_path / "in.bin").write_bytes(b"".join(blob))
    r = subprocess.run([binary, MODEL, str(tmp_path / "in.bin"), str(tmp_path / "out.bin"), str(cs), str(K), repr(threshold),
                        repr(det_threshold), repr(t_ov), str(max_det), str(int(bil))], capture_output=True, text=True, timeout=300)
    print(r.stdout[-3000:])
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
    raw = (tmp_path / "out.bin").read_bytes()
    P, T = prev.shape[1], len(face)
    kw = dict(multichannel=True, bilinear_orientations=bil, float_frames=fl)
    gk = dict(grey_frames=grey) if fl else {}
    ff = (torch.from_numpy(filt), float(bias))
    tracked, o = _rows(raw, 0, T, P)
    want_t = m.track_faces(frames, face, prev, ff, (fw, fh), cs, K, threshold, **kw, **gk)
    _check(tracked, want_t)
    sc = np.frombuffer(raw, np.uint32, T, o)
    o += 4 * T
    assert np.array_equal(sc, sd.hog_box_scores(frames, face, want_t.boxes, filt, float(bias), cs, K, **kw).cpu().numpy().view(np.uint32))
    R = int(np.frombuffer(raw, np.int32, 1, o)[0])
    got, o = _rows(raw, o + 4, R, P)
    fr = np.frombuffer(raw, np.int32, R, o)
    assert len(raw) == o + 4 * R
    want = m.track_and_detect(frames, face, prev, ff, (fw, fh), cs, K, threshold, SCALES, listed, det_threshold, track_overlap=t_ov,
                              max_detections=max_det, **kw, **gk)
    assert R == T + want.num_new and want.num_new > 0
    _check(got, want)
    assert np.array_equal(fr, want.frame.cpu().numpy())
