"""The C++14 shell's tracking step with the detector inside it, rcr::detection_model::track_and_detect
(tests/cpp/test_track_detect.cpp).

CPU: the translation unit compiles.  GPU: on grey and colour golden frames of different sizes plus a noise frame, with tracks on
faces, a duplicated track and a listed subset of frames, the shell's rows are the Python track_and_detect rows bit for bit --
landmarks, boxes, scores, alive flags and frames -- and refused arguments throw."""
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
    out = str(tmp_path_factory.mktemp("cpp") / "test_track_detect")
    cmd = ["g++", "-std=c++14", "-O1", "-Wall", "-Werror=return-type", "-I", os.path.join(ROOT, "include"),
           "-I", os.path.join(ROOT, "superviseddescent_b200", "include"), os.path.join(ROOT, "tests", "cpp", "test_track_detect.cpp"),
           "-L", os.path.dirname(lib), "-lsd_b200", f"-Wl,-rpath,{os.path.dirname(lib)}", "-lpthread", "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return out


def test_track_detect_shell_compiles_as_cxx14(binary):
    assert os.path.exists(binary)


@pytest.mark.gpu
@pytest.mark.parametrize("colour", [False, True])
def test_shell_matches_python(binary, sd, golden, tmp_path, colour):
    import synth
    from colour_examples import examples_bgr
    m = sd.load_detection_model(golden.model_path)
    grey = [golden.examples[f"gray{i}"] for i in range(5)]
    frames = (examples_bgr(golden) if colour else grey) + [synth.smooth_images(1, 360, 480, seed=7)[0]]
    prev = m.detect_faces(grey, np.arange(5), boxes=golden.examples["boxes"])
    prev = np.concatenate([prev, prev[[2]]]).astype(np.float32)
    face = np.array([0, 1, 2, 3, 4, 2], np.int32)
    cs, K, fw, fh = 8, 9, 6, 6
    rng = np.random.default_rng(int(colour))
    filt = rng.normal(0, 0.1, (3 * K + 4, fh, fw)).astype(np.float32)
    bias = np.float32(rng.normal(0, 0.5))
    listed = np.array([5, 1, 3], np.int32)
    threshold, det_threshold, t_ov, max_det = 0.0, -1.0, 0.5, 4
    blob = [np.int32(len(frames)).tobytes()]
    for f in frames:
        ch = 1 if f.ndim == 2 else 3
        blob += [np.array([f.shape[1], f.shape[0], ch], dtype=np.int32).tobytes(), np.ascontiguousarray(f).tobytes()]
    blob += [np.int32(len(face)).tobytes(), face.tobytes(), prev.tobytes(), np.array([fw, fh], np.int32).tobytes(), filt.tobytes(),
             bias.tobytes(), np.int32(len(SCALES)).tobytes(), np.array(SCALES, np.float64).tobytes(), np.int32(len(listed)).tobytes(),
             listed.tobytes()]
    (tmp_path / "in.bin").write_bytes(b"".join(blob))
    r = subprocess.run([binary, MODEL, str(tmp_path / "in.bin"), str(tmp_path / "out.bin"), str(cs), str(K), repr(threshold),
                        repr(det_threshold), repr(t_ov), str(max_det)], capture_output=True, text=True, timeout=300)
    print(r.stdout[-3000:])
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
    raw = (tmp_path / "out.bin").read_bytes()
    R = int(np.frombuffer(raw, np.int32, 1)[0])
    P = prev.shape[1]
    o = 4
    lm = np.frombuffer(raw, np.float32, R * P, o).reshape(R, P)
    o += 4 * R * P
    bx = np.frombuffer(raw, np.int32, 4 * R, o).reshape(R, 4)
    o += 16 * R
    sc = np.frombuffer(raw, np.uint32, R, o)
    alive = np.frombuffer(raw, np.int32, R, o + 4 * R)
    fr = np.frombuffer(raw, np.int32, R, o + 8 * R)
    assert len(raw) == o + 12 * R
    want = m.track_and_detect(frames, face, prev, (torch.from_numpy(filt), float(bias)), (fw, fh), cs, K, threshold, SCALES, listed,
                              det_threshold, track_overlap=t_ov, max_detections=max_det)
    assert R == len(face) + want.num_new and want.num_new > 0
    assert np.array_equal(lm, want.landmarks.cpu().numpy())
    assert np.array_equal(bx, want.boxes.cpu().numpy())
    assert np.array_equal(sc, want.scores.cpu().numpy().view(np.uint32))
    assert np.array_equal(alive.astype(bool), want.alive.cpu().numpy())
    assert np.array_equal(fr, want.frame.cpu().numpy())
