"""The C++14 shell's detect overloads for several faces per frame in frames of different sizes (tests/cpp/test_detect_frames.cpp).

CPU: the translation unit compiles.  GPU: on the reference's five example frames in colour plus a grey frame with two faces, in one
call, the shell gives the same landmarks as the Python mirror's detect_faces, bit for bit."""
import os
import subprocess

import numpy as np
import pytest

from colour_examples import examples_bgr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def frames_binary(tmp_path_factory):
    from superviseddescent_b200 import build
    lib = build.build()
    out = str(tmp_path_factory.mktemp("cpp") / "test_detect_frames")
    cmd = ["g++", "-std=c++14", "-O1", "-Wall", "-Werror=return-type", "-I", os.path.join(ROOT, "include"),
           "-I", os.path.join(ROOT, "superviseddescent_b200", "include"), os.path.join(ROOT, "tests", "cpp", "test_detect_frames.cpp"),
           "-L", os.path.dirname(lib), "-lsd_b200", f"-Wl,-rpath,{os.path.dirname(lib)}", "-lpthread", "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return out


def test_detect_frames_compiles_as_cxx14(frames_binary):
    assert os.path.exists(frames_binary)


@pytest.mark.gpu
def test_shell_detect_frames_matches_python(frames_binary, sd, golden, tmp_path):
    frames = examples_bgr(golden) + [golden.examples["gray1"]]
    boxes = [list(golden.examples["boxes"][i]) for i in range(5)]
    b1 = golden.examples["boxes"][1]
    boxes += [list(b1), [int(b1[0]) + 20, int(b1[1]) - 10, int(b1[2]), int(b1[3])]]
    face_frame = [3, 0, 5, 1, 4, 2, 5]
    boxes = [boxes[[3, 0, 5, 1, 4, 2, 6][i]] for i in range(7)]
    blob = [np.int32(len(frames)).tobytes()]
    for f in frames:
        ch = 1 if f.ndim == 2 else 3
        blob += [np.array([f.shape[1], f.shape[0], ch], dtype=np.int32).tobytes(), np.ascontiguousarray(f).tobytes()]
    blob.append(np.int32(len(face_frame)).tobytes())
    for i, b in zip(face_frame, boxes):
        blob.append(np.array([i] + list(b), dtype=np.int32).tobytes())
    (tmp_path / "in.bin").write_bytes(b"".join(blob))
    m = sd.load_detection_model(golden.model_path)
    r = subprocess.run([frames_binary, golden.model_path, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")],
                       capture_output=True, text=True, timeout=300)
    print(r.stdout[-3000:])
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
    got = np.fromfile(tmp_path / "out.bin", dtype=np.float32).reshape(len(face_frame), -1)
    want = m.detect_faces(frames, face_frame, boxes=np.array(boxes))
    assert np.array_equal(got, want)
