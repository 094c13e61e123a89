"""The C++14 shell's aligned face chips: rcr::face_chips (tests/cpp/test_face_chips.cpp).

CPU: the translation unit compiles.  GPU: on B,G,R and float frames of different sizes, with faces rotated about their boxes,
one of them invalid (NaN landmarks), the chips, both transforms and valid are the Python front end's bit for bit (face_chips
with face_chip_template), for all landmarks and for a list of landmark ids; refused arguments throw."""
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODEL = os.path.join(ROOT, "tests", "golden", "face_landmarks_model_rcr_22.bin")


@pytest.fixture(scope="module")
def binary(tmp_path_factory):
    from superviseddescent_b200 import build
    lib = build.build()
    out = str(tmp_path_factory.mktemp("cpp") / "test_face_chips")
    cmd = ["g++", "-std=c++14", "-O1", "-Wall", "-Werror=return-type", "-I", os.path.join(ROOT, "include"),
           "-I", os.path.join(ROOT, "superviseddescent_b200", "include"), os.path.join(ROOT, "tests", "cpp", "test_face_chips.cpp"),
           "-L", os.path.dirname(lib), "-lsd_b200", f"-Wl,-rpath,{os.path.dirname(lib)}", "-lpthread", "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return out


def test_face_chips_shell_compiles_as_cxx14(binary):
    assert os.path.exists(binary)


@pytest.mark.gpu
@pytest.mark.parametrize("fl,ids", [(False, None), (True, None), (False, ["37", "40", "43", "46", "31", "49", "55"])])
def test_shell_matches_python(binary, sd, golden, tmp_path, fl, ids):
    import synth
    from colour_examples import examples_bgr
    m = sd.load_detection_model(golden.model_path)
    L = m.num_landmarks
    colour = examples_bgr(golden)[:3]
    frames = [c.astype(np.float32) / np.float32(255) for c in colour] if fl else colour
    rng = np.random.default_rng(int(fl))
    mean = m.get_mean().astype(np.float32).ravel()
    face, rows = [], []
    for f, fr in enumerate(frames):
        H, W = fr.shape[:2]
        for _ in range(3):
            s = float(rng.uniform(40, min(H, W) / 2))
            cx, cy, t = rng.uniform(0, W), rng.uniform(0, H), rng.uniform(-np.pi, np.pi)
            dx, dy = mean[:L] * s, mean[L:] * s
            rows.append(np.concatenate([cx + np.cos(t) * dx - np.sin(t) * dy, cy + np.sin(t) * dx + np.cos(t) * dy]).astype(np.float32))
            face.append(f)
    x = np.stack(rows)
    x[4] = np.nan                                  # invalid whichever landmarks are used
    face = np.array(face, np.int32)
    cw, ch, padding = 56, 64, 0.2
    blob = [np.array([int(fl), len(frames)], np.int32).tobytes()]
    for f in frames:
        blob += [np.array([f.shape[1], f.shape[0], 3], dtype=np.int32).tobytes(), np.ascontiguousarray(f).tobytes()]
    blob += [np.int32(len(face)).tobytes(), face.tobytes(), x.tobytes()]
    (tmp_path / "in.bin").write_bytes(b"".join(blob))
    r = subprocess.run([binary, MODEL, str(tmp_path / "in.bin"), str(tmp_path / "out.bin"), str(cw), str(ch), repr(padding)] + (ids or []),
                       capture_output=True, text=True, timeout=300)
    print(r.stdout[-3000:])
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
    idx = None
    if ids is not None:
        from superviseddescent_b200 import _capi
        names = [_capi.lib().sd_model_landmark_id(m._m, k).decode() for k in range(L)]
        idx = [names.index(i) for i in ids]
    tm = sd.face_chip_template(m, (cw, ch), padding, idx)
    want = sd.face_chips(frames, face, x, (cw, ch), tm, idx, channels_last=True)
    raw = (tmp_path / "out.bin").read_bytes()
    n, es = len(face), 4 if fl else 1
    o = n * ch * cw * 3 * es
    chips = np.frombuffer(raw, np.uint8, o, 0)
    assert np.array_equal(chips, want.chips.cpu().numpy().view(np.uint8).ravel())
    c2f = np.frombuffer(raw, np.float64, 6 * n, o)
    f2c = np.frombuffer(raw, np.float64, 6 * n, o + 48 * n)
    valid = np.frombuffer(raw, np.int32, n, o + 96 * n).astype(bool)
    assert len(raw) == o + 100 * n
    assert np.array_equal(c2f.view(np.uint64), want.chip_to_frame.cpu().numpy().ravel().view(np.uint64))
    assert np.array_equal(f2c.view(np.uint64), want.frame_to_chip.cpu().numpy().ravel().view(np.uint64))
    assert np.array_equal(valid, want.valid.cpu().numpy())
    assert not valid[4] and valid.sum() == n - 1
