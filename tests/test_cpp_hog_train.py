"""The C++14 shell's HOG filter trainer, rcr::train_hog_filter (tests/cpp/test_hog_train.cpp).

CPU: the translation unit compiles.  GPU: on grey and colour frames (row steps wider than the pixels, one frame without a box)
the shell returns the Python train_hog_filter result bit for bit: the filter, the bias, every round's counts and solve report,
and the negative cache; refused arguments throw."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import hog_train_ref as T
from colour_examples import bgr_with_gray
from superviseddescent_b200._capi import HogTrainParamC, HogTrainReportC, HogWindowC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def train_binary(tmp_path_factory):
    from superviseddescent_b200 import build
    lib = build.build()
    out = str(tmp_path_factory.mktemp("cpp") / "test_hog_train")
    cmd = ["g++", "-std=c++14", "-O1", "-Wall", "-Werror=return-type", "-I", os.path.join(ROOT, "include"),
           "-I", os.path.join(ROOT, "superviseddescent_b200", "include"), os.path.join(ROOT, "tests", "cpp", "test_hog_train.cpp"),
           "-L", os.path.dirname(lib), "-lsd_b200", f"-Wl,-rpath,{os.path.dirname(lib)}", "-lpthread", "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return out


def test_hog_train_shell_compiles_as_cxx14(train_binary):
    assert os.path.exists(train_binary)


COUNTS = [f for f, _ in HogTrainReportC._fields_[:10] if f != "reserved"]


@pytest.mark.gpu
def test_shell_matches_python(train_binary, sd, tmp_path):
    rng = np.random.default_rng(8)
    grey, boxes = T.planted_frames(31, 6, 240, 180, sides=(48, 96))
    frames = [grey[0], bgr_with_gray(grey[1], rng.integers(-40, 41, grey[1].shape), rng.integers(-40, 41, grey[1].shape))] + list(grey[2:])
    box_frame = np.asarray([0, 1, 2, 3, 4], np.int32)             # frame 5 has no box: a pure negative frame
    boxes = boxes[:5]
    scales = T.detector_scales(240, 180, 8, 5)
    cs, K, variant, fw, fh, px, py = 8, 9, 1, 5, 5, 1, 0
    kw = dict(lam=0.02, positive_overlap=0.5, negative_overlap=0.3, flip_positives=True, rounds=2, negatives_per_frame=12,
              mine_overlap=0.5, max_negatives=50, max_iterations=40)
    prm = HogTrainParamC(kw["lam"], kw["positive_overlap"], kw["negative_overlap"], 1, kw["rounds"], kw["negatives_per_frame"],
                         kw["mine_overlap"], kw["max_negatives"], kw["max_iterations"])
    blob = [np.int32(len(frames)).tobytes()]
    for f in frames:
        ch = 1 if f.ndim == 2 else 3
        blob += [np.array([f.shape[1], f.shape[0], ch], np.int32).tobytes(), np.ascontiguousarray(f).tobytes()]
    blob += [np.int32(len(scales)).tobytes(), np.array(scales, np.float64).tobytes(), np.int32(len(boxes)).tobytes()]
    blob += [np.array([f, *b], np.int32).tobytes() for f, b in zip(box_frame, boxes)]
    blob += [np.array([cs, K, variant, fw, fh, px, py], np.int32).tobytes(), bytes(prm)]
    (tmp_path / "in.bin").write_bytes(b"".join(blob))
    r = subprocess.run([train_binary, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True, timeout=300)
    print(r.stdout[-3000:])
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
    raw = (tmp_path / "out.bin").read_bytes()
    dd = 3 * K + 4
    nf = dd * fh * fw
    filt = np.frombuffer(raw[:4 * nf], np.float32)
    bias = np.frombuffer(raw[4 * nf:4 * nf + 4], np.float32)[0]
    pos = 4 * nf + 4
    nr = int(np.frombuffer(raw[pos:pos + 4], np.int32)[0])
    pos += 4
    sz = C.sizeof(HogTrainReportC)
    reps = [HogTrainReportC.from_buffer_copy(raw[pos + k * sz:pos + (k + 1) * sz]) for k in range(nr)]
    pos += nr * sz
    nn = int(np.frombuffer(raw[pos:pos + 4], np.int32)[0])
    pos += 4
    negs = [HogWindowC.from_buffer_copy(raw[pos + k * 16:pos + (k + 1) * 16]) for k in range(nn)]
    assert pos + 16 * nn == len(raw)

    hf = sd.train_hog_filter(frames, box_frame, boxes, scales, (fw, fh), cs, K, variant, pad=(px, py), **kw)
    assert np.array_equal(filt.view(np.uint32), hf.filter.cpu().numpy().ravel().view(np.uint32))
    assert np.float32(bias).view(np.uint32) == np.float32(hf.bias).view(np.uint32)
    assert nr == len(hf.report)
    for c, p in zip(reps, hf.report):
        assert {f: int(getattr(c, f)) for f in COUNTS} == {f: p[f] for f in COUNTS}
        assert (sd._svm_report(c.solve) if c.solved else None) == p["solve"]
    S = len(scales)
    assert np.array_equal(np.asarray([(w.grid // S, w.grid % S, w.x, w.y) for w in negs], np.int32).reshape(-1, 4), hf.negatives)
    print(f"{nn} negatives, rounds {[{f: p[f] for f in COUNTS} for p in hf.report]}")
