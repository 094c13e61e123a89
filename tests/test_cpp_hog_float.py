"""The C++14 shell's HOG calls on float frames (tests/cpp/test_hog_float.cpp): rcr::vl_hog_pyramid, vl_hog_detect,
vl_hog_part_detect and train_hog_filter with multichannel = true and float_frames = true.

CPU: the translation unit compiles.  GPU: on CV_32FC1 and CV_32FC3 frames of different sizes (row steps wider than the pixels) the
shell's pyramid levels, detections, part detections and trained filter equal the Python calls' with float_frames=True bit for
bit, for both orientation modes; float_frames without multichannel, and 8-bit frames with it, throw."""
import os
import subprocess

import numpy as np
import pytest

import hog_train_ref as T
from superviseddescent_b200._capi import HogTrainParamC, HogWindowC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def float_binary(tmp_path_factory):
    from superviseddescent_b200 import build
    lib = build.build()
    out = str(tmp_path_factory.mktemp("cpp") / "test_hog_float")
    cmd = ["g++", "-std=c++14", "-O1", "-Wall", "-Werror=return-type", "-I", os.path.join(ROOT, "include"),
           "-I", os.path.join(ROOT, "superviseddescent_b200", "include"), os.path.join(ROOT, "tests", "cpp", "test_hog_float.cpp"),
           "-L", os.path.dirname(lib), "-lsd_b200", f"-Wl,-rpath,{os.path.dirname(lib)}", "-lpthread", "-o", out]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return out


def test_hog_float_shell_compiles_as_cxx14(float_binary):
    assert os.path.exists(float_binary)


@pytest.mark.gpu
@pytest.mark.parametrize("c", [1, 3])
@pytest.mark.parametrize("bil", [0, 1])
def test_shell_matches_python(float_binary, sd, tmp_path, c, bil):
    rng = np.random.default_rng(9 + bil + 2 * c)
    grey, boxes = T.planted_frames(33, 4, 240, 180, sides=(48, 96))
    frames = [np.ascontiguousarray((g[..., None] / np.float32(255) + rng.uniform(-0.1, 0.1, g.shape + (c,))).astype(np.float32))
              for g in grey]
    if c == 1:
        frames = [np.ascontiguousarray(f[..., 0]) for f in frames]
    frames[3] = np.ascontiguousarray(frames[3][:131, :197])      # another size
    box_frame, boxes = np.arange(3, dtype=np.int32), boxes[:3]   # frame 3 has no box
    scales = T.detector_scales(240, 180, 8, 5) + [2.0]
    cs, K, variant, fw, fh, P, pfw, pfh, R = 8, 9, 1, 5, 5, 2, 3, 3, 2
    dd = 3 * K + 4
    root = rng.normal(0, 0.2, (dd, fh, fw)).astype(np.float32)
    bias = np.float32(0.25)
    parts = rng.normal(0, 0.2, (P, dd, pfh, pfw)).astype(np.float32)
    anchors = rng.integers(0, 2 * fw - pfw, (P, 2)).astype(np.int32)
    deformation = np.tile(np.float32([0.05, 0.01, 0.05, -0.01]), (P, 1))
    kw = dict(lam=0.02, positive_overlap=0.5, negative_overlap=0.3, flip_positives=True, rounds=2, negatives_per_frame=12,
              mine_overlap=0.5, max_negatives=50, max_iterations=40)
    prm = HogTrainParamC(kw["lam"], kw["positive_overlap"], kw["negative_overlap"], 1, kw["rounds"], kw["negatives_per_frame"],
                         kw["mine_overlap"], kw["max_negatives"], kw["max_iterations"])
    blob = [np.int32(c).tobytes(), np.int32(len(frames)).tobytes()]
    for f in frames:
        blob += [np.array([f.shape[1], f.shape[0]], np.int32).tobytes(), f.tobytes()]
    blob += [np.int32(len(scales)).tobytes(), np.array(scales, np.float64).tobytes(), np.array([cs, K, variant, fw, fh], np.int32).tobytes(),
             root.tobytes(), bias.tobytes(), np.array([P, pfw, pfh, R], np.int32).tobytes(), parts.tobytes(), anchors.tobytes(),
             deformation.tobytes(), np.int32(len(boxes)).tobytes()]
    blob += [np.array([f, *b], np.int32).tobytes() for f, b in zip(box_frame, boxes)]
    blob += [bytes(prm)]
    (tmp_path / "in.bin").write_bytes(b"".join(blob))
    r = subprocess.run([float_binary, str(tmp_path / "in.bin"), str(tmp_path / "out.bin"), str(bil)], capture_output=True, text=True,
                       timeout=300)
    print(r.stdout[-3000:])
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]
    raw = (tmp_path / "out.bin").read_bytes()
    pos = 0

    def ints(n):
        nonlocal pos
        v = np.frombuffer(raw[pos:pos + 4 * n], np.int32)
        pos += 4 * n
        return v

    mc = dict(multichannel=True, bilinear_orientations=bool(bil), float_frames=True)
    feats, _ = sd.vl_hog_pyramid(frames, scales, cs, K, variant, **mc)
    for f in range(len(frames)):
        for s in range(len(scales)):
            rows, cols = ints(2)
            got = ints(rows * cols)
            want = feats[f][s]
            if want is None:
                assert rows == 0 and cols == 0
            else:
                assert np.array_equal(got, want.cpu().numpy().reshape(-1).view(np.int32)), (f, s)
    d = sd.vl_hog_detect(frames, scales, root[None], cs, K, threshold=-1.0, variant=variant, bias=[bias], pad=(1, 0), overlap=0.5,
                         max_candidates=4096, max_detections=30, **mc)
    for f in range(len(frames)):
        n = int(ints(1)[0])
        got = ints(9 * n).reshape(n, 9)
        m = d.frame == f
        ref = np.concatenate([d.boxes[m], d.scores[m].view(np.int32)[:, None], d.filter[m][:, None], d.level[m][:, None], d.cell[m]], 1)
        assert np.array_equal(got, ref), f
    model = sd.HogPartModel(root[None], [bias], parts[None], anchors[None], deformation[None], (0, 0), (0, 0), R)
    pd = sd.vl_hog_part_detect(frames, [s for s in scales if s <= 2], model, cs, K, -2.0, variant=variant, overlap=0.5,
                               max_candidates=4096, max_detections=30, **mc)
    total = 0
    for f in range(len(frames)):
        n = int(ints(1)[0])
        got = ints((9 + 7 * P) * n).reshape(n, 9 + 7 * P)
        m = pd.frame == f
        ref = np.concatenate([pd.boxes[m], pd.scores[m].view(np.int32)[:, None], pd.filter[m][:, None], pd.level[m][:, None], pd.cell[m],
                              np.concatenate([pd.placement[m], pd.part_scores[m].view(np.int32)[..., None], pd.parts[m]], axis=2)
                              .reshape(-1, 7 * P)], axis=1)
        assert np.array_equal(got, ref), f
        total += n
    assert total > 0
    hf = sd.train_hog_filter(frames, box_frame, boxes, scales, (fw, fh), cs, K, variant, pad=(1, 0), **kw, **mc)
    nf = dd * fh * fw
    filt = ints(nf)
    assert np.array_equal(filt, hf.filter.cpu().numpy().reshape(-1).view(np.int32))
    assert ints(1)[0] == np.float32(hf.bias).view(np.int32)
    nn = int(ints(1)[0])
    negs = [HogWindowC.from_buffer_copy(raw[pos + k * 16:pos + (k + 1) * 16]) for k in range(nn)]
    pos += 16 * nn
    assert pos == len(raw)
    S = len(scales)
    assert np.array_equal(np.asarray([(w.grid // S, w.grid % S, w.x, w.y) for w in negs], np.int32).reshape(-1, 4), hf.negatives)
