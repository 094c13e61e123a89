"""Host-side mirror of the reference's public interface for the hot path, on top of the C ABI.

Class and method names follow patrikhuber/superviseddescent:
  Regulariser, LinearRegressor                  include/superviseddescent/regressors.hpp:87-169, 318-400
  SupervisedDescentOptimiser, NoNormalisation    include/superviseddescent/superviseddescent.hpp:60-74, 85-361
  HoGParam, HogTransform                         include/rcr/adaptive_vlhog.hpp:41-60, 70-195
  InterEyeDistanceNormalisation, align_mean,
  detection_model, load/save_detection_model     include/rcr/model.hpp:64-219

The C++14 header shells (superviseddescent_b200/include/) are the drop-in for C++ callers; this module
is the same surface for Python callers, the tests and bench.py.  Matrices are row-major float32, one
sample per row; on the device they are torch CUDA tensors (torch = allocator + stream + distributed
plumbing only -- every computation below is a kernel of libsd_b200.so).
"""
from __future__ import annotations

import collections
import ctypes as C
import enum
import itertools
import math
from typing import Callable, List, Optional, Sequence

import numpy as np
import torch

from . import _capi
from ._capi import HogParam as HoGParam  # same field names as rcr::HoGParam
from ._capi import FaceChipParamC, FrameC, HogBoxC, HogDetectionC, HogGridC, HogGridsC, HogImageC, HogImagesC, HogPartMapC, HogPartModelC, HogPartPlacementC, HogPolarFieldsC, HogScoreMapC, HogTrainParamC, HogTrainReportC, HogWindowC, HostFrameC, ImageBatchC, LevelFramesC, NormalisationC, RegulariserC, SdError, SvmReportC, ptr


def _check(ctx, rc: int) -> None:
    if rc != 0:
        msg = _capi.lib().sd_last_error(ctx).decode() if ctx else "no context"
        raise SdError(rc, msg)


class Context:
    """One sd_ctx bound to a device and to torch's current stream on it."""

    def __init__(self, device: int = 0):
        if not torch.cuda.is_available():
            raise SdError(2, "no CUDA device: the engine has no CPU fallback")
        self.device = int(device)
        torch.cuda.set_device(self.device)
        self.stream = torch.cuda.current_stream(self.device)
        self._h = C.c_void_p()
        rc = _capi.lib().sd_ctx_create(self.device, C.c_void_p(self.stream.cuda_stream), C.byref(self._h))
        if rc != 0:
            raise SdError(rc, "sd_ctx_create failed (is a CUDA device visible?)")

    @property
    def h(self):
        return self._h

    def sync(self):
        _check(self._h, _capi.lib().sd_sync(self._h))

    def launches(self) -> int:
        return int(_capi.lib().sd_launch_count(self._h))

    def roi_fallbacks(self) -> int:
        return int(_capi.lib().sd_roi_fallback_count(self._h))

    def set_gram_mode(self, mode: int):
        """0 = 3xTF32 tensor-core Gram (default), 3 = unbiased 3xTF32, 1 = single-pass TF32, 2 = fp32 SIMT."""
        _check(self._h, _capi.lib().sd_set_gram_mode(self._h, int(mode)))

    def set_solver(self, mode) -> None:
        """Solver of systems with D > 256: 0 / "cholesky" = blocked Cholesky (default), 1 / "cg" = conjugate gradients on the
        tensor cores (falls back to the Cholesky if they stall)."""
        m = {"cholesky": 0, "cg": 1}.get(mode, mode)
        _check(self._h, _capi.lib().sd_set_solver(self._h, int(m)))

    def solver_iterations(self) -> int:
        """CG iterations of the last solve: +n = CG converged after n iterations and its answer was used; -n = CG ran n
        iterations, gave up, and the factorisation answered; 0 = CG was not tried."""
        return int(_capi.lib().sd_solver_iterations(self._h))

    def set_rank_diagnostic(self, on: bool) -> None:
        """With on, every solve also computes the numerical rank of its regularised system (ColPivHouseholderQRSolver's
        diagnostic); last_rank() reads it.  Off by default: it costs a pivoted factorisation of a copy of the D x D matrix."""
        _check(self._h, _capi.lib().sd_set_rank_diagnostic(self._h, int(bool(on))))

    def last_rank(self) -> int:
        """Numerical rank of the last solve's regularised system, or -1 when it was not computed (diagnostic off, or the
        distributed factorisation)."""
        return int(_capi.lib().sd_last_rank(self._h))

    def solver_timings(self):
        out = (C.c_float * 4)()
        _check(self._h, _capi.lib().sd_solver_timings(self._h, out))
        return {"At * A": out[0], "AtA + Reg": out[1], "Decomposition": out[2], "solve()": out[3]}

    def close(self):
        if self._h:
            _capi.lib().sd_ctx_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


_default_ctx: Optional[Context] = None


def default_context() -> Context:
    global _default_ctx
    if _default_ctx is None:
        dev = torch.cuda.current_device() if torch.cuda.is_available() else 0
        _default_ctx = Context(dev)
    return _default_ctx


def _tensor(a) -> torch.Tensor:
    """A tensor as given; an array (or anything numpy takes) as a tensor over a contiguous copy of it."""
    return a if isinstance(a, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(a))


def _dev(a, ctx: Context, dtype=torch.float32) -> torch.Tensor:
    return _tensor(a).to(device=f"cuda:{ctx.device}", dtype=dtype).contiguous()


# ------------------------------------------------------------------------------------------------
# regressors.hpp
# ------------------------------------------------------------------------------------------------
class RegularisationType(enum.IntEnum):
    Manual = 0
    MatrixNorm = 1


class Regulariser:
    """superviseddescent::Regulariser (regressors.hpp:87-169)."""

    RegularisationType = RegularisationType

    def __init__(self, regularisation_type: RegularisationType = RegularisationType.Manual, param: float = 0.0,
                 regularise_last_row: bool = True):
        self.regularisation_type = RegularisationType(regularisation_type)
        self.param = float(param)
        self.regularise_last_row = bool(regularise_last_row)

    def c(self) -> RegulariserC:
        return RegulariserC(int(self.regularisation_type), self.param, int(self.regularise_last_row))


class PartialPivLUSolver:
    """regressors.hpp:180-235 (also VerbosePartialPivLUSolver): the default Solver."""
    rank_revealing = False


class ColPivHouseholderQRSolver:
    """regressors.hpp:245-306: the Solver that checks invertibility.  Same solve, plus the numerical rank of the regularised
    AtA (diagonally pivoted Cholesky on the device); a deficient rank prints the reference's message (:290-293)."""
    rank_revealing = True


def _print_rank_warning(rank: int, D: int) -> None:
    """regressors.hpp:290-293"""
    print("The regularised AtA is not invertible. We continued learning, but Eigen may return garbage (their docu is not "
          f"very specific). (The rank is {rank}, full rank would be {D}). Increase lambda.")


class LinearRegressor:
    """superviseddescent::LinearRegressor<Solver> (regressors.hpp:318-400); `solver` plays the template parameter."""

    def __init__(self, regulariser: Optional[Regulariser] = None, ctx: Optional[Context] = None, solver=None):
        self.regulariser = regulariser or Regulariser()
        self.ctx = ctx
        self.solver = solver or PartialPivLUSolver()
        self.x: Optional[torch.Tensor] = None   # D x M, device
        self.last_lambda: Optional[float] = None
        self.last_rank: Optional[int] = None    # ColPivHouseholderQRSolver only: rank of the last learn / train level (-1: not computed)

    def _ctx(self) -> Context:
        if self.ctx is None:
            self.ctx = default_context()
        return self.ctx

    def learn(self, data, labels) -> bool:
        """regressors.hpp:345-350 -> Solver::solve (:199-234).  Always returns True, like the reference."""
        ctx = self._ctx()
        A = _dev(data, ctx)
        B = _dev(labels, ctx)
        N, D = A.shape
        M = B.shape[1]
        X = torch.empty((D, M), dtype=torch.float32, device=A.device)
        lam = C.c_float(0)
        reg = self.regulariser.c()
        if D > 256 and not getattr(self.solver, "rank_revealing", False):
            # the factorisation route works on centred rows (include/sd_b200.h, sd_centre_features): on a private copy
            if isinstance(data, torch.Tensor) and A.data_ptr() == data.data_ptr():
                A = A.clone()
            mu = torch.empty(D, dtype=torch.float32, device=A.device)
            _check(ctx.h, _capi.lib().sd_centre_features(ctx.h, None, ptr(A), C.c_int64(A.stride(0)), N, D, N, C.byref(reg), ptr(mu)))
            _check(ctx.h, _capi.lib().sd_learn_centred(ctx.h, None, ptr(A), C.c_int64(A.stride(0)), ptr(B), C.c_int64(B.stride(0)), N, D, M,
                                                       C.byref(reg), N, 0, ptr(mu), ptr(X), None, C.byref(lam)))
            self.x = X
            self.last_lambda = lam.value
            return True
        if getattr(self.solver, "rank_revealing", False):
            rank = C.c_int(-1)
            rc = _capi.lib().sd_learn_rank_revealing(ctx.h, ptr(A), C.c_int64(A.stride(0)), ptr(B), C.c_int64(B.stride(0)),
                                                     N, D, M, C.byref(reg), ptr(X), C.byref(lam), C.byref(rank))
            self.last_rank = rank.value
            if 0 <= rank.value < D:
                _print_rank_warning(rank.value, D)
                if rc == 5:                       # SD_ERR_NUMERIC: the factorisation of the singular matrix stopped; the reference returns garbage here
                    X.fill_(float("nan"))
                    rc = 0
            _check(ctx.h, rc)
        else:
            _check(ctx.h, _capi.lib().sd_learn(ctx.h, ptr(A), C.c_int64(A.stride(0)), ptr(B), C.c_int64(B.stride(0)),
                                               N, D, M, C.byref(reg), ptr(X), C.byref(lam)))
        self.x = X
        self.last_lambda = lam.value
        return True

    def predict(self, values) -> torch.Tensor:
        """regressors.hpp:377-381: values * x."""
        ctx = self._ctx()
        V = _dev(values, ctx)
        if V.dim() == 1:
            V = V.reshape(1, -1)
        N, D = V.shape
        M = self.x.shape[1]
        out = torch.empty((N, M), dtype=torch.float32, device=V.device)
        _check(ctx.h, _capi.lib().sd_predict(ctx.h, ptr(V), C.c_int64(V.stride(0)), N, D, ptr(self.x), M, ptr(out), C.c_int64(M)))
        return out

    def test(self, data, labels) -> float:
        """regressors.hpp:361-369: normalised least-squares residual."""
        ctx = self._ctx()
        V = _dev(data, ctx)
        Lb = _dev(labels, ctx)
        res = C.c_double(0)
        _check(ctx.h, _capi.lib().sd_test_residual(ctx.h, ptr(V), C.c_int64(V.stride(0)), ptr(Lb), C.c_int64(Lb.stride(0)),
                                                   V.shape[0], V.shape[1], ptr(self.x), self.x.shape[1], C.byref(res)))
        return res.value


# ------------------------------------------------------------------------------------------------
# normalisation strategies
# ------------------------------------------------------------------------------------------------
class NoNormalisation:
    """superviseddescent.hpp:60-74."""

    def c(self, num_landmarks: int) -> NormalisationC:
        return NormalisationC(0, 0, 0, (C.c_int32 * 4)(), (C.c_int32 * 4)())


class InterEyeDistanceNormalisation:
    """rcr::InterEyeDistanceNormalisation (model.hpp:84-116): normaliser = 1 / IED(params)."""

    def __init__(self, model_landmarks_list: Sequence[str], right_eye_identifiers: Sequence[str],
                 left_eye_identifiers: Sequence[str]):
        self.model_landmarks_list = [str(s) for s in model_landmarks_list]
        self.right_eye_identifiers = [str(s) for s in right_eye_identifiers]
        self.left_eye_identifiers = [str(s) for s in left_eye_identifiers]

    def _idx(self, ids, which):
        out = []
        for s in ids:
            if s not in self.model_landmarks_list:
                # helpers.hpp:144,153 throw std::runtime_error with this text
                raise RuntimeError(f"one of given {which}EyeIdentifiers ids not present in lms")
            out.append(self.model_landmarks_list.index(s))
        return out

    def c(self, num_landmarks: int = 0) -> NormalisationC:
        r = self._idx(self.right_eye_identifiers, "right")
        l = self._idx(self.left_eye_identifiers, "left")
        if not (1 <= len(r) <= 4 and 1 <= len(l) <= 4):
            raise ValueError("1..4 eye identifiers per eye are supported")
        return NormalisationC(1, len(r), len(l), (C.c_int32 * 4)(*(r + [0] * (4 - len(r)))), (C.c_int32 * 4)(*(l + [0] * (4 - len(l)))))


# ------------------------------------------------------------------------------------------------
# rcr::HogTransform (adaptive_vlhog.hpp:70-195), batched
# ------------------------------------------------------------------------------------------------
class FixedHogTransform:
    """The non-adaptive projection functor of the reference's hello-world (examples/landmark_detection.cpp:127-272):
    HogTransform(images, vlhog_variant, num_cells, cell_size, num_bins) -- a fixed patch of half-size
    num_cells * (cell_size / 2) around every landmark, no resize, no bias column.  Batched like HogTransform."""

    def __init__(self, images, vlhog_variant: int, num_cells: int, cell_size: int, num_bins: int, ctx: Optional["Context"] = None):
        self.ctx = ctx or default_context()
        self.images, self._batch = _device_images(images, self.ctx)     # colour: :201-206
        self.param = HoGParam(int(vlhog_variant), num_cells, cell_size, num_bins, 0.0)

    def feature_length(self, num_landmarks: int) -> int:
        return _capi.lib().sd_hog_feature_length(num_landmarks, C.byref(self.param)) - 1     # no bias column

    def __call__(self, parameters, regressor_level: int = 0, training_index=None) -> torch.Tensor:
        ctx = self.ctx
        x = _dev(parameters, ctx)
        single = x.dim() == 1
        if single:
            x = x.unsqueeze(0)
        n, L = x.shape[0], x.shape[1] // 2
        idx = None
        if training_index is not None:
            idx = torch.as_tensor(np.atleast_1d(np.asarray(training_index)), dtype=torch.int32).to(x.device)
        D = self.feature_length(L) + 1
        out = torch.empty((n, D), dtype=torch.float32, device=x.device)
        self.into(x, out, idx)
        feats = out[:, :D - 1]
        return feats[0] if single else feats

    def into(self, parameters: torch.Tensor, out: torch.Tensor, image_index: Optional[torch.Tensor] = None):
        """Writes the feature rows into out[:, :D]; column D receives the kernel's bias 1 (not part of this functor's
        output: callers overwrite or ignore it)."""
        ctx = self.ctx
        n, L = parameters.shape[0], parameters.shape[1] // 2
        _check(ctx.h, _capi.lib().sd_hog_batch(ctx.h, C.byref(self._batch), ptr(image_index) if image_index is not None else C.c_void_p(0),
                                               ptr(parameters), C.c_int64(parameters.stride(0)), n, L, None, C.byref(self.param),
                                               ptr(out), C.c_int64(out.stride(0))))


def bgr2gray(images, ctx: Optional["Context"] = None) -> torch.Tensor:
    """cv::cvtColor(BGR2GRAY) on the device (adaptive_vlhog.hpp:114-120): (count, H, W, 3) uint8 -> (count, H, W) uint8.
    Host arrays are uploaded first; the result stays in HBM."""
    ctx = ctx or default_context()
    t = _tensor(images)
    if t.dim() == 3:
        t = t.unsqueeze(0)
    if t.dtype != torch.uint8 or t.dim() != 4 or t.shape[3] != 3:
        raise ValueError("images must be (count, H, W, 3) uint8 (interleaved B, G, R)")
    t = t.to(f"cuda:{ctx.device}").contiguous()
    n, h, w, _ = t.shape
    out = torch.empty((n, h, w), dtype=torch.uint8, device=t.device)
    _check(ctx.h, _capi.lib().sd_bgr2gray(ctx.h, ptr(t), w, h, C.c_int64(t.stride(1)), C.c_int64(t.stride(0)), n,
                                          ptr(out), C.c_int64(out.stride(1)), C.c_int64(out.stride(0))))
    return out


def _device_images(images, ctx: Context):
    """The images of a HogTransform -> (the device tensor that owns them, the ImageBatchC sd_hog_batch reads).  A CUDA tensor
    (count, H, W) is used in place (copied first when it is not contiguous) and (count, H, W, 3) converted by bgr2gray; a host
    (count, H, W) array or tensor is copied in one piece.  Anything else from the host -- a list of (H, W) or (H, W, 3) frames of any sizes, or a (count, H, W, 3)
    array -- is uploaded by sd_upload_frames (_grey_frames)."""
    if not isinstance(images, (list, tuple)):
        images = _tensor(images)
        if images.dim() == 2:
            images = images.unsqueeze(0)
        if images.dtype != torch.uint8 or not (images.dim() == 3 or (images.dim() == 4 and images.shape[3] == 3)):
            raise ValueError("images must be (count, H, W) uint8, (count, H, W, 3) uint8, or a list of such frames of any sizes")
        if images.dim() == 3:       # grey: from the host in one copy, however many frames; on the device, contiguous
            images = images.to(f"cuda:{ctx.device}").contiguous()
        elif images.is_cuda:
            images = bgr2gray(images, ctx)
    keep, ib, _ = _grey_frames(images, ctx, lambda w, h: None)
    if ib is None:
        # no frames: sd_upload_frames refuses an empty batch, so this call always raises its SdError
        return _upload_host_frames([], ctx)
    return keep, ib


def _upload_host_frames(recs, ctx: Context):
    """sd_host_frame records -> (the device tensor that owns the grey frames, the ImageBatchC sd_hog_batch reads)."""
    dev = f"cuda:{ctx.device}"
    table = (HostFrameC * len(recs))(*recs)
    nbytes = C.c_size_t(0)
    _check(ctx.h, _capi.lib().sd_upload_frames(ctx.h, table, len(recs), None, C.byref(nbytes), None))
    buf = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
    ib = ImageBatchC()
    _check(ctx.h, _capi.lib().sd_upload_frames(ctx.h, table, len(recs), ptr(buf), C.byref(nbytes), C.byref(ib)))
    return buf, ib


# ------------------------------------------------------------------------------------------------
# batches of the dense-HOG calls: items packed end to end, descriptor tables, result buffers
# ------------------------------------------------------------------------------------------------
def _starts(counts):
    """The offset of each item when items of these element counts lie end to end."""
    return list(itertools.accumulate(counts, initial=0))[:-1]


def _pack(items, dev):
    """Tensors -> (one device buffer of their elements, end to end, in one copy; the element offset of each)."""
    return torch.cat([t.reshape(-1) for t in items]).to(dev), _starts([t.numel() for t in items])


def _device_table(descs, dev) -> torch.Tensor:
    """A non-empty list of descriptors of one ctypes Structure type, as one table in a device tensor that owns its bytes."""
    table = (type(descs[0]) * len(descs))(*descs)
    return torch.from_numpy(np.frombuffer(bytes(table), dtype=np.uint8).copy()).to(dev)


def _results(shapes, dev, zero: bool = False):
    """The float32 results of a call, in one new device buffer -> (buffer, element offsets, results).

    shapes: one tuple, the shape of a batch tensor, which is the buffer itself (offsets None); or a list of per-item shapes,
    laid end to end and returned as a list of views, None for an item whose shape is None.  The buffer of a list has at least
    one element, so that a call whose items are all empty still gets a valid pointer.  zero: the buffer starts zeroed."""
    alloc = torch.zeros if zero else torch.empty
    if isinstance(shapes, tuple):
        out = alloc(shapes, dtype=torch.float32, device=dev)
        return out, None, out
    counts = [0 if s is None else math.prod(s) for s in shapes]
    offsets = _starts(counts)
    out = alloc(max(sum(counts), 1), dtype=torch.float32, device=dev)
    return out, offsets, [None if s is None else out[o:o + c].view(s) for o, c, s in zip(offsets, counts, shapes)]


def _dense_results(ctx, sizes, frame, cell_size: int, num_bins: int, variant: int, run):
    """The dense HOG of frames of sizes [(H, W)], written by run(out, offsets).  frame: the (H, W) of every frame when the call
    describes its frames as one batch, without a descriptor table; the result is then one (count, dd, hogH, hogW) tensor
    (offsets None), and for no frames run is not called.  Otherwise it is a list of (dd, hogH, hogW) views of one buffer, at
    the int64 element offsets that offsets holds on the device."""
    dev = f"cuda:{ctx.device}"
    if frame is not None:
        h, w = frame
        out, _, res = _results((len(sizes),) + hog_dense_shape(w, h, cell_size, num_bins, variant), dev)
        if sizes:
            run(out, None)
        return res
    out, offsets, res = _results([hog_dense_shape(w, h, cell_size, num_bins, variant) for h, w in sizes], dev)
    run(out, torch.tensor(offsets, dtype=torch.int64, device=dev))
    return res


# ------------------------------------------------------------------------------------------------
# dense HOG of whole frames: vl_hog_put_image + vl_hog_extract (hog.h:104-139)
# ------------------------------------------------------------------------------------------------
def hog_dense_shape(width: int, height: int, cell_size: int, num_bins: int, variant: int = 1):
    """(dd, hogH, hogW) of the dense HOG of a width x height frame (hog.c:542-548); SdError for an invalid configuration."""
    w, h, d = C.c_int(), C.c_int(), C.c_int()
    rc = _capi.lib().sd_hog_dense_shape(int(width), int(height), int(cell_size), int(num_bins), int(variant), C.byref(w), C.byref(h),
                                        C.byref(d))
    if rc:
        raise SdError(rc, f"invalid dense HOG configuration: {width} x {height} px, cell_size {cell_size}, num_bins {num_bins}, "
                          f"variant {variant} (frames > 3 px and at least half a cell, cell_size 1..32, num_bins 1..16)")
    return d.value, h.value, w.value


def _grey_frames(frames, ctx: Context, check):
    """The 8-bit frames of hog_dense / vl_hog_pyramid -> (the device tensor that owns them, their ImageBatchC, [(H, W)] per frame).
    A CUDA (count, H, W) uint8 tensor is used in place; host frames are uploaded by sd_upload_frames after check(W, H) has
    accepted every size.  An empty list of host frames gives (None, None, [])."""
    if isinstance(frames, torch.Tensor) and frames.is_cuda:
        if frames.dtype != torch.uint8 or frames.dim() != 3:
            raise ValueError("a device tensor of frames must be (count, H, W) uint8")
        t = frames.to(f"cuda:{ctx.device}")
        if t.stride(2) != 1:
            t = t.contiguous()
        n, h, w = t.shape
        return t, ImageBatchC(C.c_void_p(t.data_ptr()), w, h, t.stride(1), t.stride(0), n), [(h, w)] * n
    if isinstance(frames, (list, tuple)):
        frames = list(frames)
    else:
        a = frames.numpy() if isinstance(frames, torch.Tensor) else np.asarray(frames)
        if a.dtype != np.uint8 or not (a.ndim == 3 or (a.ndim == 4 and a.shape[3] == 3)):
            raise ValueError("frames must be (count, H, W) uint8, (count, H, W, 3) uint8, or a list of such frames of any sizes")
        frames = list(a)
    recs, arrays = _host_frames(frames)                   # arrays: the bytes stay alive until the upload returns
    sizes = [(r.height, r.width) for r in recs]
    if not recs:
        return None, None, []
    for h, w in set(sizes):
        check(w, h)                                       # refuse before the upload
    keep, ib = _upload_host_frames(recs, ctx)
    return keep, ib, sizes


def hog_dense(frames, cell_size: int, num_bins: int, variant: int = 1, ctx: Optional[Context] = None):
    """VLFeat HOG of whole 8-bit frames (vl_hog_new(variant, num_bins) + vl_hog_put_image(frame, 1 channel, cell_size) +
    vl_hog_extract) on the device, in VLFeat's planar layout [dd][hogH][hogW] with x fastest.

    frames: a CUDA uint8 tensor (count, H, W), used in place; or host frames -- a (count, H, W) or (count, H, W, 3) uint8 array,
    or a list of (H, W) / (H, W, 3) uint8 frames of any sizes -- uploaded by sd_upload_frames (B,G,R colour converted to grey
    there, as HogTransform does).  variant: 1 = UoCTTI (dd = 3K + 4), 0 = Dalal-Triggs (dd = 4K).
    Returns one (count, dd, hogH, hogW) float32 CUDA tensor when all frames have one size, else a list of (dd, hogH, hogW)
    tensors."""
    ctx = ctx or default_context()
    lib = _capi.lib()
    keep, ib, sizes = _grey_frames(frames, ctx, lambda w, h: hog_dense_shape(w, h, cell_size, num_bins, variant))
    if ib is None:
        return []
    return _dense_results(ctx, sizes, None if ib.d_frames else (ib.height, ib.width), cell_size, num_bins, variant,
                          lambda out, offsets: _check(ctx.h, lib.sd_hog_dense(ctx.h, C.byref(ib), int(cell_size), int(num_bins),
                                                                              int(variant), ptr(out), ptr(offsets))))


_VL_HOG_DTYPES = {torch.uint8: 0, torch.float32: 1}    # SD_HOG_U8, SD_HOG_F32


def _vl_hog_frame(t: torch.Tensor, channels_last: bool, batched: bool):
    """(channels, sd_hog_image fields) of one frame, or of the first frame of a batch, read through t's strides."""
    s = t.stride()[1:] if batched else t.stride()
    shape = t.shape[1:] if batched else t.shape
    if len(shape) == 2:
        (h, w), (rs, ps), c, cst = shape, s, 1, 0
    elif channels_last:
        (h, w, c), (rs, ps, cst) = shape, s
    else:
        (c, h, w), (cst, rs, ps) = shape, s
    return c, HogImageC(w, h, 0, rs, ps, cst)


def vl_hog(images, cell_size: int, num_bins: int, variant: int = 1, bilinear_orientations: bool = False, channels_last: bool = False,
           ctx: Optional[Context] = None):
    """VLFeat HOG of whole uint8 or float32 frames of one or more channels (vl_hog_new(variant, num_bins) +
    vl_hog_set_use_bilinear_orientation_assignments(bilinear_orientations) + vl_hog_put_image(frame, channels, cell_size) +
    vl_hog_extract) on the device, in VLFeat's planar layout [dd][hogH][hogW] with x fastest.

    images: a batch -- an array or tensor (count, H, W), (count, C, H, W), or (count, H, W, C) with channels_last=True -- or a
    list of frames of any sizes, (H, W), (C, H, W) or (H, W, C), all of one dtype and one C.  CUDA tensors are read in place
    through their strides; host frames are copied into one device buffer.  At each pixel the gradient comes from the channel
    with the largest gradient; channels are used as given (for OpenCV frames channel 0 is B).  bilinear_orientations: every
    pixel votes into its two nearest orientation bins.  variant: 1 = UoCTTI (dd = 3K + 4), 0 = Dalal-Triggs (dd = 4K).
    Returns one (count, dd, hogH, hogW) float32 CUDA tensor when all frames have one size, else a list of (dd, hogH, hogW)
    tensors."""
    ctx = ctx or default_context()
    lib = _capi.lib()
    keep, ib, sizes = _hog_images(images, channels_last, ctx, lambda w, h: hog_dense_shape(w, h, cell_size, num_bins, variant))
    if ib is None:
        return []
    bil = int(bool(bilinear_orientations))
    return _dense_results(ctx, sizes, None if ib.d_frames else (ib.frame.height, ib.frame.width), cell_size, num_bins, variant,
                          lambda out, offsets: _check(ctx.h, lib.sd_hog_dense_images(ctx.h, C.byref(ib), int(cell_size), int(num_bins),
                                                                                     int(variant), bil, ptr(out), ptr(offsets))))


def _hog_images(images, channels_last: bool, ctx: Context, check, float_only: bool = False, frames_out=None):
    """The frames of vl_hog, or of the multichannel=True route of the sliding-window calls -> (what owns their device bytes,
    their HogImagesC, [(H, W)] per frame).  A batch is read through its strides (a CUDA tensor in place, a host one after one
    copy); a list of frames is packed end to end in one device buffer after check(W, H) has accepted every size, with a
    descriptor table when the sizes differ.  An empty list gives (None, None, []).  float_only: frames of another dtype than
    float32 are refused before any upload.  frames_out (a list): receives each frame's HogImageC, offsets from the data."""
    dev = f"cuda:{ctx.device}"

    def dtype_of(t):
        if float_only and t.dtype != torch.float32:
            raise ValueError("float_frames=True takes float32 frames")
        if t.dtype not in _VL_HOG_DTYPES:
            raise ValueError("frames must be uint8 or float32")
        return _VL_HOG_DTYPES[t.dtype]

    ib = HogImagesC()
    ib.d_frames = None
    if isinstance(images, (list, tuple)):
        frames = [_tensor(f) for f in images]
        if not frames:
            return None, None, []
        if any(f.dim() not in (2, 3) for f in frames):
            raise ValueError("every frame of a list must be (H, W), (C, H, W), or (H, W, C) with channels_last=True")
        if len({f.dtype for f in frames}) != 1:
            raise ValueError("all frames must have one dtype")
        dt = dtype_of(frames[0])
        frames = [f.contiguous() for f in frames]
        descs = [_vl_hog_frame(f, channels_last, False) for f in frames]
        if len({c for c, _ in descs}) != 1:
            raise ValueError("all frames must have one number of channels")
        sizes = [(d.height, d.width) for _, d in descs]
        for h, w in set(sizes):
            check(w, h)                                       # refuse before the upload
        data, offsets = _pack(frames, dev)
        for (_, d), o in zip(descs, offsets):
            d.offset = o
        if frames_out is not None:
            frames_out.extend(d for _, d in descs)
        ib.channels, ib.count = descs[0][0], len(frames)
        keep = data
        if len(set(sizes)) == 1:
            ib.frame, ib.image_stride = descs[0][1], frames[0].numel()
        else:
            table = _device_table([d for _, d in descs], dev)
            ib.d_frames = table.data_ptr()
            keep = (data, table)
    else:
        t = _tensor(images)
        if t.dim() not in (3, 4):
            raise ValueError("a batch of frames must be (count, H, W), (count, C, H, W), or (count, H, W, C) with channels_last=True")
        dt = dtype_of(t)
        data = keep = t.to(dev)
        ib.channels, ib.frame = _vl_hog_frame(data, channels_last, True)
        ib.count, ib.image_stride = data.shape[0], data.stride(0)
        sizes = [(ib.frame.height, ib.frame.width)] * ib.count
        if frames_out is not None:
            f = ib.frame
            frames_out.extend(HogImageC(f.width, f.height, f.offset + i * ib.image_stride, f.row_stride, f.pixel_stride, f.channel_stride)
                              for i in range(ib.count))
    ib.d_data, ib.dtype = data.data_ptr(), dt
    return keep, ib, sizes


# The distinct frames of a HogTransform are uploaded when their grey bytes fit in this share of the device's free memory (read when
# the transform is first used); otherwise they stay in host memory and train() / test() gather them per level.
DEVICE_FRAME_SHARE = 0.5
# bytes of one staging half of the host route (sd_level_frames.stage_half_bytes); 0: the library's default
HOST_STAGE_HALF = 0


def _round16(v: int) -> int:
    return (v + 15) // 16 * 16


def _free_device_bytes(device: int) -> int:
    """Free device memory, counting what torch has reserved but not handed out."""
    return torch.cuda.mem_get_info(device)[0] + torch.cuda.memory_reserved(device) - torch.cuda.memory_allocated(device)


class _PinnedBuffer:
    """bytes of pinned host memory from sd_host_alloc (exactly that size), as a numpy uint8 array; freed with the object"""

    def __init__(self, ctx: Context, nbytes: int):
        self.ctx, self._p = ctx, C.c_void_p()
        _check(ctx.h, _capi.lib().sd_host_alloc(ctx.h, C.c_size_t(nbytes), C.byref(self._p)))
        self.array = np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(self._p.value))

    def __del__(self):
        try:
            if self._p:
                _capi.lib().sd_host_free(self.ctx.h, self._p)
                self._p = C.c_void_p()
        except Exception:
            pass


# sd_level_frames / sd_hog_batch: OR-ed into a sample's frame index, the sample is a sample of the frame's left-right mirror
SAMPLE_MIRRORED = 1 << 30

# sd_sample_warp as a numpy record (56 bytes, the C layout)
_WARP_DTYPE = np.dtype([("m", "<f8", (6,)), ("width", "<i4"), ("height", "<i4")])


def _warp_table(warps, warp_sizes, frame_sizes, dev) -> torch.Tensor:
    """(N, 2, 3) V-to-frame matrices and (N, 2) (Wv, Hv) sizes (default: frame_sizes, the (N, 2) sizes of each sample's frame,
    or None when they are not known) -> the device table of N sd_sample_warp records, as bytes."""
    m = np.asarray(warps.cpu() if isinstance(warps, torch.Tensor) else warps, dtype=np.float64)
    if m.ndim != 3 or m.shape[1:] != (2, 3):
        raise ValueError(f"warps must be (N, 2, 3), got {m.shape}")
    n = m.shape[0]
    if warp_sizes is None:
        if frame_sizes is None:
            raise ValueError("warp_sizes is needed: the frames' sizes are not known here")
        warp_sizes = frame_sizes
    sz = np.asarray(warp_sizes.cpu() if isinstance(warp_sizes, torch.Tensor) else warp_sizes, dtype=np.int64)
    sz = np.broadcast_to(sz, (n, 2)) if sz.shape == (2,) else sz
    if sz.shape != (n, 2):
        raise ValueError(f"warp_sizes must be (N, 2) (Wv, Hv) for {n} warps, got {sz.shape}")
    rec = np.zeros(n, dtype=_WARP_DTYPE)
    rec["m"] = m.reshape(n, 6)
    rec["width"], rec["height"] = np.clip(sz[:, 0], -2 ** 31, 2 ** 31 - 1), np.clip(sz[:, 1], -2 ** 31, 2 ** 31 - 1)
    return torch.from_numpy(rec.view(np.uint8).copy()).to(dev)


def rotation_warp(centre, angle: float, scale: float = 1.0) -> np.ndarray:
    """The V-to-frame matrix (2 x 3 float64) whose V is the frame rotated by angle degrees about centre and scaled by scale:
    the inverse of cv2.getRotationMatrix2D(centre, angle, scale) (angle counter-clockwise, as cv2), in closed form.  Its V is
    what cv2.warpAffine(frame, cv2.getRotationMatrix2D(centre, angle, scale), size) gives."""
    cx, cy = float(centre[0]), float(centre[1])
    a = math.radians(float(angle))
    alpha, beta = math.cos(a) * float(scale), math.sin(a) * float(scale)
    # getRotationMatrix2D: [[alpha, beta, (1 - alpha) cx - beta cy], [-beta, alpha, beta cx + (1 - alpha) cy]]
    return invert_warp(np.array([[alpha, beta, (1 - alpha) * cx - beta * cy], [-beta, alpha, beta * cx + (1 - alpha) * cy]]))


def invert_warp(M) -> np.ndarray:
    """The exact algebraic inverse, in float64, of one (2, 3) affine matrix or of each of (N, 2, 3)."""
    m = np.asarray(M, dtype=np.float64)
    if m.shape[-2:] != (2, 3) or m.ndim not in (2, 3):
        raise ValueError(f"invert_warp: M must be (2, 3) or (N, 2, 3), got {m.shape}")
    a, b, c, d, e, f = (m[..., i // 3, i % 3] for i in range(6))
    det = a * e - b * d
    if np.any(det == 0) or not np.all(np.isfinite(det)):
        raise ValueError("invert_warp: a matrix is singular or not finite")
    ia, ib, id_, ie = e / det, -b / det, -d / det, a / det
    out = np.empty_like(m)
    out[..., 0, 0], out[..., 0, 1], out[..., 0, 2] = ia, ib, -(ia * c + ib * f)
    out[..., 1, 0], out[..., 1, 1], out[..., 1, 2] = id_, ie, -(id_ * c + ie * f)
    return out


def warp_landmarks(x, M) -> np.ndarray:
    """Landmarks x ((N, 2L) rows [x.., y..], or one (2L,) row) mapped through one (2, 3) matrix or one per row ((N, 2, 3)), in
    float64, returned as float32: ground truth into a warp's V with invert_warp(warp), results back to the frame with the warp."""
    x = np.asarray(x, dtype=np.float32)
    single = x.ndim == 1
    x = np.atleast_2d(x)
    m = np.asarray(M, dtype=np.float64)
    L = x.shape[1] // 2
    if x.ndim != 2 or x.shape[1] != 2 * L or L < 1:
        raise ValueError("warp_landmarks: x must be (N, 2L) or (2L,)")
    if m.shape == (2, 3):
        m = np.broadcast_to(m, (x.shape[0], 2, 3))
    if m.shape != (x.shape[0], 2, 3):
        raise ValueError(f"warp_landmarks: M must be (2, 3) or ({x.shape[0]}, 2, 3), got {m.shape}")
    px, py = x[:, :L].astype(np.float64), x[:, L:].astype(np.float64)
    out = np.empty_like(x)
    out[:, :L] = m[:, 0, 0:1] * px + m[:, 0, 1:2] * py + m[:, 0, 2:3]
    out[:, L:] = m[:, 1, 0:1] * px + m[:, 1, 1:2] * py + m[:, 1, 2:3]
    return out[0] if single else out


class HogTransform:
    """Projection functor h.  images: (count, H, W) uint8 (8UC1) or (count, H, W, 3) uint8 (8UC3, B G R: converted
    once on the device as adaptive_vlhog.hpp:114-120 does per call), on host or device, or a list of such frames of any
    sizes.

    A list may name one frame several times (rcr-train makes 11 samples per photo): entries that are the same object or share
    data pointer, shape and strides are one frame, held once.  image_index (optional, N ints): sample i reads images[image_index[i]]
    (default: sample i reads images[i]).  mirrored (optional, N bools, one per sample as image_index): sample i is a sample of the
    left-right mirror of its frame (np.fliplr, cv::flip(f, 1)), with its landmarks in the mirror's coordinates (mirror_landmarks);
    the frame is still held once and read right to left, and every row is bit for bit that of the mirror passed as a frame of
    its own.  warps (optional, (N, 2, 3) float64, one per sample as mirrored; not with mirrored): sample i is a sample of
    V_i = cv2.warpAffine(grey frame, warps[i], warp_sizes[i], INTER_LINEAR | WARP_INVERSE_MAP) (sd_sample_warp; rotation_warp),
    with its landmarks in V_i's coordinates; V_i is never built, and every row is bit for bit that of V_i passed as a frame of its
    own.  warp_sizes ((N, 2) (Wv, Hv)) defaults to each sample's frame size.  The flags and warps hold wherever the transform's sample map is used: __call__ and debug without a training_index, into
    without an image_index, and the optimiser's train / test / predict.  Host frames whose grey bytes fit in DEVICE_FRAME_SHARE of the free device memory are
    uploaded when the transform is first used; larger sets stay in host memory and the optimiser gathers them level by level.
    Frames the levels can read in place (pinned and aligned, sd_host_frame_in_place) are read at every level, so changing them
    after the first use changes the result; the others are copied once, on first use, into one pinned buffer.  Until the first
    use the transform holds references to the arrays of a list: do not change them before it.

    __call__(parameters, regressor_level, training_index) keeps the reference's meaning
    (adaptive_vlhog.hpp:109) but takes ALL rows at once: parameters is (N, 2L) and training_index an
    optional (N,) int array of indices into images (default: the sample -> frame map above), read unmirrored.  A single (2L,) row
    with an int training_index is accepted too (predict()'s call shape, superviseddescent.hpp:332).
    """

    def __init__(self, images, hog_params: Sequence[HoGParam], model_landmarks_list: Sequence[str],
                 right_eye_identifiers: Sequence[str], left_eye_identifiers: Sequence[str], ctx: Optional[Context] = None,
                 image_index=None, mirrored=None, warps=None, warp_sizes=None):
        self.ctx = ctx or default_context()
        self.hog_params = list(hog_params)
        self.norm = InterEyeDistanceNormalisation(model_landmarks_list, right_eye_identifiers, left_eye_identifiers)
        self.num_landmarks = len(self.norm.model_landmarks_list)
        self.images = None            # device bytes that hold the frames (device route)
        self._batch = None
        self._host = None             # (HostFrameC table, arrays that own the bytes) on the host route
        self._frames = None           # distinct host frames, until the route is chosen
        self._list_frame = None       # list entry -> distinct frame (None: entry i is frame i)
        if isinstance(images, (list, tuple)):
            self._frames, self._list_frame = self._distinct(images)
        else:
            self.images, self._batch = _device_images(images, self.ctx)
        n_list = len(images)
        if image_index is not None:
            idx = np.ascontiguousarray(image_index, dtype=np.int64).ravel()
            if idx.size and (idx.min() < 0 or idx.max() >= n_list):
                raise ValueError("image_index refers to an image that is not in the list")
            sample = (self._list_frame[idx] if self._list_frame is not None else idx).astype(np.int32)
        else:
            sample = self._list_frame
        n_samples = idx.size if image_index is not None else n_list
        if mirrored is not None and warps is not None:
            raise ValueError("HogTransform: mirrored and warps exclude each other (a mirror is the warp [-1, 0, W - 1; 0, 1, 0])")
        self._sample_warp = None
        if warps is not None:
            base = sample if sample is not None else np.arange(n_samples, dtype=np.int32)
            if self._frames is not None:
                fsz = np.array([(r.width, r.height) for r, _ in self._frames], dtype=np.int64)[base]
            else:
                fsz = None if self._batch.d_frames else np.array([(self._batch.width, self._batch.height)] * n_samples, dtype=np.int64)
            if len(np.asarray(warps.cpu() if isinstance(warps, torch.Tensor) else warps)) != n_samples:
                raise ValueError(f"warps has {len(warps)} entries for {n_samples} samples")
            self._sample_warp = _warp_table(warps, warp_sizes, fsz, f"cuda:{self.ctx.device}")
        if mirrored is not None:
            flags = np.ascontiguousarray(mirrored, dtype=bool).ravel()
            if flags.size != n_samples:
                raise ValueError(f"mirrored has {flags.size} entries for {n_samples} samples")
            base = sample if sample is not None else np.arange(n_samples, dtype=np.int32)
            sample = np.where(flags, base | np.int32(SAMPLE_MIRRORED), base).astype(np.int32)
        self._sample_frame = None if sample is None else torch.from_numpy(np.ascontiguousarray(sample, dtype=np.int32)).to(f"cuda:{self.ctx.device}")

    @staticmethod
    def _distinct(images):
        """(list of (sd_host_frame, owning array) of the distinct frames, list entry -> frame index)"""
        frames, index, seen = [], np.empty(len(images), dtype=np.int32), {}
        for i, (rec, a) in enumerate(zip(*_host_frames(images))):
            key = (a.ctypes.data, a.shape, a.strides)
            if key not in seen:
                seen[key] = len(frames)
                frames.append((rec, a))
            index[i] = seen[key]
        return frames, index

    def _choose_route(self):
        """Once, on first use: upload the distinct frames when their grey bytes fit in DEVICE_FRAME_SHARE of the free device
        memory, else keep them in host memory."""
        if self._frames is None:
            return
        frames, self._frames = self._frames, None
        recs = [r for r, _ in frames]
        grey = sum(r.height * _round16(r.width) for r in recs)
        if grey <= DEVICE_FRAME_SHARE * _free_device_bytes(self.ctx.device):
            self.images, self._batch = _upload_host_frames(recs, self.ctx)
            return
        # host route: pinned frames with 16-byte aligned rows (and every 16-pixel step of a row inside it) are read in place; the
        # others are packed once into one pinned buffer at such a pitch
        lib = _capi.lib()

        def in_place(r):
            ok = C.c_int(0)
            _check(self.ctx.h, lib.sd_host_frame_in_place(self.ctx.h, C.byref(r), C.byref(ok)))
            return bool(ok.value)
        pack = [not in_place(r) for r, _ in frames]
        pitch = [r.channels * _round16(r.width) for r, _ in frames]
        total = sum(p * r.height for (r, _), p, k in zip(frames, pitch, pack) if k)
        buf = _PinnedBuffer(self.ctx, total) if total else None
        out, keep, off = [], [a for _, a in frames], 0
        for (r, a), p, k in zip(frames, pitch, pack):
            if k:
                dst = buf.array[off:off + p * r.height].reshape(r.height, p)
                dst[:, :r.width * r.channels] = a.reshape(r.height, r.width * r.channels)
                off += p * r.height
                r = HostFrameC(dst.ctypes.data, r.width, r.height, p, r.channels)
            out.append(r)
        self._host = ((HostFrameC * len(out))(*out), keep, buf)

    def on_device(self) -> bool:
        """Whether the frames are resident on the device (False: they stay in host memory and are gathered per level)."""
        self._choose_route()
        return self._host is None

    def batch(self) -> ImageBatchC:
        self._choose_route()
        if self._host is not None:
            raise SdError(1, "HogTransform: the frames stay in host memory (they do not fit on the device); only the optimiser's "
                             "train() / test() / predict() read them")
        return self._batch

    def sample_frame(self, n: int) -> Optional[torch.Tensor]:
        """Device (n,) int32 index: sample i reads frame sample_frame[i] of batch() (None: frame i)."""
        if self._sample_frame is None:
            return None
        if n > self._sample_frame.numel():
            raise ValueError(f"{n} samples but the image list / image_index has {self._sample_frame.numel()}")
        return self._sample_frame[:n]

    def level_frames(self, n: int) -> LevelFramesC:
        """The sd_level_frames of n samples for sd_train_level / sd_apply_level: the device batch or the host frames, and the
        sample -> frame index.  It holds references to what it points at."""
        index = self.sample_frame(n)
        warp = self.sample_warp(n)
        f = LevelFramesC(d_sample_frame=ptr(index), stage_half_bytes=HOST_STAGE_HALF, d_sample_warp=ptr(warp))
        if self.on_device():
            f.images = C.pointer(self._batch)
        else:
            f.host_frames, f.num_host_frames = self._host[0], len(self._host[0])
        f.keep = (index, warp, self._batch, self._host)
        return f

    def sample_warp(self, n: int) -> Optional[torch.Tensor]:
        """The device table of the first n samples' sd_sample_warp records, as bytes (None: no warps)."""
        if self._sample_warp is None:
            return None
        if n * _WARP_DTYPE.itemsize > self._sample_warp.numel():
            raise ValueError(f"{n} samples but warps has {self._sample_warp.numel() // _WARP_DTYPE.itemsize}")
        return self._sample_warp[:n * _WARP_DTYPE.itemsize]

    def feature_length(self, level: int) -> int:
        return _capi.lib().sd_hog_feature_length(self.num_landmarks, C.byref(self.hog_params[level]))

    def into(self, parameters: torch.Tensor, level: int, out: torch.Tensor, image_index: Optional[torch.Tensor] = None):
        """Writes the feature rows into out[:, :D] (out may be wider: extended [A | b] operand).  image_index: frames of batch()
        (default: sample_frame, with the samples' warps)."""
        n = parameters.shape[0]
        warp = self.sample_warp(n) if image_index is None else None
        if image_index is None:
            image_index = self.sample_frame(n)
        self._into(parameters, level, out, image_index, warp)

    def _into(self, parameters: torch.Tensor, level: int, out: torch.Tensor, image_index, warp):
        ctx = self.ctx
        n = parameters.shape[0]
        eyes = self.norm.c()
        ib = self.batch()
        idx_ptr = ptr(image_index) if image_index is not None else C.c_void_p(0)
        args = (ctx.h, C.byref(ib), idx_ptr, ptr(parameters), C.c_int64(parameters.stride(0)), n, self.num_landmarks, C.byref(eyes),
                C.byref(self.hog_params[level]))
        if warp is not None:
            _check(ctx.h, _capi.lib().sd_hog_batch_warped(*args, ptr(warp), ptr(out), C.c_int64(out.stride(0))))
        else:
            _check(ctx.h, _capi.lib().sd_hog_batch(*args, ptr(out), C.c_int64(out.stride(0))))

    def _frame_index(self, training_index, n: int, single: bool, device) -> Optional[torch.Tensor]:
        """training_index (indices into images) -> frames of batch()"""
        if training_index is None:
            return torch.zeros(1, dtype=torch.int32, device=device) if single else self.sample_frame(n)
        if np.isscalar(training_index):
            training_index = [int(training_index)] * n
        idx = np.asarray(training_index, dtype=np.int64)
        if self._list_frame is not None:
            idx = self._list_frame[idx]
        return torch.from_numpy(np.ascontiguousarray(idx, dtype=np.int32)).to(device)

    def __call__(self, parameters, regressor_level: int, training_index=None) -> torch.Tensor:
        x = _dev(parameters, self.ctx)
        single = x.dim() == 1
        if single:
            x = x.reshape(1, -1)
        idx = self._frame_index(training_index, x.shape[0], single, x.device)
        warp = self.sample_warp(x.shape[0]) if training_index is None and not single else None
        D = self.feature_length(regressor_level)
        out = torch.empty((x.shape[0], D), dtype=torch.float32, device=x.device)
        self._into(x, regressor_level, out, idx, warp)
        return out[0] if single else out

    def debug(self, parameters, level: int, training_index=None):
        """Integer parity taps: (geometry [N,L,3] = cx,cy,half ; patches [N,L,fs,fs] u8 ; bins [N,L,fs,fs] i8)."""
        ctx = self.ctx
        x = _dev(parameters, ctx)
        n = x.shape[0]
        p = self.hog_params[level]
        fs = p.num_cells * p.cell_size
        L = self.num_landmarks
        geo = torch.empty((n, L, 3), dtype=torch.int32, device=x.device)
        patches = torch.empty((n, L, fs, fs), dtype=torch.uint8, device=x.device)
        bins = torch.empty((n, L, fs, fs), dtype=torch.int8, device=x.device)
        idx = self._frame_index(training_index, n, False, x.device)
        warp = self.sample_warp(n) if training_index is None else None
        eyes = self.norm.c()
        ib = self.batch()
        args = (ctx.h, C.byref(ib), ptr(idx), ptr(x), C.c_int64(x.stride(0)), n, L, C.byref(eyes), C.byref(p))
        if warp is not None:
            _check(ctx.h, _capi.lib().sd_hog_debug_warped(*args, ptr(warp), ptr(geo), ptr(patches), ptr(bins)))
        else:
            _check(ctx.h, _capi.lib().sd_hog_debug(*args, ptr(geo), ptr(patches), ptr(bins)))
        return geo, patches, bins


# ------------------------------------------------------------------------------------------------
# projections that run on the device
# ------------------------------------------------------------------------------------------------
class DeviceProjection:
    """A projection h that writes the feature rows of many samples at once on the device (a pose model's 3-D projection, random
    or pixel features, a torch module).  The optimiser runs its levels through sd_train_level_projected /
    sd_apply_level_projected: in chunks (rows_per_chunk), on several ranks (comm / group / distributed_solve), with the rank
    diagnostic -- everything a HogTransform level has.  Subclass it, or provide the two methods:

      feature_length(level) -> int                  D of the level
      project(x, level, first_row, out) -> None     x: (rows, P) CUDA tensor view of this rank's parameter rows
                                                    [first_row, first_row + rows); out: (rows, D) view into the chunk buffer
                                                    (rows are further apart than D): write the features into it

    project runs with the library's stream as torch's current stream and must queue its work there.  In training it is called
    twice for every chunk but the last (once for the Gram, once for the update), so it must be deterministic.  An exception it
    raises fails the level and is re-raised from train() / test()."""

    def feature_length(self, level: int) -> int:
        raise NotImplementedError

    def project(self, x: torch.Tensor, level: int, first_row: int, out: torch.Tensor) -> None:
        raise NotImplementedError


def _is_device_projection(h) -> bool:
    return callable(getattr(h, "project", None)) and callable(getattr(h, "feature_length", None))


class _LevelProjection:
    """The sd_level_projection of a DeviceProjection on one level.  The callback hands project() views of the optimiser's own
    parameter tensor x and chunk buffer buf (the library passes pointers into exactly those), under the context's stream; an
    exception is kept for raise_error().  close() right after the C call drops the callback and with it every reference to x and
    buf, so the chunk buffer is freed with the optimiser's own reference (the callback does not refer back to this object: no
    cycle waits for the garbage collector)."""

    def __init__(self, ctx: Context, h, level: int, x: torch.Tensor, buf: torch.Tensor):
        errors = self._errors = []
        D = int(h.feature_length(level))
        sp = _capi.lib().sd_ctx_stream(ctx.h) or 0
        current = torch.cuda.current_stream(ctx.device)
        stream = current if current.cuda_stream == sp else torch.cuda.ExternalStream(sp, device=torch.device("cuda", ctx.device))

        def fn(user, c, lvl, d_x, ldx, first_row, rows, d_out, ld):
            try:
                xs, out = x[first_row:first_row + rows], buf[:rows, :D]
                if (d_x or 0) != xs.data_ptr() or ldx != x.stride(0) or (d_out or 0) != out.data_ptr() or ld != buf.stride(0):
                    raise RuntimeError("projection callback: the level passed rows outside the optimiser's tensors")
                with torch.cuda.stream(stream):
                    h.project(xs, lvl, first_row, out)
                return 0
            except BaseException as e:   # noqa: B902 -- nothing may unwind through the C frames; re-raised by raise_error
                errors.append(e)
                return 1

        self._fn = _capi.ProjectFn(fn)                                      # alive as long as the descriptor
        self.c = _capi.LevelProjectionC(self._fn, None, level, D)

    def close(self) -> None:
        self._fn = self.c = None

    def raise_error(self) -> None:
        if self._errors:
            raise self._errors.pop()


# ------------------------------------------------------------------------------------------------
# projections that run on the host
# ------------------------------------------------------------------------------------------------
class HostProjection:
    """A projection h that writes the feature rows of many samples at once on the host (numpy features, CPU descriptors, the
    reference's own functors through RowwiseProjection).  The optimiser runs its levels through sd_train_level_host_projected /
    sd_apply_level_host_projected: the library calls project_host batch by batch into pinned staging and uploads each batch
    while the next one is filled, so the host works while the GPU does; in chunks (rows_per_chunk), on several ranks (comm /
    group / distributed_solve), with the rank diagnostic -- everything a DeviceProjection level has.  Subclass it, or provide the
    two methods:

      feature_length(level) -> int                  D of the level
      project_host(x, level, first_row, out) -> None
                                                    x: (rows, P) read-only float32 numpy view of this rank's parameter rows
                                                    [first_row, first_row + rows); out: (rows, D) float32 numpy view into a
                                                    pinned staging half (rows are further apart than D): write the features into it

    stage_half_bytes (optional attribute): bytes of one staging half, 0 = the library's default (48 MB); a batch is as many rows
    as fit one half, at least one.  In training project_host is called twice for every chunk but the last (once for the Gram,
    once for the update), so it must be deterministic.  It runs on the thread that called train() / test().  An exception it
    raises fails the level and is re-raised from train() / test()."""

    stage_half_bytes = 0

    def feature_length(self, level: int) -> int:
        raise NotImplementedError

    def project_host(self, x: np.ndarray, level: int, first_row: int, out: np.ndarray) -> None:
        raise NotImplementedError


class RowwiseProjection(HostProjection):
    """A per-row projection functor h(x_row, level, index) -> row / float (the reference's ProjectionFunction, e.g. the pose
    example's) as a HostProjection: project_host calls h row by row, exactly as the plain-functor route does, so the level gets
    the same feature rows -- but through the level pipeline (chunks, several ranks, the host filling rows while the GPU works).
    feature_length: D of every level, or a sequence with one D per level."""

    def __init__(self, h: Callable, feature_length):
        self.h = h
        self.lengths = feature_length

    def feature_length(self, level: int) -> int:
        return int(self.lengths if np.isscalar(self.lengths) else self.lengths[level])

    def project_host(self, x: np.ndarray, level: int, first_row: int, out: np.ndarray) -> None:
        D = out.shape[1]
        for i in range(x.shape[0]):
            row = np.atleast_1d(np.asarray(self.h(x[i].copy(), level, first_row + i), dtype=np.float32)).ravel()
            if row.size != D:
                raise ValueError(f"RowwiseProjection: h returned {row.size} values for row {first_row + i}, feature_length is {D}")
            out[i] = row


def _is_host_projection(h) -> bool:
    return callable(getattr(h, "project_host", None)) and callable(getattr(h, "feature_length", None))


class _LevelHostProjection:
    """The sd_level_host_projection of a HostProjection on one level.  The callback hands project_host() numpy views of the
    pinned copy of the parameter rows and of the staging half; an exception is kept for raise_error().  As for
    _LevelProjection, close() right after the C call drops the callback, and the callback does not refer back to this object."""

    def __init__(self, h, level: int):
        errors = self._errors = []
        D = int(h.feature_length(level))

        def fn(user, lvl, h_x, ldx, first_row, rows, h_out, ld_out):
            try:
                x = np.ctypeslib.as_array((C.c_float * (rows * ldx)).from_address(h_x)).reshape(rows, ldx)
                x.flags.writeable = False                                   # the second pass of training reads it again
                out = np.ctypeslib.as_array((C.c_float * (rows * ld_out)).from_address(h_out)).reshape(rows, ld_out)[:, :D]
                h.project_host(x, lvl, first_row, out)
                return 0
            except BaseException as e:   # noqa: B902 -- nothing may unwind through the C frames; re-raised by raise_error
                errors.append(e)
                return 1

        self._fn = _capi.HostProjectFn(fn)                                  # alive as long as the descriptor
        self.c = _capi.LevelHostProjectionC(self._fn, None, level, D, int(getattr(h, "stage_half_bytes", 0) or 0))

    def close(self) -> None:
        self._fn = self.c = None

    def raise_error(self) -> None:
        if self._errors:
            raise self._errors.pop()


# ------------------------------------------------------------------------------------------------
# superviseddescent.hpp: the cascade
# ------------------------------------------------------------------------------------------------
class SupervisedDescentOptimiser:
    """superviseddescent::SupervisedDescentOptimiser<LinearRegressor, Normalisation> (superviseddescent.hpp:85-361).

    projection: a HogTransform or a DeviceProjection (both stay on the device), a HostProjection (rows filled on the host and
    uploaded in a pipeline; RowwiseProjection wraps a per-row functor), or any callable
    h(x_row: np.ndarray, regressor_level: int, sample_index: int) -> row / float, evaluated on the host
    exactly as the reference evaluates user functors (superviseddescent.hpp:178-189).  train / test / predict try them in that
    order: HogTransform, an object with project(), an object with project_host(), a callable.
    """

    def __init__(self, regressors: List[LinearRegressor], normalisation=None, ctx: Optional[Context] = None):
        self.regressors = list(regressors)
        self.normalisation_strategy = normalisation or NoNormalisation()
        self.ctx = ctx
        self.chunk_rows: List[int] = []   # feature rows per chunk of each level of the last train() on the device route

    def _ctx(self) -> Context:
        if self.ctx is None:
            self.ctx = default_context()
        for r in self.regressors:
            if r.ctx is None:
                r.ctx = self.ctx
        return self.ctx

    # -- projection of all rows into an (N, ld) buffer with `extra` spare columns on the right
    def _project(self, h, x: torch.Tensor, level: int, extra: int) -> (torch.Tensor, int):
        ctx = self._ctx()
        n = x.shape[0]
        if isinstance(h, HogTransform):
            D = h.feature_length(level)
            ld = (D + extra + 3) // 4 * 4
            buf = torch.empty((n, ld), dtype=torch.float32, device=x.device)
            h.into(x, level, buf)
            return buf, D
        if isinstance(h, FixedHogTransform):
            D = h.feature_length(x.shape[1] // 2)
            ld = (D + max(extra, 1) + 3) // 4 * 4                 # the kernel's bias lands in the first spare column
            buf = torch.empty((n, ld), dtype=torch.float32, device=x.device)
            h.into(x, buf)
            return buf, D
        xs = x.cpu().numpy()
        rows = [np.atleast_1d(np.asarray(h(xs[i].copy(), level, i), dtype=np.float32)).ravel() for i in range(n)]
        D = rows[0].size
        ld = (D + extra + 3) // 4 * 4
        host = np.zeros((n, ld), dtype=np.float32)
        host[:, :D] = np.stack(rows)
        return _dev(host, ctx), D

    def _chunk_rows(self, rows_per_chunk, frames: Optional[LevelFramesC], n: int, D: int, P: int, comm_h, route: int) -> int:
        """Rows per chunk of a HogTransform, DeviceProjection or HostProjection level (frames None for the last two):
        rows_per_chunk (at most n), or -- None / 0
        -- the most that fit beside the solve and the staging of host frames (sd_level_chunk_rows; memory torch has reserved but
        not handed out counts as free, so a warm caching allocator does not split a level that fits)."""
        if rows_per_chunk:
            return max(1, min(int(rows_per_chunk), n))
        ctx = self._ctx()
        free = _free_device_bytes(ctx.device)
        rows = C.c_int(0)
        _check(ctx.h, _capi.lib().sd_level_chunk_rows(ctx.h, comm_h, C.byref(frames) if frames is not None else None, C.c_int64(n), D, P,
                                                      route, C.c_size_t(free), C.byref(rows)))
        return rows.value

    def train(self, parameters, initialisations, templates, projection, on_training_epoch_callback=None, group=None, comm=None,
              distributed_solve=None, rows_per_chunk=None):
        """superviseddescent.hpp:165-219.  Multi-GPU: pass `comm` (a parallel.Communicator) or a torch.distributed `group`
        (a communicator is then made from it) -- each rank passes its own shard of rows; per level the C ABI does ONE exchange of
        [AtA | Atb] and the solve (SURVEY 8e).  distributed_solve: None = by size (shared CG below parallel.DIST_SOLVE_MIN_D features,
        the distributed factorisation from there), True = reduce-scatter +
        distributed blocked Cholesky, False = all-reduce + replicated solve, "cg" = all-reduce + conjugate gradients shared by the
        ranks.
        A HogTransform projection trains each level with sd_train_level, through a buffer of rows_per_chunk feature rows (None:
        as many as fit on the device, which is all of them whenever the level fits -- then the result is that of one pass over
        all rows).  Templates need the whole level in one chunk.  Frames that stay in host memory are gathered level by level
        (same results), the chunk buffer sized beside the staging they need.  A DeviceProjection trains the same way through
        sd_train_level_projected; an exception its project() raises is re-raised here (on several ranks the other ranks raise
        SdError: the level fails on every rank).  The automatic chunk leaves a DeviceProjection only the library's 512 MB reserve
        for its own temporaries: one that needs more per row passes rows_per_chunk.  A HostProjection trains the same way through
        sd_train_level_host_projected, with the same chunking, ranks and error rules."""
        from . import parallel
        ctx = self._ctx()
        lib = _capi.lib()
        x_gt = _dev(parameters, ctx)
        cur = _dev(initialisations, ctx).clone()
        n, P = cur.shape
        tmpl = _dev(templates, ctx) if templates is not None and np.size(templates) > 0 else None
        own_comm = False
        if comm is None and group is not None:
            comm, own_comm = parallel.Communicator(ctx, group), True
        distributed = comm is not None and comm.size > 1
        n_global = comm.sum_int(n) if distributed else n
        hog = isinstance(projection, HogTransform)
        batched = not hog and _is_device_projection(projection)             # a DeviceProjection
        hosted = not hog and not batched and _is_host_projection(projection)  # a HostProjection
        self.chunk_rows = []                                                 # rows per chunk of each level-call level

        def route(D):
            if not distributed:
                return 0
            if distributed_solve is None:
                return 1 if D >= parallel.DIST_SOLVE_MIN_D else 2          # big systems: distributed factorisation; else shared CG
            return 2 if distributed_solve == "cg" else int(bool(distributed_solve))

        ch = comm.h if distributed else None
        frames = projection.level_frames(n) if hog else None
        for level, reg in enumerate(self.regressors):
            norm = self.normalisation_strategy.c(P // 2)
            lam = C.c_float(0)
            rc_ = reg.regulariser.c()
            qr = getattr(reg.solver, "rank_revealing", False)                # ColPivHouseholderQRSolver: rank of this level's system
            if qr:
                ctx.set_rank_diagnostic(True)                                # before the chunk query: the rank copy counts there
            nxt = torch.empty_like(cur)
            proj = None
            if hog or batched or hosted:                                     # 1)-4) through a buffer of `rows` feature rows
                D = projection.feature_length(level)
                X = torch.empty((D, P), dtype=torch.float32, device=cur.device)
                ld = (D + P + 3) // 4 * 4
                rows = max(n, 1) if tmpl is not None else self._chunk_rows(rows_per_chunk, frames, n, D, P, ch, route(D))
                self.chunk_rows.append(rows)
                buf = torch.empty((rows, ld), dtype=torch.float32, device=cur.device)
                ldt = C.c_int64(tmpl.stride(0) if tmpl is not None else 0)
                if hog:
                    eyes = projection.norm.c()
                    rc = lib.sd_train_level(ctx.h, ch, C.byref(frames), ptr(cur), ptr(x_gt), n, P // 2, C.c_int64(n_global), C.byref(eyes),
                                            C.byref(projection.hog_params[level]), C.byref(norm), ptr(tmpl), ldt, C.byref(rc_), route(D),
                                            ptr(buf), C.c_int64(ld), rows, ptr(X), ptr(nxt), C.byref(lam))
                elif batched:
                    proj = _LevelProjection(ctx, projection, level, cur, buf)
                    rc = lib.sd_train_level_projected(ctx.h, ch, C.byref(proj.c), ptr(cur), ptr(x_gt), n, P, n_global, C.byref(norm),
                                                      ptr(tmpl), ldt, C.byref(rc_), route(D), ptr(buf), ld, rows, ptr(X), ptr(nxt),
                                                      C.byref(lam))
                    proj.close()
                else:
                    proj = _LevelHostProjection(projection, level)
                    rc = lib.sd_train_level_host_projected(ctx.h, ch, C.byref(proj.c), ptr(cur), ptr(x_gt), n, P, n_global, C.byref(norm),
                                                           ptr(tmpl), ldt, C.byref(rc_), route(D), ptr(buf), ld, rows, ptr(X), ptr(nxt),
                                                           C.byref(lam))
                    proj.close()
                del buf
            else:
                A, D = self._project(projection, cur, level, extra=P)         # 1) features (:173-189)
                if tmpl is not None:                                         #    observed = features - templates (:191-197)
                    _check(ctx.h, lib.sd_subtract_templates(ctx.h, ptr(A), C.c_int64(A.stride(0)), ptr(tmpl), C.c_int64(tmpl.stride(0)), n, D))
                Bv = A[:, D:D + P]                                           # 2) b = (x - x_gt) .* norm(x)  (:199-205)
                _check(ctx.h, lib.sd_cascade_targets(ctx.h, ptr(cur), ptr(x_gt), n, P, C.byref(norm), ptr(Bv), C.c_int64(A.stride(0))))
                X = torch.empty((D, P), dtype=torch.float32, device=cur.device)  # 3) learn (:207), on centred rows (sd_centre_features)
                Xc = torch.empty((D, P), dtype=torch.float32, device=cur.device)
                mu = torch.empty(D, dtype=torch.float32, device=cur.device)
                _check(ctx.h, lib.sd_centre_features(ctx.h, ch, ptr(A), C.c_int64(A.stride(0)), n, D, n_global, C.byref(rc_), ptr(mu)))
                rc = lib.sd_learn_centred(ctx.h, ch, ptr(A), C.c_int64(A.stride(0)), ptr(Bv), C.c_int64(A.stride(0)), n, D, P,
                                          C.byref(rc_), n_global, route(D), ptr(mu), ptr(X), ptr(Xc), C.byref(lam))
                if rc == 0:                                                  # 4) x <- x - (A X) .* 1/norm(x) (:209-215); A is centred now: Xc
                    rc = lib.sd_cascade_update(ctx.h, ptr(A), C.c_int64(A.stride(0)), n, D, ptr(Xc), P, ptr(cur), C.byref(norm), ptr(nxt))
                del A, Bv
            if qr:
                ctx.set_rank_diagnostic(False)
                reg.last_rank = ctx.last_rank()
                if 0 <= reg.last_rank < D:
                    _print_rank_warning(reg.last_rank, D)
            if proj is not None:
                proj.raise_error()
            # a factorisation that broke down raises (with the rank in the message): NaN weights would poison the next level
            _check(ctx.h, rc)
            reg.x, reg.last_lambda = X, lam.value                            #    X: the model (for uncentred features)
            cur = nxt
            if on_training_epoch_callback is not None:                       # 5) callback (:217)
                on_training_epoch_callback(comm.allgather_rows(cur) if distributed else cur)
        ctx.sync()                                                           # surfaces flags raised by the projection kernels
        if own_comm:
            comm.close()
        return cur

    def test(self, initialisations, templates, projection, on_regressor_iteration_callback=None, rows_per_chunk=None):
        """superviseddescent.hpp:262-306.  A HogTransform projection runs each level with sd_apply_level, a DeviceProjection
        with sd_apply_level_projected, a HostProjection with sd_apply_level_host_projected, through a buffer of rows_per_chunk
        feature rows (None: as many as fit, as in train())."""
        ctx = self._ctx()
        lib = _capi.lib()
        cur = _dev(initialisations, ctx).clone()
        if cur.dim() == 1:
            cur = cur.reshape(1, -1)
        n, P = cur.shape
        tmpl = _dev(templates, ctx) if templates is not None and np.size(templates) > 0 else None
        hog = isinstance(projection, HogTransform)
        batched = not hog and _is_device_projection(projection)
        hosted = not hog and not batched and _is_host_projection(projection)
        frames = projection.level_frames(n) if hog else None
        for level, reg in enumerate(self.regressors):
            norm = self.normalisation_strategy.c(P // 2)
            nxt = torch.empty_like(cur)
            if hog or batched or hosted:
                D = projection.feature_length(level)
                ld = (D + 3) // 4 * 4
                rows = self._chunk_rows(rows_per_chunk, frames, n, D, P, None, 0)
                buf = torch.empty((rows, ld), dtype=torch.float32, device=cur.device)
                ldt = C.c_int64(tmpl.stride(0) if tmpl is not None else 0)
                if hog:
                    eyes = projection.norm.c()
                    _check(ctx.h, lib.sd_apply_level(ctx.h, C.byref(frames), ptr(cur), n, P // 2, C.byref(eyes), C.byref(projection.hog_params[level]),
                                                     C.byref(norm), ptr(tmpl), ldt, ptr(reg.x), ptr(buf), C.c_int64(ld), rows, ptr(nxt)))
                else:
                    if batched:
                        proj = _LevelProjection(ctx, projection, level, cur, buf)
                        rc = lib.sd_apply_level_projected(ctx.h, C.byref(proj.c), ptr(cur), n, P, C.byref(norm), ptr(tmpl), ldt,
                                                          ptr(reg.x), ptr(buf), ld, rows, ptr(nxt))
                    else:
                        proj = _LevelHostProjection(projection, level)
                        rc = lib.sd_apply_level_host_projected(ctx.h, C.byref(proj.c), ptr(cur), n, P, C.byref(norm), ptr(tmpl), ldt,
                                                               ptr(reg.x), ptr(buf), ld, rows, ptr(nxt))
                    proj.close()
                    proj.raise_error()
                    _check(ctx.h, rc)
                del buf
            else:
                A, D = self._project(projection, cur, level, extra=0)
                if tmpl is not None:
                    _check(ctx.h, lib.sd_subtract_templates(ctx.h, ptr(A), C.c_int64(A.stride(0)), ptr(tmpl), C.c_int64(tmpl.stride(0)), n, D))
                _check(ctx.h, lib.sd_cascade_update(ctx.h, ptr(A), C.c_int64(A.stride(0)), n, D, ptr(reg.x), P, ptr(cur), C.byref(norm), ptr(nxt)))
            cur = nxt
            if on_regressor_iteration_callback is not None:
                on_regressor_iteration_callback(cur)
        return cur

    def predict(self, initialisations, templates, projection, rows_per_chunk=None):
        """superviseddescent.hpp:323-344 (same arithmetic as test(), no callback)."""
        return self.test(initialisations, templates, projection, rows_per_chunk=rows_per_chunk)


# ------------------------------------------------------------------------------------------------
# rcr/model.hpp
# ------------------------------------------------------------------------------------------------
def align_mean(mean, facebox, scaling_x=1.0, scaling_y=1.0, translation_x=0.0, translation_y=0.0) -> np.ndarray:
    """rcr::align_mean (model.hpp:64-76); facebox = (x, y, width, height)."""
    mean = np.ascontiguousarray(mean, dtype=np.float32).ravel()
    out = np.empty_like(mean)
    rc = _capi.lib().sd_align_mean(mean.ctypes.data_as(C.c_void_p), mean.size // 2, int(facebox[0]), int(facebox[1]),
                                   int(facebox[2]), int(facebox[3]), C.c_float(scaling_x), C.c_float(scaling_y),
                                   C.c_float(translation_x), C.c_float(translation_y), out.ctypes.data_as(C.c_void_p))
    if rc:
        raise SdError(rc, "sd_align_mean")
    return out


def perturb(facebox, translation_x: float, translation_y: float, scaling: float = 1.0):
    """perturb() of apps/rcr/rcr-train.cpp:130-146: (x, y, w, h) -> perturbed (x, y, w, h)."""
    out = (C.c_int32 * 4)()
    rc = _capi.lib().sd_perturb_box(int(facebox[0]), int(facebox[1]), int(facebox[2]), int(facebox[3]), C.c_float(translation_x),
                                    C.c_float(translation_y), C.c_float(scaling), out)
    if rc != 0:
        raise SdError(rc, "sd_perturb_box")
    return tuple(int(v) for v in out)


# ibug-68's left-right pairs (1-based ids): jaw 1-17, brows 18-27, nose 32-36, eyes 37-48, outer lip 49-60, inner lip 61-68.  Every
# other id (9, 28-31, 34, 52, 58, 63, 67) is its own mirror.
IBUG68_MIRROR_PAIRS = (tuple((i, 18 - i) for i in range(1, 9)) + tuple((i, 45 - i) for i in range(18, 23)) + ((32, 36), (33, 35))
                       + ((37, 46), (38, 45), (39, 44), (40, 43), (41, 48), (42, 47))
                       + ((49, 55), (50, 54), (51, 53), (56, 60), (57, 59)) + ((61, 65), (62, 64), (66, 68)))
_IBUG68_MIRROR = {**{a: b for a, b in IBUG68_MIRROR_PAIRS}, **{b: a for a, b in IBUG68_MIRROR_PAIRS}}


def mirror_permutation(landmark_ids: Sequence[str]) -> np.ndarray:
    """The left-right correspondence of a model's landmark list under ibug-68 ids (the rcr_22 and ibug-68 lists use them): perm[l]
    is the position of landmark l's mirror partner in the list.  Raises ValueError when an id is not an ibug-68 id or its partner
    is not in the list.  A caller with another id scheme passes its own permutation to mirror_landmarks."""
    ids = [str(i) for i in landmark_ids]
    pos = {v: k for k, v in enumerate(ids)}
    perm = np.empty(len(ids), dtype=np.int64)
    for k, v in enumerate(ids):
        try:
            n = int(v)
        except ValueError:
            raise ValueError(f"mirror_permutation: landmark id {v!r} is not an ibug-68 id") from None
        if not 1 <= n <= 68:
            raise ValueError(f"mirror_permutation: landmark id {v!r} is not an ibug-68 id")
        partner = str(_IBUG68_MIRROR.get(n, n))
        if partner not in pos:
            raise ValueError(f"mirror_permutation: the mirror partner {partner} of landmark {v} is not in the list")
        perm[k] = pos[partner]
    return perm


def mirror_landmarks(x, frame_width, perm) -> np.ndarray:
    """Landmarks of the left-right mirrored frames: x is (N, 2L) float32 rows [x_0 .. x_{L-1}, y_0 .. y_{L-1}] (or one (2L,) row),
    frame_width one width or one per row, perm a landmark permutation (mirror_permutation).  x'[l] = W - 1 - x[perm[l]] and
    y'[l] = y[perm[l]], in float32: the pixel at column u of a frame is at column W - 1 - u of its mirror (np.fliplr, cv::flip)."""
    x = np.asarray(x, dtype=np.float32)
    single = x.ndim == 1
    x = np.atleast_2d(x)
    perm = np.asarray(perm, dtype=np.int64)
    L = x.shape[1] // 2
    if x.shape[1] != 2 * L or perm.shape != (L,):
        raise ValueError("mirror_landmarks: x must be (N, 2L) and perm (L,)")
    w = np.broadcast_to(np.asarray(frame_width, dtype=np.float32).reshape(-1, 1), (x.shape[0], 1))
    out = np.empty_like(x)
    out[:, :L] = (w - np.float32(1)) - x[:, perm]
    out[:, L:] = x[:, L + perm]
    return out[0] if single else out


def mirror_box(box, frame_width: int):
    """The box (x, y, w, h) of a frame as a box of its left-right mirror: (W - x - w, y, w, h)."""
    x, y, w, h = (int(v) for v in box)
    return (int(frame_width) - x - w, y, w, h)


def calculate_normalised_landmark_errors(predictions, groundtruth, model_landmarks: Sequence[str], right_eye_identifiers: Sequence[str],
                                         left_eye_identifiers: Sequence[str], ctx: Optional[Context] = None) -> torch.Tensor:
    """calculate_normalised_landmark_errors() of apps/rcr/rcr-train.cpp:200-212: (N, L) per-landmark L2 errors divided by
    the inter-eye distance of the prediction; the mean over everything is the figure rcr-train prints (:520-524)."""
    ctx = ctx or default_context()
    p = _dev(predictions, ctx)
    g = _dev(groundtruth, ctx)
    n, L = p.shape[0], p.shape[1] // 2
    eyes = InterEyeDistanceNormalisation(model_landmarks, right_eye_identifiers, left_eye_identifiers).c(L)
    out = torch.empty((n, L), dtype=torch.float32, device=p.device)
    _check(ctx.h, _capi.lib().sd_normalised_landmark_errors(ctx.h, ptr(p), C.c_int64(p.stride(0)), ptr(g), C.c_int64(g.stride(0)), n, L,
                                                            C.byref(eyes), ptr(out), C.c_int64(out.stride(0))))
    return out


def _np_ptr(a) -> C.c_void_p:
    return C.c_void_p(0) if a is None else a.ctypes.data_as(C.c_void_p)


def _host_frame(frame):
    """(H, W) / (H, W, C) uint8 numpy array or CPU tensor -> (sd_host_frame, the array that owns the bytes).  The rows keep
    their pitch; the pixels of a row must be packed (copied otherwise)."""
    a = frame.numpy() if isinstance(frame, torch.Tensor) else np.asarray(frame)   # a tensor's numpy() shares (pinned) memory
    if a.dtype != np.uint8:
        a = np.ascontiguousarray(a, dtype=np.uint8)
    if a.ndim not in (2, 3):
        raise ValueError("every frame must be (H, W) or (H, W, 3) uint8")
    ch = 1 if a.ndim == 2 else a.shape[2]
    if a.strides[0] <= 0 or a.strides[1] != ch or (a.ndim == 3 and a.strides[2] != 1):
        a = np.ascontiguousarray(a)
    return HostFrameC(a.ctypes.data, a.shape[1], a.shape[0], a.strides[0], ch), a


def _host_frames(frames):
    """(H, W) / (H, W, 3) uint8 host frames -> (their sd_host_frame records, the arrays that own the bytes the records point
    to)."""
    recs, arrays = [], []
    for f in frames:
        rec, a = _host_frame(f)
        if a.ndim == 3 and a.shape[2] != 3:
            raise ValueError("every frame must be (H, W) uint8 or (H, W, 3) uint8")
        recs.append(rec)
        arrays.append(a)
    return recs, arrays


class detection_model:
    """rcr::detection_model (model.hpp:122-183) resident on the GPU."""

    def __init__(self, handle, ctx: Context):
        self._m = handle
        self.ctx = ctx
        lib = _capi.lib()
        self.num_levels = lib.sd_model_num_levels(handle)
        self.num_landmarks = lib.sd_model_num_landmarks(handle)
        self.landmark_ids = [lib.sd_model_landmark_id(handle, i).decode() for i in range(self.num_landmarks)]

    @classmethod
    def from_parts(cls, optimised_model: SupervisedDescentOptimiser, mean, landmark_ids, hog_params, right_eye_ids,
                   left_eye_ids, ctx: Optional[Context] = None) -> "detection_model":
        """detection_model(optimised_model, mean, landmark_ids, hog_params, right_eye_ids, left_eye_ids) (model.hpp:128)."""
        ctx = ctx or default_context()
        S = len(optimised_model.regressors)
        ws = [np.ascontiguousarray(r.x.cpu().numpy(), dtype=np.float32) for r in optimised_model.regressors]
        wp = (C.c_void_p * S)(*[w.ctypes.data_as(C.c_void_p) for w in ws])
        regs = (RegulariserC * S)(*[r.regulariser.c() for r in optimised_model.regressors])
        hps = (HoGParam * S)(*hog_params)
        mean = np.ascontiguousarray(mean, dtype=np.float32).ravel()
        ids = (C.c_char_p * len(landmark_ids))(*[str(s).encode() for s in landmark_ids])
        rid = (C.c_char_p * len(right_eye_ids))(*[str(s).encode() for s in right_eye_ids])
        lid = (C.c_char_p * len(left_eye_ids))(*[str(s).encode() for s in left_eye_ids])
        h = C.c_void_p()
        _check(ctx.h, _capi.lib().sd_model_create(ctx.h, S, len(landmark_ids), wp, regs, hps, mean.ctypes.data_as(C.c_void_p),
                                                  ids, rid, len(right_eye_ids), lid, len(left_eye_ids), C.byref(h)))
        return cls(h, ctx)

    def get_mean(self) -> np.ndarray:
        out = np.empty(2 * self.num_landmarks, dtype=np.float32)
        _capi.lib().sd_model_get_mean(self._m, out.ctypes.data_as(C.c_void_p))
        return out

    def hog_param(self, level: int) -> HoGParam:
        p = HoGParam()
        _capi.lib().sd_model_hog_param(self._m, level, C.byref(p))
        return p

    def weights(self, level: int) -> np.ndarray:
        r, c = C.c_int(0), C.c_int(0)
        _capi.lib().sd_model_get_weights(self._m, level, None, C.byref(r), C.byref(c))
        out = np.empty((r.value, c.value), dtype=np.float32)
        _capi.lib().sd_model_get_weights(self._m, level, out.ctypes.data_as(C.c_void_p), None, None)
        return out

    def detect(self, image, facebox_or_initialisation) -> np.ndarray:
        """detect(image, facebox) / detect(image, initialisation) (model.hpp:132-157): one frame, grey or colour, returns the 2L
        row."""
        arg = np.asarray(facebox_or_initialisation)
        if arg.size == 4:
            return self.detect_faces([image], [0], boxes=arg.reshape(1, 4))[0]
        return self.detect_faces([image], [0], initialisations=arg.reshape(1, -1))[0]

    def detect_faces(self, frames, face_frame, boxes=None, initialisations=None, warps=None, warp_sizes=None) -> np.ndarray:
        """detect(image, facebox) / detect(image, initialisation) for any number of faces in host frames of any sizes
        (sd_detect_faces_host).  frames: a sequence of (H, W) grey or (H, W, 3) B,G,R uint8 numpy arrays or CPU tensors; face i
        lies in frames[face_frame[i]].  Give exactly one of boxes ((F, 4): x, y, w, h) and initialisations ((F, 2L), e.g. the
        previous video frame's landmarks).  A row pitch other than the row's bytes (strides[0]) is honoured; pinned frames with
        16-byte aligned rows take the zero-copy region-of-interest route.  Returns (F, 2L) landmarks in the order of face_frame.

        warps ((F, 2, 3) float64, optional): face i is a face of V_i = cv2.warpAffine(grey frame, warps[i], warp_sizes[i],
        INTER_LINEAR | WARP_INVERSE_MAP) (default size: its frame's); boxes, initialisations and the landmarks are in V_i's
        coordinates, bit for bit detect on V_i.  The referenced frames are uploaded once (sd_upload_frames) and the warped device
        entry runs (sd_detect_faces_device_warped); V_i is never built."""
        if warps is not None:
            return self._detect_faces_warped(frames, face_frame, boxes, initialisations, warps, warp_sizes)
        recs, keep = [], []
        for f in frames:
            rec, a = _host_frame(f)
            recs.append(rec)
            keep.append(a)                                   # the bytes stay alive until the call returns
        table = (HostFrameC * max(len(recs), 1))(*recs)
        idx = np.ascontiguousarray(face_frame, dtype=np.int32).ravel()
        n = idx.size
        P = 2 * self.num_landmarks
        b = None if boxes is None else np.ascontiguousarray(boxes, dtype=np.int32).reshape(n, 4)
        x0 = None if initialisations is None else np.ascontiguousarray(initialisations, dtype=np.float32).reshape(n, P)
        out = np.empty((n, P), dtype=np.float32)
        _check(self.ctx.h, _capi.lib().sd_detect_faces_host(self.ctx.h, self._m, table, len(recs), _np_ptr(idx), n, _np_ptr(b),
                                                            _np_ptr(x0), _np_ptr(out)))
        return out

    def _detect_faces_warped(self, frames, face_frame, boxes, initialisations, warps, warp_sizes) -> np.ndarray:
        idx = np.ascontiguousarray(face_frame, dtype=np.int64).ravel()
        n = idx.size
        P = 2 * self.num_landmarks
        if (boxes is None) == (initialisations is None):
            raise ValueError("detect_faces: give exactly one of boxes and initialisations")
        if n == 0:
            return np.empty((0, P), dtype=np.float32)
        if idx.min() < 0 or idx.max() >= len(frames):
            raise ValueError("detect_faces: a face refers to a frame that is not in the list")
        used = np.unique(idx)
        recs, keep = _host_frames([frames[f] for f in used])
        dev, ib = _upload_host_frames(recs, self.ctx)
        local = np.searchsorted(used, idx).astype(np.int32)
        if initialisations is None:
            mean = self.get_mean()
            x0 = np.stack([align_mean(mean, b) for b in np.asarray(boxes, dtype=np.int64).reshape(n, 4)])
        else:
            x0 = np.ascontiguousarray(initialisations, dtype=np.float32).reshape(n, P)
        sizes = np.array([(recs[k].width, recs[k].height) for k in local], dtype=np.int64)
        d = f"cuda:{self.ctx.device}"
        table = _warp_table(warps, warp_sizes, sizes, d)
        if table.numel() != n * _WARP_DTYPE.itemsize:
            raise ValueError(f"warps has {table.numel() // _WARP_DTYPE.itemsize} entries for {n} faces")
        fi = torch.from_numpy(local).to(d)
        xd = torch.from_numpy(np.ascontiguousarray(x0, dtype=np.float32)).to(d)
        out = torch.empty((n, P), dtype=torch.float32, device=d)
        _check(self.ctx.h, _capi.lib().sd_detect_faces_device_warped(self.ctx.h, self._m, C.byref(ib), ptr(fi), ptr(table), ptr(xd), n,
                                                                     ptr(out)))
        del dev, keep
        return out.cpu().numpy()

    def detect_batch(self, images: np.ndarray, boxes: np.ndarray) -> np.ndarray:
        """Batched detect(image, facebox) with HOST buffers (copies are part of the call): (count, H, W) grey or
        (count, H, W, 3) colour frames, one face box each."""
        if isinstance(images, torch.Tensor):
            images_np = images.numpy()
        else:
            images_np = np.ascontiguousarray(images, dtype=np.uint8)
        n = images_np.shape[0]
        if images_np.ndim == 4:
            return self.detect_faces(list(images_np), np.arange(n), boxes=boxes)
        _, h, w = images_np.shape
        boxes = np.ascontiguousarray(boxes, dtype=np.int32).reshape(n, 4)
        out = np.empty((n, 2 * self.num_landmarks), dtype=np.float32)
        _check(self.ctx.h, _capi.lib().sd_detect_batch_host(self.ctx.h, self._m, images_np.ctypes.data_as(C.c_void_p), n, w, h,
                                                            images_np.strides[1], boxes.ctypes.data_as(C.c_void_p),
                                                            out.ctypes.data_as(C.c_void_p)))
        return out

    def detect_batch_device(self, images: torch.Tensor, x0: torch.Tensor, image_index=None, warps=None, warp_sizes=None) -> torch.Tensor:
        """Batched detect(image, initialisation), frames and landmarks already resident in HBM.  Face i starts from x0[i] and
        lies in images[image_index[i]] (default: images[i]), so a frame with several faces is resident once.  warps ((n, 2, 3)
        float64, optional; warp_sizes (n, 2), default the frames' size): face i is a face of the V of warps[i] as in detect_faces,
        x0 and the result in V's coordinates."""
        n = x0.shape[0]
        h, w = images.shape[1], images.shape[2]
        ib = ImageBatchC(C.c_void_p(images.data_ptr()), w, h, images.stride(1), images.stride(0), images.shape[0])
        idx = None if image_index is None else torch.as_tensor(image_index, dtype=torch.int32).to(images.device).contiguous()
        out = torch.empty((n, 2 * self.num_landmarks), dtype=torch.float32, device=images.device)
        if warps is not None:
            table = _warp_table(warps, warp_sizes, np.array([(w, h)] * n, dtype=np.int64), images.device)
            if table.numel() != n * _WARP_DTYPE.itemsize:
                raise ValueError(f"warps has {table.numel() // _WARP_DTYPE.itemsize} entries for {n} faces")
            _check(self.ctx.h, _capi.lib().sd_detect_faces_device_warped(self.ctx.h, self._m, C.byref(ib), ptr(idx), ptr(table), ptr(x0),
                                                                         n, ptr(out)))
            return out
        _check(self.ctx.h, _capi.lib().sd_detect_faces_device(self.ctx.h, self._m, C.byref(ib), ptr(idx), ptr(x0), n, ptr(out)))
        return out

    def track_faces(self, frames, face_frame, previous, face_filter, filter_size, cell_size: int, num_bins: int, threshold: float,
                    variant: int = 1, multichannel: bool = False, bilinear_orientations: bool = False, float_frames: bool = False,
                    grey_frames=None) -> "TrackedFaces":
        """One tracking step (sd_track_faces): track t lies in frames[face_frame[t]] and had the landmarks previous[t] ((T, 2L)).
        Each track restarts the cascade from align_mean of track_boxes(previous), scores the box of its new landmarks with the
        face filter (hog_box_scores) and stays alive while that box is valid, its score exceeds threshold and no cascade level had
        an empty patch.  A dead track whose previous box was degenerate keeps its previous landmarks.  frames as hog_dense takes
        them (a CUDA (count, H, W) uint8 tensor in place, or host frames uploaded with colour converted to grey); face_filter a
        HogFilter of train_hog_filter (or a (filter, bias) pair) with filter_size = (fw, fh).  There is no tracker state: drop the
        dead tracks and start new ones from vl_hog_detect boxes.  Returns TrackedFaces of CUDA tensors.

        multichannel, bilinear_orientations and float_frames as vl_hog_detect takes them: a filter trained on colour or float
        frames (train_hog_filter with the same values) scores the boxes on the frames as given (sd_track_faces_images), while the
        cascade reads grey frames: those of 8-bit B, G, R frames converted on the device after one upload, 8-bit grey frames as
        they are, and for float frames or other channel counts grey_frames (frames as detect_faces takes them, of the same sizes)."""
        ctx = self.ctx
        dev = f"cuda:{ctx.device}"
        keep, ib, hi = _track_frames(frames, ctx, multichannel, bilinear_orientations, float_frames, grey_frames, "track_faces")
        P = 2 * self.num_landmarks
        prev = _dev(previous, ctx).reshape(-1, P).contiguous()
        T = prev.shape[0]
        idx = _dev_int32(face_frame, dev).reshape(-1)
        if idx.numel() != T:
            raise ValueError("face_frame and previous must have one entry per track")
        f, fw, fh = _box_filter(face_filter[0], filter_size, num_bins, variant, dev)
        out = TrackedFaces(torch.empty((T, P), dtype=torch.float32, device=dev), torch.empty((T, 4), dtype=torch.int32, device=dev),
                           torch.empty(T, dtype=torch.float32, device=dev), torch.empty(T, dtype=torch.uint8, device=dev))
        lib = _capi.lib()
        call, frames_args = ((lib.sd_track_faces, [C.byref(ib)]) if hi is None else
                             (lib.sd_track_faces_images, [C.byref(ib), C.byref(hi), int(bool(bilinear_orientations))]))
        _check(ctx.h, call(ctx.h, self._m, *frames_args, ptr(idx), ptr(prev), T, ptr(f), fw, fh, C.c_float(float(face_filter[1])),
                           int(cell_size), int(num_bins), int(variant), C.c_float(float(threshold)), ptr(out.landmarks), ptr(out.boxes),
                           ptr(out.scores), ptr(out.alive)))
        return out._replace(alive=out.alive.bool())

    def track_and_detect(self, frames, face_frame, previous, face_filter, filter_size, cell_size: int, num_bins: int,
                         threshold: float, scales, detect_frames, detect_threshold: float, variant: int = 1, pad=(0, 0),
                         nms_overlap: float = 0.5, track_overlap: float = 0.5, max_candidates: int = 4096,
                         max_detections: int = 16, multichannel: bool = False, bilinear_orientations: bool = False,
                         float_frames: bool = False, grey_frames=None) -> "TrackStep":
        """One tracking step that also detects (sd_track_detect_faces).  The T tracks (face_frame, previous) are stepped as
        track_faces steps them.  On each frame of detect_frames (distinct frame indices, in the order given) the face filter runs
        as vl_hog_detect runs it (scales, pad, detect_threshold, nms_overlap, max_candidates, max_detections); a detection is
        dropped when a track of its frame alive after the step overlaps it by IoU > track_overlap, and every other one starts a
        new row: detect_faces from its box, then scored and ended as a track.  Last, within each frame the alive rows are kept
        greedily in the order (old rows first, score descending, row index) unless a kept row overlaps them by IoU >
        track_overlap; track_overlap = 1 neither drops nor merges.  Returns TrackStep of CUDA tensors: rows 0..T-1 are the old
        tracks, rows T.. the num_new new ones.  multichannel, bilinear_orientations, float_frames and grey_frames as track_faces
        takes them: with multichannel the box scores and the detector (vl_hog_detect(multichannel=True, ...)) read the frames as
        given, the cascade their grey (sd_track_detect_faces_images)."""
        ctx = self.ctx
        dev = f"cuda:{ctx.device}"
        keep, ib, hi = _track_frames(frames, ctx, multichannel, bilinear_orientations, float_frames, grey_frames, "track_and_detect")
        P = 2 * self.num_landmarks
        prev = _dev(previous, ctx).reshape(-1, P).contiguous()
        T = prev.shape[0]
        idx = _dev_int32(face_frame, dev).reshape(-1)
        if idx.numel() != T:
            raise ValueError("face_frame and previous must have one entry per track")
        f, fw, fh = _box_filter(face_filter[0], filter_size, num_bins, variant, dev)
        listed = np.ascontiguousarray(detect_frames, dtype=np.int32).ravel()
        sc = np.ascontiguousarray(scales, dtype=np.float64).ravel()
        pad_x, pad_y = (int(v) for v in pad)
        param = _capi.TrackDetectParamC(sc.ctypes.data_as(C.c_void_p), sc.size, pad_x, pad_y, float(detect_threshold),
                                        float(nms_overlap), float(track_overlap), int(max_candidates), int(max_detections))
        R = T + listed.size * max(int(max_detections), 0)
        out = TrackStep(torch.empty((R, P), dtype=torch.float32, device=dev), torch.empty((R, 4), dtype=torch.int32, device=dev),
                        torch.empty(R, dtype=torch.float32, device=dev), torch.empty(R, dtype=torch.uint8, device=dev),
                        torch.empty(R, dtype=torch.int32, device=dev), 0)
        n = C.c_int32(0)
        lib = _capi.lib()
        call, frames_args = ((lib.sd_track_detect_faces, [C.byref(ib)]) if hi is None else
                             (lib.sd_track_detect_faces_images, [C.byref(ib), C.byref(hi), int(bool(bilinear_orientations))]))
        _check(ctx.h, call(ctx.h, self._m, *frames_args, ptr(idx), ptr(prev), T, ptr(f), fw, fh, C.c_float(float(face_filter[1])),
                           int(cell_size), int(num_bins), int(variant), C.c_float(float(threshold)), _np_ptr(listed), listed.size,
                           C.byref(param), ptr(out.landmarks), ptr(out.boxes), ptr(out.scores), ptr(out.alive), ptr(out.frame),
                           C.byref(n)))
        r = T + n.value
        return TrackStep(out.landmarks[:r], out.boxes[:r], out.scores[:r], out.alive[:r].bool(), out.frame[:r], n.value)

    def save(self, filename: str) -> None:
        _check(self.ctx.h, _capi.lib().sd_model_save(self.ctx.h, self._m, filename.encode()))

    def __del__(self):
        try:
            if self._m:
                _capi.lib().sd_model_destroy(self._m)
                self._m = None
        except Exception:
            pass


TrackedFaces = collections.namedtuple("TrackedFaces", "landmarks boxes scores alive")
TrackedFaces.__doc__ = """Result of detection_model.track_faces, CUDA tensors: landmarks (T, 2L) float32, boxes (T, 4) int32 (x, y, w, h:
the track_boxes box of the new landmarks), scores (T,) float32 (its hog_box_scores score, NaN for a degenerate box) and alive (T,)
bool."""

TrackStep = collections.namedtuple("TrackStep", "landmarks boxes scores alive frame num_new")
TrackStep.__doc__ = """Result of detection_model.track_and_detect: rows 0..T-1 are the old tracks, rows T..T+num_new-1 the new ones, as CUDA
tensors landmarks (R, 2L) float32, boxes (R, 4) int32, scores (R,) float32, alive (R,) bool and frame (R,) int32; num_new an int."""


class FaceTracker:
    """The state of a multi-stream face tracker: the live rows' landmarks, frames and integer ids, and the next id.  Each step
    is one track_and_detect call; frames holds one frame per stream, and a stream keeps its frame index from step to step.
    Extra keyword arguments (variant, pad, nms_overlap, track_overlap, max_candidates, max_detections, and multichannel,
    bilinear_orientations, float_frames for a filter trained on colour or float frames) go to track_and_detect."""

    def __init__(self, model: detection_model, face_filter, filter_size, cell_size: int, num_bins: int, threshold: float, scales,
                 detect_threshold: float, **options):
        self.model = model
        self.args = dict(face_filter=face_filter, filter_size=filter_size, cell_size=cell_size, num_bins=num_bins,
                         threshold=threshold, scales=scales, detect_threshold=detect_threshold, **options)
        dev = f"cuda:{model.ctx.device}"
        self.landmarks = torch.empty((0, 2 * model.num_landmarks), dtype=torch.float32, device=dev)
        self.frame = torch.empty(0, dtype=torch.int32, device=dev)
        self.ids = torch.empty(0, dtype=torch.int64, device=dev)
        self.next_id = 0

    def step(self, frames, detect_frames=None, grey_frames=None):
        """Steps every live track on frames and runs the detector on detect_frames (default: the frames without a live track).
        Old rows keep their ids, new rows take fresh ids in row order, and the rows that are not alive are dropped.  grey_frames:
        the cascade's frames, for float frames (see track_faces).  Returns (ids, frame, landmarks, boxes) of the live rows."""
        if detect_frames is None:
            live = set(self.frame.tolist())
            detect_frames = [f for f in range(len(frames)) if f not in live]
        extra = {} if grey_frames is None else {"grey_frames": grey_frames}
        r = self.model.track_and_detect(frames, self.frame, self.landmarks, detect_frames=detect_frames, **extra, **self.args)
        ids = torch.cat([self.ids, torch.arange(self.next_id, self.next_id + r.num_new, device=self.ids.device)])
        self.next_id += r.num_new
        self.ids, self.frame, self.landmarks = ids[r.alive], r.frame[r.alive], r.landmarks[r.alive]
        return self.ids, self.frame, self.landmarks, r.boxes[r.alive]


def _check_float_frames(hi, float_frames: bool) -> None:
    """float32 frames are resized by the float rule, which float_frames=True selects (as vl_hog_pyramid refuses them without)."""
    if hi.dtype == _VL_HOG_DTYPES[torch.float32] and not float_frames:
        raise ValueError("float32 frames need float_frames=True")


def _track_frames(frames, ctx: Context, multichannel: bool, bilinear_orientations: bool, float_frames: bool, grey_frames, fn: str):
    """The frames of a tracking step -> (what owns their device bytes, the grey ImageBatchC the cascade reads, the HogImagesC the
    filter reads or None for grey frames).  Without multichannel the frames are _grey_frames'.  With it they keep their channels
    (_window_frames), and the cascade's grey frames come from grey_frames when given; else from the frames themselves: 8-bit
    B, G, R frames through sd_bgr2gray_images (one upload), 8-bit grey frames read in place.  Other frames need grey_frames."""
    none = lambda w, h: None
    if not multichannel:
        if grey_frames is not None:
            raise ValueError("grey_frames needs multichannel=True (grey frames are the cascade's frames)")
        keep, ib, _ = _window_frames(frames, ctx, none, False, bilinear_orientations, float_frames)
        if ib is None:
            raise ValueError(f"{fn} needs at least one frame")
        return keep, ib, None
    descs = []
    keep, hi, sizes = _window_frames(frames, ctx, none, True, bilinear_orientations, float_frames, descs)
    if hi is None:
        raise ValueError(f"{fn} needs at least one frame")
    _check_float_frames(hi, float_frames)
    if grey_frames is not None:
        gkeep, ib, _ = _grey_frames(grey_frames, ctx, none)
        if ib is None:
            raise ValueError("grey_frames holds no frame")
        return (keep, gkeep), ib, hi
    dev = f"cuda:{ctx.device}"
    if hi.dtype == _VL_HOG_DTYPES[torch.uint8] and hi.channels == 3:
        # sized by sd_bgr2gray_images' stated layout from the host sizes, so the frame table is read back by the conversion only
        nbytes = C.c_size_t(sum(h * _round16(w) for h, w in sizes) + (0 if len(set(sizes)) == 1 else len(sizes) * C.sizeof(FrameC)))
        buf = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
        ib = ImageBatchC()
        _check(ctx.h, _capi.lib().sd_bgr2gray_images(ctx.h, C.byref(hi), ptr(buf), C.byref(nbytes), C.byref(ib)))
        return (keep, buf), ib, hi
    if hi.dtype == _VL_HOG_DTYPES[torch.uint8] and hi.channels == 1:
        if all(d.pixel_stride == 1 for d in descs):          # grey frames read in place, through their own descriptors
            if not hi.d_frames:
                f = hi.frame
                return keep, ImageBatchC(C.c_void_p(hi.d_data + f.offset), f.width, f.height, f.row_stride, hi.image_stride, hi.count), hi
            table = _device_table([FrameC(d.width, d.height, d.row_stride, 0, d.offset) for d in descs], dev)
            ib = ImageBatchC()
            ib.d_data, ib.count, ib.d_frames = hi.d_data, hi.count, table.data_ptr()
            return (keep, table), ib, hi
        # a batch whose grey pixels are not contiguous along rows (a strided view): one contiguous copy on the device
        g = keep.reshape(keep.shape[:3]).contiguous()
        n, h, w = g.shape
        return (keep, g), ImageBatchC(C.c_void_p(g.data_ptr()), w, h, g.stride(1), g.stride(0), n), hi
    raise ValueError(f"{fn}: the cascade reads grey 8-bit frames; pass them as grey_frames= for float frames or frames of "
                     f"{hi.channels} channels")


def _dev_int32(a, dev) -> torch.Tensor:
    return _tensor(np.asarray(a, dtype=np.int32) if not isinstance(a, torch.Tensor) else a).to(dev, torch.int32).contiguous()


def _box_filter(filt, filter_size, num_bins: int, variant: int, dev):
    """A (dd, fh, fw) or (1, dd, fh, fw) float32 filter -> (its contiguous device tensor, fw, fh), checked against filter_size."""
    f = _tensor(filt).to(dev, torch.float32)
    if f.dim() == 4 and f.shape[0] == 1:
        f = f[0]
    fw, fh = (int(v) for v in filter_size)
    dd = _hog_dims(num_bins, variant)
    if tuple(f.shape) != (dd, fh, fw):
        raise ValueError(f"the filter must be ({dd}, {fh}, {fw}) for filter_size ({fw}, {fh}), got {tuple(f.shape)}")
    return f.contiguous(), fw, fh


def track_boxes(landmarks, model: detection_model):
    """The face box of each row of landmarks ((T, 2L), [x.., y..]) under the model's mean (sd_track_boxes): the integer box B
    whose align_mean has the landmarks' enclosing box, the inverse of align_mean at scaling 1 and translation 0.  Returns (boxes
    (T, 4) int32, valid (T,) bool) CUDA tensors; an invalid (degenerate) row has the box (0, 0, 0, 0)."""
    ctx = model.ctx
    x = _dev(landmarks, ctx).reshape(-1, 2 * model.num_landmarks).contiguous()
    T = x.shape[0]
    boxes = torch.empty((T, 4), dtype=torch.int32, device=x.device)
    valid = torch.empty(T, dtype=torch.uint8, device=x.device)
    _check(ctx.h, _capi.lib().sd_track_boxes(ctx.h, model._m, ptr(x), T, ptr(boxes), ptr(valid)))
    return boxes, valid.bool()


def hog_box_scores(frames, box_frame, boxes, filter, bias: float, cell_size: int, num_bins: int, variant: int = 1,
                   ctx: Optional[Context] = None, multichannel: bool = False, bilinear_orientations: bool = False,
                   float_frames: bool = False) -> torch.Tensor:
    """A HOG filter's score at each box (sd_hog_box_scores): box i ((x, y, w, h) of frames[box_frame[i]]) with one cell of
    context on every side, zero outside the frame, resized by cv::resize INTER_LINEAR to (fw + 2) x (fh + 2) cells of cell_size
    px, its hog_dense features scored by vl_hog_correlate with the filter ((dd, fh, fw)) and bias at every one of the 3 x 3
    positions; the box's score is the largest (a NaN never is).  frames as hog_dense takes them.  multichannel,
    bilinear_orientations and float_frames as vl_hog_detect takes them (sd_hog_box_scores_images): each channel of the context
    rectangle is resized on its own by the rule of the frames' dtype and the crop's features are vl_hog's.  Returns (n,) float32
    on the device."""
    ctx = ctx or default_context()
    dev = f"cuda:{ctx.device}"
    keep, ib, sizes = _window_frames(frames, ctx, lambda w, h: None, multichannel, bilinear_orientations, float_frames)
    if ib is None:
        raise ValueError("hog_box_scores needs at least one frame")
    if multichannel:
        _check_float_frames(ib, float_frames)
    f = _tensor(filter)
    f, fw, fh = _box_filter(f, (f.shape[-1], f.shape[-2]), num_bins, variant, dev)
    bf = _dev_int32(box_frame, dev).reshape(-1)
    bx = _dev_int32(boxes, dev).reshape(-1, 4)
    n = bf.numel()
    if bx.shape[0] != n:
        raise ValueError("box_frame and boxes must have one entry per box")
    out = torch.empty(n, dtype=torch.float32, device=dev)
    lib = _capi.lib()
    call, frames_args = ((lib.sd_hog_box_scores_images, [C.byref(ib), int(bool(bilinear_orientations))]) if multichannel else
                         (lib.sd_hog_box_scores, [C.byref(ib)]))
    _check(ctx.h, call(ctx.h, *frames_args, ptr(bf), ptr(bx), n, ptr(f), fw, fh, C.c_float(float(bias)), int(cell_size), int(num_bins),
                       int(variant), ptr(out)))
    return out


FaceChips = collections.namedtuple("FaceChips", "chips chip_to_frame frame_to_chip valid")
FaceChips.__doc__ = """Result of face_chips, CUDA tensors: chips (n, h, w, C) in the frames' dtype (channels last), chip_to_frame and
frame_to_chip (n, 2, 3) float64 (the fitted similarity [a, -b, tx; b, a, ty] and its inverse) and valid (n,) bool.  An invalid
face has a zero chip and zero transforms."""


def _chip_size(size):
    w, h = (int(size), int(size)) if np.isscalar(size) else (int(v) for v in size)
    return w, h


def face_chip_template(model: detection_model, size, padding: float = 0.25, landmarks=None) -> np.ndarray:
    """The default template of face_chips (sd_face_chip_template): landmark k of the model's mean goes to ((m_x[k] + 0.5 +
    padding) / (1 + 2 padding)) * width, and y alike with height, so align_mean's unit box grown by padding on each side fills a
    chip of size ((w, h) or one side).  landmarks: the indices to place (default all).  Returns (n, 2) float64."""
    w, h = _chip_size(size)
    idx = None if landmarks is None else np.ascontiguousarray(landmarks, dtype=np.int32).ravel()
    n = model.num_landmarks if idx is None else idx.size
    out = np.empty((n, 2), dtype=np.float64)
    rc = _capi.lib().sd_face_chip_template(model._m, w, h, C.c_double(float(padding)), n, None if idx is None else _np_ptr(idx),
                                           _np_ptr(out))
    if rc:
        raise SdError(rc, "sd_face_chip_template: bad arguments (size >= 1, padding > -0.5 and finite, indices in range)")
    return out


def face_chips(frames, face_frame, landmarks, size, template, landmark_index=None, channels_last: bool = False,
               ctx: Optional[Context] = None) -> FaceChips:
    """Aligned face chips (sd_face_chips): for face i, the least-squares similarity from template ((n, 2) chip pixels) to its
    landmarks landmark_index (default all) of landmarks[i] ((N, 2L) float32, [x.., y..]), and the chip of size ((w, h) or one
    side) cut from frames[face_frame[i]] as cv2.warpAffine(frame, M, (w, h), INTER_LINEAR | WARP_INVERSE_MAP, BORDER_CONSTANT, 0)
    does, bit for bit.  frames as vl_hog takes them (uint8 or float32, 1..16 channels; CUDA tensors read in place, host frames
    uploaded once; channels_last for (H, W, C) frames); face_frame and landmarks may be CUDA tensors, e.g. a TrackStep's frame
    and landmarks.  Returns FaceChips."""
    ctx = ctx or default_context()
    dev = f"cuda:{ctx.device}"
    w, h = _chip_size(size)
    keep, ib, _ = _hog_images(frames, channels_last, ctx, lambda fw, fh: None)
    if ib is None:
        raise ValueError("face_chips needs at least one frame")
    ff = _dev_int32(face_frame, dev).reshape(-1)
    x = _dev(landmarks, ctx)
    if x.dim() != 2 or x.shape[1] % 2 or x.shape[0] != ff.numel():
        raise ValueError("landmarks must be (N, 2L), one row per entry of face_frame")
    if x.stride(1) != 1:
        x = x.contiguous()
    L = x.shape[1] // 2
    idx = np.ascontiguousarray(np.arange(L) if landmark_index is None else landmark_index, dtype=np.int32).ravel()
    tm = np.ascontiguousarray(template, dtype=np.float64)
    if tm.shape != (idx.size, 2):
        raise ValueError(f"template must be ({idx.size}, 2), one point per used landmark, got {tm.shape}")
    n = ff.numel()
    chips = torch.empty((n, h, w, ib.channels), dtype=torch.uint8 if ib.dtype == _VL_HOG_DTYPES[torch.uint8] else torch.float32,
                        device=dev)
    c2f = torch.empty((n, 2, 3), dtype=torch.float64, device=dev)
    f2c = torch.empty((n, 2, 3), dtype=torch.float64, device=dev)
    valid = torch.empty(n, dtype=torch.uint8, device=dev)
    p = FaceChipParamC(w, h, idx.size, _np_ptr(idx), _np_ptr(tm))
    _check(ctx.h, _capi.lib().sd_face_chips(ctx.h, C.byref(ib), ptr(ff), ptr(x), x.stride(0) if n else 2 * L, n, L, C.byref(p),
                                            ptr(chips), ptr(c2f), ptr(f2c), ptr(valid)))
    return FaceChips(chips, c2f, f2c, valid.bool())


def load_detection_model(filename: str, ctx: Optional[Context] = None) -> detection_model:
    """rcr::load_detection_model (model.hpp:192-205)."""
    ctx = ctx or default_context()
    h = C.c_void_p()
    _check(ctx.h, _capi.lib().sd_model_load(ctx.h, filename.encode(), C.byref(h)))
    return detection_model(h, ctx)


def save_detection_model(model: detection_model, filename: str) -> None:
    """rcr::save_detection_model (model.hpp:214-219)."""
    model.save(filename)


def vl_hog_polar(modulus, angle, cell_size: int, num_bins: int, variant: int = 1, directed: bool = True,
                 bilinear_orientations: bool = False, ctx: Optional[Context] = None):
    """VLFeat HOG of gradient fields the caller computed (vl_hog_new(variant, num_bins) +
    vl_hog_set_use_bilinear_orientation_assignments(bilinear_orientations) + vl_hog_put_polar_field(modulus, angle, directed,
    cell_size) + vl_hog_extract) on the device, in VLFeat's planar layout [dd][hogH][hogW] with x fastest.

    modulus, angle: float32 fields, paired element by element -- two arrays or tensors (count, H, W) of one shape, or two lists
    of (H, W) fields of any sizes.  angle is in radians, measured from the x axis towards y (rows grow downwards); it is taken
    modulo 2 pi (directed) or pi.  Every pixel votes, the border included; a modulus <= 0 or a non-finite angle does not.
    CUDA tensors of one device and equal strides are read in place; anything else is made contiguous and uploaded.
    bilinear_orientations: every pixel votes into its two nearest orientation bins.  variant: 1 = UoCTTI (dd = 3K + 4),
    0 = Dalal-Triggs (dd = 4K).  Returns one (count, dd, hogH, hogW) float32 CUDA tensor when all fields have one size, else a
    list of (dd, hogH, hogW) tensors.  ValueError for fields that are not float32, not of the shapes above, or not paired."""
    ctx = ctx or default_context()
    dev = torch.device(f"cuda:{ctx.device}")
    lib = _capi.lib()

    def checked(m, a, dims):
        m, a = _tensor(m), _tensor(a)
        if m.dtype != torch.float32 or a.dtype != torch.float32:
            raise ValueError("modulus and angle must be float32")
        if m.dim() != dims or tuple(m.shape) != tuple(a.shape):
            raise ValueError(f"modulus and angle must be {'(count, H, W)' if dims == 3 else '(H, W)'} fields of one shape")
        return m, a

    fb = HogPolarFieldsC()
    fb.d_frames = None
    if isinstance(modulus, (list, tuple)) or isinstance(angle, (list, tuple)):
        if not (isinstance(modulus, (list, tuple)) and isinstance(angle, (list, tuple))) or len(modulus) != len(angle):
            raise ValueError("modulus and angle must both be lists of one length")
        pairs = [checked(m, a, 2) for m, a in zip(modulus, angle)]
        if not pairs:
            return []
        sizes = [tuple(m.shape) for m, _ in pairs]
        for h, w in set(sizes):
            hog_dense_shape(w, h, cell_size, num_bins, variant)   # refuse before the upload
        keep_m, offsets = _pack([m for m, _ in pairs], dev)
        keep_a, _ = _pack([a for _, a in pairs], dev)
        descs = [HogImageC(w, h, o, w, 1, 0) for (h, w), o in zip(sizes, offsets)]
        fb.count = len(pairs)
        if len(set(sizes)) == 1:
            fb.frame, fb.image_stride = descs[0], sizes[0][0] * sizes[0][1]
        else:
            keep_table = _device_table(descs, dev)
            fb.d_frames = keep_table.data_ptr()
    else:
        m, a = checked(modulus, angle, 3)
        if not (m.device == dev and a.device == dev and m.stride() == a.stride()):
            m, a = m.contiguous().to(dev), a.contiguous().to(dev)
        keep_m, keep_a = m, a
        n, h, w = m.shape
        fb.count, fb.frame, fb.image_stride = n, HogImageC(w, h, 0, m.stride(1), m.stride(2), 0), m.stride(0)
        sizes = [(h, w)] * n
    fb.d_modulus, fb.d_angle = keep_m.data_ptr(), keep_a.data_ptr()
    flags = (int(cell_size), int(num_bins), int(variant), int(bool(directed)), int(bool(bilinear_orientations)))
    return _dense_results(ctx, sizes, None if fb.d_frames else (fb.frame.height, fb.frame.width), cell_size, num_bins, variant,
                          lambda out, offsets: _check(ctx.h, lib.sd_hog_dense_polar(ctx.h, C.byref(fb), *flags, ptr(out), ptr(offsets))))


GLYPH_SIZE = 21     # SD_HOG_GLYPH_SIZE: pixels per side of a rendered cell (hog.c:183)


def _hog_dims(num_bins: int, variant: int) -> int:
    if variant not in (0, 1) or not 1 <= int(num_bins) <= 16:
        raise ValueError(f"num_bins must be in 1..16 and variant 0 or 1 (got {num_bins}, {variant})")
    return 3 * int(num_bins) + 4 if variant == 1 else 4 * int(num_bins)


def vl_hog_permutation(variant: int, num_bins: int) -> np.ndarray:
    """vl_hog_get_permutation of vl_hog_new(variant, num_bins): int64 array of dd entries with
    flipped[i] = features[perm[i]] for the features of the left-right mirrored image.  Host only."""
    dd = _hog_dims(num_bins, variant)
    out = np.zeros(dd, np.int64)
    _check(None, _capi.lib().sd_hog_permutation(int(num_bins), int(variant), C.c_void_p(out.ctypes.data)))
    return out


def vl_hog_glyphs(num_bins: int, transposed: bool = False) -> np.ndarray:
    """The glyphs of vl_hog_new(.., num_bins, transposed): a (num_bins, 21, 21) float32 array of 0 and 1, glyph k at [k]
    (row-major; transposed=True gives hog.c's column-major glyphs).  Host only."""
    _hog_dims(num_bins, 1)
    out = np.zeros((int(num_bins), GLYPH_SIZE, GLYPH_SIZE), np.float32)
    _check(None, _capi.lib().sd_hog_glyphs(int(num_bins), int(bool(transposed)), C.c_void_p(out.ctypes.data)))
    return out


def _hog_grids(features, num_bins: int, variant: int, out_size, ctx: Context, zero: bool):
    """The planar features of vl_hog_render / vl_hog_flip -- a (B, dd, h, w) batch or a list of (dd, h, w) grids -> (grids
    struct, device tensors it points to, result buffer, results): a (B,) + out_size(h, w) tensor, or a list of out_size(h, w)
    tensors, whose descriptors hold their offsets.  An empty list gives a count of 0 and no results."""
    dd = _hog_dims(num_bins, variant)
    dev = f"cuda:{ctx.device}"
    g = HogGridsC()
    g.d_grids = None
    if isinstance(features, (list, tuple)):
        grids = [_tensor(f) for f in features]
        if any(f.dtype != torch.float32 for f in grids):
            raise ValueError("features must be float32")
        if any(f.dim() != 3 or f.shape[0] != dd for f in grids):
            raise ValueError(f"every grid must be (dd, h, w) with dd = {dd}")
        g.count = len(grids)
        if not grids:
            return g, (), None, []
        sizes = [tuple(f.shape[1:]) for f in grids]
        keep, offsets = _pack(grids, dev)
        out, out_offsets, results = _results([out_size(h, w) for h, w in sizes], dev, zero)
        keep_table = _device_table([HogGridC(w, h, o, oo) for (h, w), o, oo in zip(sizes, offsets, out_offsets)], dev)
        g.d_features, g.d_grids = keep.data_ptr(), keep_table.data_ptr()
        return g, (keep, keep_table), out, results
    t = _tensor(features)
    if t.dtype != torch.float32:
        raise ValueError("features must be float32")
    if t.dim() != 4 or t.shape[1] != dd:
        raise ValueError(f"features must be (B, dd, h, w) with dd = {dd}, or a list of (dd, h, w) grids")
    keep = t.to(dev).contiguous()
    b, _, h, w = keep.shape
    g.d_features, g.count, g.width, g.height = keep.data_ptr(), b, w, h
    out, _, results = _results((b,) + tuple(out_size(h, w)), dev, zero)
    return g, (keep,), out, results


def vl_hog_render(features, num_bins: int, variant: int = 1, ctx: Optional[Context] = None):
    """vl_hog_render of planar HOG features on the device (sd_hog_render): a (B, dd, h, w) batch, or a list of (dd, h, w)
    grids of any sizes, each rendered into a fresh zeroed image of (h * 21, w * 21) floats -- cell (x, y) as the 21 x 21 glyph
    tile at (21 y, 21 x), every orientation's bar weighted by the sum of its planes, clamped to the cell's weight range.
    Returns a (B, h * 21, w * 21) float32 CUDA tensor, or a list of (h * 21, w * 21) tensors."""
    ctx = ctx or default_context()
    g, keep, out, results = _hog_grids(features, num_bins, variant, lambda h, w: (h * GLYPH_SIZE, w * GLYPH_SIZE), ctx, zero=True)
    if g.count:
        _check(ctx.h, _capi.lib().sd_hog_render(ctx.h, C.byref(g), int(num_bins), int(variant), 0, ptr(out)))
    return results


def vl_hog_flip(features, num_bins: int, variant: int = 1, ctx: Optional[Context] = None):
    """Left-right flip of planar HOG features on the device (sd_hog_relayout): the features of the mirrored image,
    out[i][y][x] = features[perm[i]][y][w - 1 - x] with perm = vl_hog_permutation(variant, num_bins).  features: a
    (B, dd, h, w) batch or a list of (dd, h, w) grids; returns the same shapes as fresh CUDA tensors."""
    ctx = ctx or default_context()
    g, keep, out, results = _hog_grids(features, num_bins, variant, lambda h, w: (_hog_dims(num_bins, variant), h, w), ctx,
                                       zero=False)
    if g.count:
        _check(ctx.h, _capi.lib().sd_hog_relayout(ctx.h, C.byref(g), int(num_bins), int(variant), 1, 0, ptr(out)))
    return results


# ------------------------------------------------------------------------------------------------
# HOG pyramids and filters: the two batched primitives of a sliding-window detector
# ------------------------------------------------------------------------------------------------
def hog_pyramid_shape(width: int, height: int, scale: float, cell_size: int, num_bins: int, variant: int = 1):
    """((level_w, level_h), (dd, hogH, hogW)) of a width x height frame at scale (sd_hog_pyramid_shape); hogH = hogW = 0 for an
    empty level.  SdError for an invalid scale or configuration."""
    o = [C.c_int() for _ in range(5)]
    rc = _capi.lib().sd_hog_pyramid_shape(int(width), int(height), float(scale), int(cell_size), int(num_bins), int(variant),
                                          *[C.byref(v) for v in o])
    if rc:
        raise SdError(rc, f"invalid HOG pyramid level: {width} x {height} px at scale {scale}, cell_size {cell_size}, num_bins "
                          f"{num_bins}, variant {variant} (scales finite and in (0, 4], cell_size 1..32, num_bins 1..16)")
    lw, lh, w, h, d = (v.value for v in o)
    return (lw, lh), (d, h, w)


def _window_frames(frames, ctx: Context, check, multichannel: bool, bilinear_orientations: bool, float_frames: bool, frames_out=None):
    """The frames of vl_hog_pyramid and train_hog_filter -> (owner, batch, sizes): _hog_images' (channels last) with
    multichannel, _grey_frames' without.  bilinear_orientations and float_frames need multichannel, and float_frames float32
    frames."""
    if bilinear_orientations and not multichannel:
        raise ValueError("bilinear_orientations needs multichannel=True (grey frames pass as they are)")
    if float_frames and not multichannel:
        raise ValueError("float_frames needs multichannel=True (float frames keep their channels)")
    return _hog_images(frames, True, ctx, check, float_frames, frames_out) if multichannel else _grey_frames(frames, ctx, check)


def vl_hog_pyramid(frames, scales, cell_size: int, num_bins: int, variant: int = 1, ctx: Optional[Context] = None,
                   multichannel: bool = False, bilinear_orientations: bool = False, float_frames: bool = False):
    """Dense HOG of every frame at every scale in one call (sd_hog_pyramid): level s of a W x H frame is the frame resized by
    cv::resize INTER_LINEAR to floor(W * s + 0.5) x floor(H * s + 0.5), and its features are hog_dense's of that level.

    frames: as hog_dense takes them: colour frames are converted to grey.  multichannel=True keeps the channels
    (sd_hog_pyramid_images): frames are uint8, channels last -- a host or CUDA (count, H, W) or (count, H, W, C) array or tensor
    (CUDA tensors read in place through their strides), or a list of (H, W) or (H, W, C) frames of any sizes with one C -- each
    channel is resized on its own, and at each pixel the channel with the largest gradient votes, as vl_hog does;
    bilinear_orientations (multichannel only): every pixel votes into its two nearest orientation bins.  float_frames
    (multichannel only, sd_hog_pyramid_float): the frames are float32 in the same layouts, each channel resized by
    cv::resize's float INTER_LINEAR rule (include/sd_b200.h), its values and range taken as given.  Returns (features,
    sizes): features[f][s] is a (dd, hogH, hogW) float32 CUDA view into one buffer, or None for an empty level (smaller than
    4 px or than half a cell); sizes[f][s] = (level_w, level_h)."""
    ctx = ctx or default_context()
    scales = [float(s) for s in scales]
    if not scales:
        raise ValueError("vl_hog_pyramid needs at least one scale")

    def check(w, h):
        for s in scales:
            hog_pyramid_shape(w, h, s, cell_size, num_bins, variant)

    keep, ib, sizes = _window_frames(frames, ctx, check, multichannel, bilinear_orientations, float_frames)
    if not sizes:
        return [], []
    levels = [[hog_pyramid_shape(w, h, s, cell_size, num_bins, variant) for s in scales] for h, w in sizes]
    dev = f"cuda:{ctx.device}"
    out, offsets, feats = _results([shape if shape[1] else None for row in levels for _, shape in row], dev)
    d_off = torch.tensor(offsets, dtype=torch.int64, device=dev)
    h_scales = (C.c_double * len(scales))(*scales)
    if multichannel:
        call = _capi.lib().sd_hog_pyramid_float if float_frames else _capi.lib().sd_hog_pyramid_images
        _check(ctx.h, call(ctx.h, C.byref(ib), h_scales, len(scales), int(cell_size), int(num_bins), int(variant),
                           int(bool(bilinear_orientations)), ptr(out), ptr(d_off)))
    else:
        _check(ctx.h, _capi.lib().sd_hog_pyramid(ctx.h, C.byref(ib), h_scales, len(scales), int(cell_size), int(num_bins),
                                                 int(variant), ptr(out), ptr(d_off)))
    S = len(scales)
    return [feats[i:i + S] for i in range(0, len(feats), S)], [[lv for lv, _ in row] for row in levels]


def vl_hog_correlate(maps, filters, num_bins: int, variant: int = 1, bias=None, pad=(0, 0), ctx: Optional[Context] = None):
    """Scores of a bank of HOG filters over a list of HOG grids (sd_hog_correlate):
        S[q, y, x] = bias[q] + sum_{c, dy, dx} filters[q, c, dy, dx] * M[c, y + dy - pad_y, x + dx - pad_x],   M = 0 outside,
    float32 FMAs in a fixed order (no TF32).  maps: a list of (dd, h, w) float32 CUDA tensors; maps that are contiguous views
    of one storage (as vl_hog_pyramid returns them) are read in place, others are packed first.  filters: (Q, dd, fh, fw);
    bias: (Q,) or None; pad = (pad_x, pad_y), each in [0, filter side - 1].  Returns one (Q, oh, ow) tensor per map,
    oh = h + 2 pad_y - fh + 1 and ow = w + 2 pad_x - fw + 1 (an empty tensor where either is <= 0)."""
    ctx = ctx or default_context()
    dd = _hog_dims(num_bins, variant)
    dev = f"cuda:{ctx.device}"
    f = _tensor(filters)
    if f.dtype != torch.float32 or f.dim() != 4 or f.shape[1] != dd:
        raise ValueError(f"filters must be a float32 (Q, dd, fh, fw) tensor with dd = {dd}")
    f = f.to(dev).contiguous()
    q, _, fh, fw = f.shape
    b = None
    if bias is not None:
        b = _tensor(bias).to(dev, torch.float32).contiguous()
        if b.shape != (q,):
            raise ValueError(f"bias must have one value per filter ({q})")
    pad_x, pad_y = (int(p) for p in pad)
    maps = list(maps)
    _check_maps(maps, dd)
    if not maps:
        return []
    # a map smaller than the filter scores nothing: an empty (Q, oh, ow) tensor
    out, out_offs, scores = _results([(q, max(m.shape[1] + 2 * pad_y - fh + 1, 0), max(m.shape[2] + 2 * pad_x - fw + 1, 0))
                                      for m in maps], dev)
    g, keep = _maps_table(maps, dd, dev, out_offs)
    _check(ctx.h, _capi.lib().sd_hog_correlate(ctx.h, C.byref(g), int(num_bins), int(variant), ptr(f), int(q), int(fw), int(fh),
                                               ptr(b), pad_x, pad_y, ptr(out)))
    return scores


HogDetections = collections.namedtuple("HogDetections", "frame boxes scores filter level cell above")
HogDetections.__doc__ = """Detections of vl_hog_detect, in frame order and then in the rule's order within each frame: frame (n,) int32,
boxes (n, 4) int32 (x, y, w, h in frame pixels), scores (n,) float32, filter (n,) int32, level (n,) int32 (the scale index),
cell (n, 2) int32 (the score position x, y in its level), and above (num_frames,) int64, each frame's candidate count."""


def vl_hog_detect(frames, scales, filters, cell_size: int, num_bins: int, threshold: float, variant: int = 1, bias=None, pad=(0, 0),
                  overlap: float = 0.5, max_candidates: int = 4096, max_detections: int = 256,
                  ctx: Optional[Context] = None, multichannel: bool = False, bilinear_orientations: bool = False,
                  float_frames: bool = False) -> HogDetections:
    """A sliding-window detector over image pyramids: vl_hog_pyramid of every frame at every scale, vl_hog_correlate of the
    filter bank on every level (read in place), and one sd_hog_detections call over all score maps: the scores above threshold,
    their boxes in frame pixels, the first max_candidates of each frame by score, and greedy non-maximum suppression at IoU
    overlap over all filters as one class, up to max_detections per frame.  frames, scales, filters, bias, pad, multichannel,
    bilinear_orientations and float_frames as vl_hog_pyramid and vl_hog_correlate take them; filters trained with
    multichannel, bilinear_orientations or float_frames are scored with the same.  Returns HogDetections;
    detect_faces(frames, d.frame, boxes=d.boxes) takes the result as it is."""
    ctx = ctx or default_context()
    f = _tensor(filters)
    if f.dim() != 4:
        raise ValueError("filters must be a (Q, dd, fh, fw) tensor")
    q, _, fh, fw = f.shape
    pad_x, pad_y = (int(p) for p in pad)
    feats, levels = vl_hog_pyramid(frames, scales, cell_size, num_bins, variant, ctx=ctx, multichannel=multichannel,
                                   bilinear_orientations=bilinear_orientations, float_frames=float_frames)
    n = len(feats)
    if n == 0:
        return _detections(None, None, None)[0]
    sizes = _frame_sizes(frames, n)
    which = [(i, s) for i in range(n) for s in range(len(scales)) if feats[i][s] is not None]
    scores = vl_hog_correlate([feats[i][s] for i, s in which], f, num_bins, variant, bias=bias, pad=(pad_x, pad_y), ctx=ctx)
    dev = f"cuda:{ctx.device}"
    md = int(max_detections)
    out = torch.empty((n, max(md, 1), len(HogDetectionC._fields_)), dtype=torch.int32, device=dev)
    count = torch.empty(n, dtype=torch.int32, device=dev)
    above = torch.empty(n, dtype=torch.int64, device=dev)
    table, base = None, None
    if which:
        base = scores[0].untyped_storage().data_ptr()    # the maps' scores are views of one buffer
        table = _device_table([HogScoreMapC(i, s, sizes[i][0], sizes[i][1], levels[i][s][0], levels[i][s][1], sc.shape[2], sc.shape[1],
                                            sc.storage_offset()) for (i, s), sc in zip(which, scores)], dev)
    _check(ctx.h, _capi.lib().sd_hog_detections(ctx.h, ptr(base), ptr(table), len(which), n, int(q), int(cell_size), int(fw), int(fh),
                                                pad_x, pad_y, float(threshold), float(overlap), int(max_candidates), md, ptr(out),
                                                ptr(count), ptr(above)))
    return _detections(out, count, above)[0]


def _frame_sizes(frames, n: int):
    """(width, height) of each of the n frames of a frames argument as vl_hog_pyramid takes it."""
    if isinstance(frames, (list, tuple)):
        return [(int(fr.shape[1]), int(fr.shape[0])) for fr in frames]
    return [(int(frames.shape[2]), int(frames.shape[1]))] * n


def _frame_rows(rows, counts):
    """rows[i, :counts[i]] of every frame i, end to end."""
    return np.concatenate([rows[i, :c] for i, c in enumerate(counts)] + [np.zeros((0,) + rows.shape[2:], rows.dtype)])


def _detections(out, count, above):
    """The output of one sd_hog_detections call on the host -> (HogDetections, each frame's detection count).  out, count,
    above: its (n, max_detections, 9) int32, (n,) int32 and (n,) int64 device tensors, or None for a call without frames."""
    if out is None:
        rows, counts, above = np.zeros((0, 1, len(HogDetectionC._fields_)), np.int32), np.zeros(0, np.int64), np.zeros(0, np.int64)
    else:
        rows, counts, above = out.cpu().numpy(), count.cpu().numpy().astype(np.int64), above.cpu().numpy()
    r = _frame_rows(rows, counts)
    return HogDetections(np.repeat(np.arange(len(counts), dtype=np.int32), counts), np.ascontiguousarray(r[:, 0:4]),
                         np.ascontiguousarray(r[:, 4]).view(np.float32), np.ascontiguousarray(r[:, 5]), np.ascontiguousarray(r[:, 6]),
                         np.ascontiguousarray(r[:, 7:9]), above), counts


# ------------------------------------------------------------------------------------------------
# training HOG filters: window rows, a squared-hinge SVM and hard-negative mining
# ------------------------------------------------------------------------------------------------
def _check_maps(maps, dd: int) -> None:
    if any(not isinstance(m, torch.Tensor) or not m.is_cuda or m.dtype != torch.float32 or m.dim() != 3 or m.shape[0] != dd
           for m in maps):
        raise ValueError(f"every map must be a float32 CUDA tensor (dd, h, w) with dd = {dd}")


def _maps_table(maps, dd: int, dev, out_offsets=None):
    """A non-empty list of (dd, h, w) float32 CUDA maps -> (HogGridsC, tensors it points to): read in place when they are
    contiguous views of one storage (as vl_hog_pyramid returns them), packed otherwise.  out_offsets: each map's element offset
    in the call's output, 0 for every map when None."""
    _check_maps(maps, dd)
    maps = [m.to(dev) for m in maps]
    stor = maps[0].untyped_storage().data_ptr()
    if all(m.is_contiguous() and m.untyped_storage().data_ptr() == stor for m in maps):
        base, keep = stor, maps
        offs = [(m.data_ptr() - base) // 4 for m in maps]
    else:
        keep, offs = _pack(maps, dev)
        base = keep.data_ptr()
    out_offsets = out_offsets or [0] * len(maps)
    table = _device_table([HogGridC(m.shape[2], m.shape[1], o, oo) for m, o, oo in zip(maps, offs, out_offsets)], dev)
    g = HogGridsC()
    g.d_features, g.count, g.width, g.height, g.d_grids = base, len(maps), 0, 0, table.data_ptr()
    return g, (keep, table)


def vl_hog_windows(maps, windows, filter_size, num_bins: int, variant: int = 1, pad=(0, 0), ctx: Optional[Context] = None):
    """The feature rows of score positions (sd_hog_windows): row r is the window that score (x, y) of vl_hog_correlate on map
    `grid` reads, in the filter layout [dd][fh][fw] flattened, then a 1.0 bias column -- D = dd * fh * fw + 1 floats.  flip = 1
    gives the window of the mirrored image (vl_hog_flip of the block).  maps: a list of (dd, h, w) float32 CUDA tensors as
    vl_hog_correlate takes them; windows: an (n, 4) int array of (grid, x, y, flip); filter_size = (fw, fh).  Returns an (n, D)
    float32 CUDA tensor."""
    ctx = ctx or default_context()
    dd = _hog_dims(num_bins, variant)
    dev = f"cuda:{ctx.device}"
    fw, fh = (int(v) for v in filter_size)
    pad_x, pad_y = (int(v) for v in pad)
    w = np.ascontiguousarray(np.asarray(windows, np.int32).reshape(-1, 4))
    n, D = w.shape[0], dd * fw * fh + 1
    rows = torch.empty((max(n, 1), D), dtype=torch.float32, device=dev)
    maps = list(maps)
    if not maps:
        raise ValueError("vl_hog_windows needs at least one map")
    g, keep = _maps_table(maps, dd, dev)
    d_w = torch.from_numpy(w if n else np.zeros((1, 4), np.int32)).to(dev)
    _check(ctx.h, _capi.lib().sd_hog_windows(ctx.h, C.byref(g), int(num_bins), int(variant), fw, fh, pad_x, pad_y, ptr(d_w), n,
                                             ptr(rows), C.c_int64(D)))
    return rows[:n]


def hog_box_windows(width: int, height: int, boxes, scales, filter_size, cell_size: int, num_bins: int, variant: int = 1,
                    pad=(0, 0), positive_overlap: float = 0.5):
    """For each ground-truth box (x, y, w, h) of one width x height frame, the window of the frame's pyramid that covers it best
    (sd_hog_box_windows, host only): the largest exact IoU between the box and the integer box sd_hog_detections reports for a
    score position, ties to the lower level, then y, then x.  Returns (windows, iou): an (n, 3) int32 array of (level, x, y),
    level -1 where the best IoU is below positive_overlap, and the (n,) float64 IoU of each box's best window."""
    b = np.ascontiguousarray(np.asarray(boxes, np.int32).reshape(-1, 4))
    n = b.shape[0]
    sc = (C.c_double * max(len(scales), 1))(*[float(s) for s in scales])
    out = (HogWindowC * max(n, 1))()
    iou = np.zeros(max(n, 1), np.float64)
    fw, fh = (int(v) for v in filter_size)
    pad_x, pad_y = (int(v) for v in pad)
    rc = _capi.lib().sd_hog_box_windows(int(width), int(height), sc, len(scales), int(cell_size), int(num_bins), int(variant), fw, fh,
                                        pad_x, pad_y, float(positive_overlap), C.c_void_p(b.ctypes.data), n, out,
                                        C.c_void_p(iou.ctypes.data))
    if rc:
        raise SdError(rc, f"invalid hog_box_windows arguments: frame {width} x {height}, scales {list(scales)}, filter {fw} x {fh}, "
                          f"pad ({pad_x}, {pad_y}), cell_size {cell_size}, positive_overlap {positive_overlap}, or a box with w or h < 1")
    win = np.array([(out[i].grid, out[i].x, out[i].y) for i in range(n)], np.int32).reshape(n, 3)
    return win, iou[:n].copy()


SvmReport = collections.namedtuple("SvmReport", "iterations active stop objective")
SvmReport.__doc__ = """Report of learn_squared_hinge: Newton steps, the final active-set size, the stop reason ("converged",
"no decrease" or "iteration cap") and the objective f in float64."""
_SVM_STOP = {0: "converged", 1: "no decrease", 2: "iteration cap"}


def _svm_report(r) -> SvmReport:
    return SvmReport(int(r.iterations), int(r.active), _SVM_STOP[int(r.stop)], float(r.objective))


def learn_squared_hinge(A, y, lam: float, max_iterations: int = 50, ctx: Optional[Context] = None):
    """Linear SVM with squared hinge loss on the device (sd_learn_squared_hinge): w minimising
        lam / 2 * sum_{j < D-1} w_j^2 + 1/2 * sum_i max(0, 1 - y_i a_i . w)^2
    over the rows of A (N x D; the last column all ones: the unregularised bias), y_i = +1 or -1, by the primal finite Newton
    method on the learn path.  Returns (w, SvmReport): w a (D,) float32 CUDA tensor."""
    ctx = ctx or default_context()
    A = _dev(A, ctx)
    yy = _dev(y, ctx).reshape(-1)
    if A.dim() != 2 or yy.shape[0] != A.shape[0]:
        raise ValueError("A must be (N, D) and y (N,)")
    N, D = A.shape
    w = torch.empty(D, dtype=torch.float32, device=A.device)
    rep = SvmReportC()
    _check(ctx.h, _capi.lib().sd_learn_squared_hinge(ctx.h, ptr(A), C.c_int64(A.stride(0)), ptr(yy), N, D, float(lam),
                                                     int(max_iterations), ptr(w), C.byref(rep)))
    return w, _svm_report(rep)


HogFilter = collections.namedtuple("HogFilter", "filter bias negatives report")
HogFilter.__doc__ = """Result of train_hog_filter: filter (dd, fh, fw) float32 CUDA tensor, bias (float), negatives (n, 4) int32
array of the negative cache in slot order (frame, level, x, y), and report, one dict per mining round (the fields of
sd_hog_train_report, the solve as an SvmReport, or None when the round's solve was skipped; times_ms, the round's phases in
milliseconds, and gathered_bytes).  positive_overlap reaches the library as a float: the positives are hog_box_windows(...,
positive_overlap=float(np.float32(positive_overlap))).  The filter is one for the features it was trained on: one trained with
multichannel, bilinear_orientations or float_frames is scored by vl_hog_detect with the same values."""


def train_hog_filter(frames, box_frame, boxes, scales, filter_size, cell_size: int, num_bins: int, variant: int = 1, pad=(0, 0),
                     lam: float = 0.01, positive_overlap: float = 0.5, negative_overlap: float = 0.3, flip_positives: bool = False,
                     rounds: int = 3, negatives_per_frame: int = 32, mine_overlap: float = 0.5, max_negatives: int = 8192,
                     max_iterations: int = 50, ctx: Optional[Context] = None, multichannel: bool = False,
                     bilinear_orientations: bool = False, float_frames: bool = False) -> HogFilter:
    """Train a HOG filter for vl_hog_detect (sd_hog_train_filter): each box's best window as a positive (hog_box_windows, with
    its mirror if flip_positives), round 0 with the mean positive minus its mean as the filter, then `rounds` rounds of
    hard-negative mining at the margin (threshold -1) and a squared-hinge SVM (learn_squared_hinge) each.  frames,
    multichannel, bilinear_orientations and float_frames as vl_hog_pyramid takes them (multichannel:
    sd_hog_train_filter_images, with float_frames sd_hog_train_filter_float); box_frame (n,) and boxes (n, 4) (x, y, w, h) in
    the layout of HogDetections.  vl_hog_detect(frames, scales, hf.filter[None], ..., bias=[hf.bias]) with the same
    multichannel, bilinear_orientations and float_frames takes the result as it is."""
    ctx = ctx or default_context()
    dd = _hog_dims(num_bins, variant)
    fw, fh = (int(v) for v in filter_size)
    pad_x, pad_y = (int(v) for v in pad)
    scales = [float(s) for s in scales]
    if not scales:
        raise ValueError("train_hog_filter needs at least one scale")

    def check(w, h):
        for s in scales:
            hog_pyramid_shape(w, h, s, cell_size, num_bins, variant)

    keep, ib, sizes = _window_frames(frames, ctx, check, multichannel, bilinear_orientations, float_frames)
    if not sizes:
        raise ValueError("train_hog_filter needs at least one frame")
    bf = np.asarray(box_frame, np.int64).reshape(-1)
    bx = np.asarray(boxes, np.int64).reshape(-1, 4)
    if bf.shape[0] != bx.shape[0]:
        raise ValueError("box_frame and boxes must have one entry per box")
    nb = bx.shape[0]
    hb = (HogBoxC * max(nb, 1))(*[HogBoxC(int(f), *(int(v) for v in b)) for f, b in zip(bf, bx)])
    prm = HogTrainParamC(float(lam), float(positive_overlap), float(negative_overlap), int(bool(flip_positives)), int(rounds),
                         int(negatives_per_frame), float(mine_overlap), int(max_negatives), int(max_iterations))
    dev = f"cuda:{ctx.device}"
    filt = torch.empty((dd, fh, fw), dtype=torch.float32, device=dev)
    bias = C.c_float(0)
    reps = (HogTrainReportC * (int(rounds) + 1))() if rounds >= 0 else None
    negs = (HogWindowC * max(int(max_negatives), 1))()
    nn = C.c_int(0)
    sc = (C.c_double * len(scales))(*scales)
    lib = _capi.lib()
    rest = (hb, nb, sc, len(scales), int(cell_size), int(num_bins), int(variant), fw, fh, pad_x, pad_y, C.byref(prm), ptr(filt),
            C.byref(bias), reps, negs, C.byref(nn))
    if multichannel:
        call = lib.sd_hog_train_filter_float if float_frames else lib.sd_hog_train_filter_images
        _check(ctx.h, call(ctx.h, C.byref(ib), int(bool(bilinear_orientations)), *rest))
    else:
        _check(ctx.h, lib.sd_hog_train_filter(ctx.h, C.byref(ib), *rest))
    S = len(scales)
    neg = np.array([(negs[k].grid // S, negs[k].grid % S, negs[k].x, negs[k].y) for k in range(nn.value)], np.int32).reshape(-1, 4)
    report = []
    for r in reps:
        d = {f: int(getattr(r, f)) for f, _ in HogTrainReportC._fields_[:10] if f != "reserved"}
        d["solve"] = _svm_report(r.solve) if r.solved else None
        d["times_ms"] = {f[:-3]: float(getattr(r, f)) for f in ("pyramid_ms", "scores_ms", "detect_ms", "host_ms", "gather_ms", "solve_ms")}
        d["gathered_bytes"] = float(r.gathered_bytes)
        report.append(d)
    return HogFilter(filt, float(bias.value), neg, report)


# ------------------------------------------------------------------------------------------------
# deformable part models: bounded and exact distance transforms, star-model scores and part placements
# ------------------------------------------------------------------------------------------------
PART_MAX_DISPLACEMENT = 32   # SD_HOG_PART_MAX_DISPLACEMENT
PART_MAX_PARTS = 32          # SD_HOG_PART_MAX_PARTS


class HogPartModel:
    """A star model of Q components for vl_hog_part_detect: root (Q, dd, fh, fw) filters with bias (Q,), parts (Q, P, dd, pfh, pfw)
    filters scored at twice the root's resolution, anchors (Q, P, 2) int (ax, ay) in part-level cells relative to twice the root
    window's top-left cell, deformation (Q, P, 4) (w0, w1, w2, w3): a displacement (dx, dy) costs w0 dx^2 + w1 dx + w2 dy^2 + w3 dy,
    pad = (pad_x, pad_y) of the root correlate, part_pad of the part correlate, and max_displacement R bounding |dx| and |dy|,
    or None for the exact, unbounded transform of DPM (which needs w0 > 0 and w2 > 0).  The filters are ones for the features they were trained on: a model of colour HOG (vl_hog_pyramid's multichannel,
    bilinear_orientations and float_frames) is scored by vl_hog_part_detect with the same values."""

    def __init__(self, root, bias, parts, anchors, deformation, pad=(0, 0), part_pad=(0, 0), max_displacement: Optional[int] = 4):
        self.root = _tensor(root).to(torch.float32).contiguous()
        self.bias = _tensor(bias).to(torch.float32).reshape(-1).contiguous()
        self.parts = _tensor(parts).to(torch.float32).contiguous()
        self.anchors = np.ascontiguousarray(np.asarray(anchors, np.int64)).astype(np.int32)
        self.deformation = np.ascontiguousarray(np.asarray(deformation, np.float32))
        self.pad = tuple(int(v) for v in pad)
        self.part_pad = tuple(int(v) for v in part_pad)
        self.max_displacement = None if max_displacement is None else int(max_displacement)
        if self.root.dim() != 4 or self.parts.dim() != 5:
            raise ValueError("root must be (Q, dd, fh, fw) and parts (Q, P, dd, pfh, pfw)")
        q, dd = self.root.shape[:2]
        if self.parts.shape[0] != q or self.parts.shape[2] != dd:
            raise ValueError("parts must be (Q, P, dd, pfh, pfw) with the root's Q and dd")
        p = self.parts.shape[1]
        if self.bias.shape != (q,) or self.anchors.shape != (q, p, 2) or self.deformation.shape != (q, p, 4):
            raise ValueError(f"bias must be ({q},), anchors ({q}, {p}, 2) and deformation ({q}, {p}, 4)")

    @property
    def num_components(self) -> int:
        return self.root.shape[0]

    @property
    def num_parts(self) -> int:
        return self.parts.shape[1]

    def flipped(self, num_bins: int, variant: int = 1, ctx: Optional[Context] = None) -> "HogPartModel":
        """The model of the left-right mirrored image: vl_hog_flip of the root and every part, anchors ax' = 2 fw - ax - pfw, and
        w1 negated (a displacement dx becomes -dx).  Pads and R are kept."""
        q, p, dd, pfh, pfw = self.parts.shape
        fw = self.root.shape[3]
        root = vl_hog_flip(self.root, num_bins, variant, ctx=ctx)
        parts = vl_hog_flip(self.parts.reshape(q * p, dd, pfh, pfw), num_bins, variant, ctx=ctx).reshape(q, p, dd, pfh, pfw)
        anchors = self.anchors.copy()
        anchors[..., 0] = 2 * fw - anchors[..., 0] - pfw
        deformation = self.deformation.copy()
        deformation[..., 1] = -deformation[..., 1]
        return HogPartModel(root, self.bias.clone(), parts, anchors, deformation, self.pad, self.part_pad, self.max_displacement)

    def _c(self, dev):
        """(HogPartModelC, the device anchors it points to)."""
        q, p, _, pfh, pfw = self.parts.shape
        _, _, fh, fw = self.root.shape
        anchors = torch.from_numpy(self.anchors).to(dev)
        return HogPartModelC(q, p, fw, fh, pfw, pfh, self.pad[0], self.pad[1], self.part_pad[0], self.part_pad[1],
                             anchors.data_ptr()), anchors


def _deformation(deformation, planes: int):
    d = np.ascontiguousarray(np.asarray(deformation, np.float32).reshape(-1))
    if d.size != 4 * planes:
        raise ValueError(f"deformation must hold 4 values per plane ({planes} planes)")
    return d, C.c_void_p(d.ctypes.data)


def vl_hog_distance_transform(maps, deformation, max_displacement: Optional[int] = None, ctx: Optional[Context] = None):
    """The generalised distance transform of score maps on the device:
        D(v, u) = max over (dx, dy) of s(v + dy, u + dx) - (w0 dx^2 + w1 dx + w2 dy^2 + w3 dy),
    separably, and where that maximum is, (u + dx, v + dy).  max_displacement None: the exact, unbounded transform of DPM
    (sd_hog_distance_transform_exact: lower envelopes in float64, finite scores only; w0 > 0 and w2 > 0); an integer R in
    [0, 32]: |dx|, |dy| <= R in float32 (sd_hog_distance_transform).  The rules and tie breaks are in include/sd_b200.h.  maps:
    a (N, P, h, w) float32 tensor, or a list of (P, h, w) maps of any sizes; deformation: (P, 4), plane k's (w0, w1, w2, w3).
    Returns (values, placements) in the shapes of maps, placements with a trailing (u, v) axis of int32 ((-1, -1) where the
    rule places nothing)."""
    ctx = ctx or default_context()
    dev = f"cuda:{ctx.device}"
    single = not isinstance(maps, (list, tuple))
    items = [_tensor(maps)] if single else [_tensor(m) for m in maps]
    if any(t.dtype != torch.float32 or t.dim() != (4 if single else 3) for t in items):
        raise ValueError("maps must be a float32 (N, P, h, w) tensor or a list of (P, h, w) tensors")
    if not items or (single and items[0].shape[0] == 0):
        return (items[0].clone(), torch.zeros(tuple(items[0].shape) + (2,), dtype=torch.int32, device=items[0].device)) if single else ([], [])
    planes = items[0].shape[-3]
    if any(t.shape[-3] != planes for t in items):
        raise ValueError("every map must have the same number of planes")
    d, d_ptr = _deformation(deformation, planes)
    g = HogGridsC()
    g.d_grids = None
    if single:
        keep = items[0].to(dev).contiguous()
        n, _, h, w = keep.shape
        g.d_features, g.count, g.width, g.height = keep.data_ptr(), n, w, h
        values = torch.empty_like(keep)
        place = torch.empty(tuple(keep.shape) + (2,), dtype=torch.int32, device=dev)
        table = None
    else:
        keep, offs = _pack(items, dev)
        values = torch.empty_like(keep)
        place = torch.empty((keep.numel(), 2), dtype=torch.int32, device=dev)
        table = _device_table([HogGridC(t.shape[2], t.shape[1], o, o) for t, o in zip(items, offs)], dev)
        g.d_features, g.count, g.width, g.height, g.d_grids = keep.data_ptr(), len(items), 0, 0, table.data_ptr()
    lib = _capi.lib()
    if max_displacement is None:
        _check(ctx.h, lib.sd_hog_distance_transform_exact(ctx.h, C.byref(g), int(planes), d_ptr, ptr(values), ptr(place)))
    else:
        _check(ctx.h, lib.sd_hog_distance_transform(ctx.h, C.byref(g), int(planes), d_ptr, int(max_displacement), ptr(values),
                                                    ptr(place)))
    if single:
        return values, place
    return ([values[o:o + t.numel()].view(t.shape) for t, o in zip(items, offs)],
            [place[o:o + t.numel()].view(tuple(t.shape) + (2,)) for t, o in zip(items, offs)])


def vl_hog_part_scores(root_scores, part_values, model: HogPartModel, ctx: Optional[Context] = None):
    """The star model's score maps (sd_hog_part_scores): for each root map (Q, oh, ow) of vl_hog_correlate with the model's root
    filters, and its transformed part maps (Q * P, ph, pw) of vl_hog_distance_transform (or None: every anchor is outside),
        total = root[q, y, x] + D[q P + p, v0, u0] for p = 0 .. P - 1 in order, in float32,
    at u0 = 2 (x - pad_x) + ax + part_pad_x, v0 alike, and -inf where any anchor lies outside the part map.  Returns one
    (Q, oh, ow) float32 CUDA tensor per root map."""
    ctx = ctx or default_context()
    dev = f"cuda:{ctx.device}"
    roots = [_tensor(r) for r in root_scores]
    parts = [None if v is None else _tensor(v) for v in part_values]
    if len(roots) != len(parts):
        raise ValueError("one part map (or None) per root map")
    q, p = model.num_components, model.num_parts
    if any(r.dtype != torch.float32 or r.dim() != 3 or r.shape[0] != q for r in roots):
        raise ValueError(f"root maps must be float32 (Q, oh, ow) with Q = {q}")
    if any(v is not None and (v.dtype != torch.float32 or v.dim() != 3 or v.shape[0] != q * p) for v in parts):
        raise ValueError(f"part maps must be float32 (Q * P, ph, pw) with Q * P = {q * p}")
    if not roots:
        return []
    keep_r, roff = _pack(roots, dev)
    present = [v for v in parts if v is not None]
    keep_p, poff = _pack(present, dev) if present else (torch.zeros(1, device=dev), [])
    poff = iter(poff)
    descs, out_shapes = [], []
    for r, v in zip(roots, parts):
        pw, ph, po = (v.shape[2], v.shape[1], next(poff)) if v is not None else (0, 0, 0)
        descs.append((r.shape[2], r.shape[1], pw, ph, po))
        out_shapes.append(tuple(r.shape))
    out, ooff, res = _results(out_shapes, dev)
    table = _device_table([HogPartMapC(0, k, 1, 1, 1, 1, w, h, pw, ph, ro, po, oo)
                           for k, ((w, h, pw, ph, po), ro, oo) in enumerate(zip(descs, roff, ooff))], dev)
    mc, anchors = model._c(dev)
    _check(ctx.h, _capi.lib().sd_hog_part_scores(ctx.h, ptr(keep_r), ptr(keep_p), ptr(table), len(roots), C.byref(mc), ptr(out)))
    return res


HogPartDetections = collections.namedtuple("HogPartDetections", HogDetections._fields + ("parts", "placement", "part_scores"))
HogPartDetections.__doc__ = """Detections of vl_hog_part_detect: the fields of HogDetections (filter is the component q), plus parts
(n, P, 4) int32 part boxes (x, y, w, h in frame pixels, zero where a part has no placement), placement (n, P, 2) int32 (u, v) part
score positions ((-1, -1) for none) and part_scores (n, P) float32, each part's transformed score D at its anchor."""


def vl_hog_part_detect(frames, scales, model: HogPartModel, cell_size: int, num_bins: int, threshold: float, variant: int = 1,
                       overlap: float = 0.5, max_candidates: int = 4096, max_detections: int = 256,
                       ctx: Optional[Context] = None, multichannel: bool = False,
                       bilinear_orientations: bool = False, float_frames: bool = False) -> HogPartDetections:
    """A star-model detector over image pyramids: one vl_hog_pyramid over the root scales and their doubles (a scale present in
    both is computed once; root scales must be <= 2), vl_hog_correlate of the root filters (bias included) on the root levels and
    of all Q * P part filters on the part levels, each read in place; vl_hog_distance_transform of the part maps; the star
    model's scores (vl_hog_part_scores); sd_hog_detections over them with the root's filter size and pad, all components as one
    class; and the part placements of every detection (sd_hog_part_placements, or with the model's max_displacement None, the
    exact transform's placement maps read at the anchors by sd_hog_part_placements_mapped).  One host read-back at the end.  frames,
    multichannel, bilinear_orientations and float_frames as vl_hog_pyramid takes them.  Returns HogPartDetections; detect_faces(frames,
    d.frame, boxes=d.boxes) takes the result as it is."""
    ctx = ctx or default_context()
    dev = f"cuda:{ctx.device}"
    q, p, dd, pfh, pfw = model.parts.shape
    _, _, fh, fw = model.root.shape
    if dd != _hog_dims(num_bins, variant):
        raise ValueError(f"the model's dd ({dd}) is not that of num_bins {num_bins}, variant {variant}")
    scales = [float(s) for s in scales]
    if not scales or any(not 0 < s <= 2 for s in scales):
        raise ValueError("vl_hog_part_detect needs root scales in (0, 2]")
    every = list(dict.fromkeys(scales + [2 * s for s in scales]))
    ri, pi = [every.index(s) for s in scales], [every.index(2 * s) for s in scales]
    feats, levels = vl_hog_pyramid(frames, every, cell_size, num_bins, variant, ctx=ctx, multichannel=multichannel,
                                   bilinear_orientations=bilinear_orientations, float_frames=float_frames)
    n = len(feats)
    if n == 0:
        return _part_detections(_detections(None, None, None), np.zeros((0, 1, p, len(HogPartPlacementC._fields_)), np.int32))
    sizes = _frame_sizes(frames, n)
    which = [(i, s) for i in range(n) for s in range(len(scales)) if feats[i][ri[s]] is not None]
    roots = vl_hog_correlate([feats[i][ri[s]] for i, s in which], model.root, num_bins, variant, bias=model.bias, pad=model.pad,
                             ctx=ctx) if which else []
    kept = [(i, s, r) for (i, s), r in zip(which, roots) if r.numel()]
    # every part level of a kept root map, once
    plevels = list(dict.fromkeys((i, pi[s]) for i, s, _ in kept if feats[i][pi[s]] is not None))
    pscores = vl_hog_correlate([feats[i][l] for i, l in plevels], model.parts.reshape(q * p, dd, pfh, pfw), num_bins, variant,
                               pad=model.part_pad, ctx=ctx) if plevels else []
    pmap = {key: sc for key, sc in zip(plevels, pscores) if sc.numel()}
    d, d_ptr = _deformation(model.deformation, q * p)
    R = model.max_displacement
    lib = _capi.lib()
    if pmap:
        stor = next(iter(pmap.values())).untyped_storage()
        raw = torch.empty(0, dtype=torch.float32, device=dev).set_(stor)
        values = torch.empty_like(raw)
        pmaps = torch.empty((raw.numel() if R is None else 1, 2), dtype=torch.int32, device=dev)
        g = HogGridsC()
        gt = _device_table([HogGridC(sc.shape[2], sc.shape[1], sc.storage_offset(), sc.storage_offset()) for sc in pmap.values()], dev)
        g.d_features, g.count, g.width, g.height, g.d_grids = raw.data_ptr(), len(pmap), 0, 0, gt.data_ptr()
        if R is None:
            _check(ctx.h, lib.sd_hog_distance_transform_exact(ctx.h, C.byref(g), q * p, d_ptr, ptr(values), ptr(pmaps)))
        else:
            _check(ctx.h, lib.sd_hog_distance_transform(ctx.h, C.byref(g), q * p, d_ptr, int(R), ptr(values), None))
    else:
        raw = values = torch.zeros(1, dtype=torch.float32, device=dev)
        pmaps = torch.zeros((1, 2), dtype=torch.int32, device=dev)
    mc, anchors = model._c(dev)
    md = int(max_detections)
    out = torch.empty((n, max(md, 1), len(HogDetectionC._fields_)), dtype=torch.int32, device=dev)
    count = torch.empty(n, dtype=torch.int32, device=dev)
    above = torch.empty(n, dtype=torch.int64, device=dev)
    place = torch.empty((n, max(md, 1), p, len(HogPartPlacementC._fields_)), dtype=torch.int32, device=dev)
    table = score_table = total = None
    if kept:
        rbase = kept[0][2].untyped_storage()
        total = torch.empty(rbase.nbytes() // 4, dtype=torch.float32, device=dev)
        descs, sdescs = [], []
        for i, s, r in kept:
            sc = pmap.get((i, pi[s]))
            plw, plh = levels[i][pi[s]]
            pw, ph, po = (sc.shape[2], sc.shape[1], sc.storage_offset()) if sc is not None else (0, 0, 0)
            off = r.storage_offset()
            descs.append(HogPartMapC(i, s, sizes[i][0], sizes[i][1], plw, plh, r.shape[2], r.shape[1], pw, ph, off, po, off))
            sdescs.append(HogScoreMapC(i, s, sizes[i][0], sizes[i][1], levels[i][ri[s]][0], levels[i][ri[s]][1], r.shape[2], r.shape[1],
                                       off))
        table = _device_table(descs, dev)
        score_table = _device_table(sdescs, dev)
        _check(ctx.h, lib.sd_hog_part_scores(ctx.h, ptr(kept[0][2].untyped_storage().data_ptr()), ptr(values), ptr(table), len(kept),
                                             C.byref(mc), ptr(total)))
    _check(ctx.h, lib.sd_hog_detections(ctx.h, ptr(total), ptr(score_table), len(kept), n, int(q), int(cell_size), int(fw), int(fh),
                                        model.pad[0], model.pad[1], float(threshold), float(overlap), int(max_candidates), md,
                                        ptr(out), ptr(count), ptr(above)))
    if R is None:
        _check(ctx.h, lib.sd_hog_part_placements_mapped(ctx.h, ptr(values), ptr(pmaps), ptr(table), len(kept), C.byref(mc),
                                                        int(cell_size), ptr(out), ptr(count), n, md, ptr(place)))
    else:
        _check(ctx.h, lib.sd_hog_part_placements(ctx.h, ptr(raw), ptr(table), len(kept), C.byref(mc), d_ptr, int(R), int(cell_size),
                                                 ptr(out), ptr(count), n, md, ptr(place)))
    return _part_detections(_detections(out, count, above), place.cpu().numpy())


def _part_detections(detections, place):
    """HogPartDetections from _detections' result and the (n, max_detections, P, 7) int32 sd_hog_part_placement rows."""
    d, counts = detections
    pr = _frame_rows(place, counts)
    return HogPartDetections(*d, np.ascontiguousarray(pr[:, :, 3:7]), np.ascontiguousarray(pr[:, :, 0:2]),
                             np.ascontiguousarray(pr[:, :, 2]).view(np.float32))
