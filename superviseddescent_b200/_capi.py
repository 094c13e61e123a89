"""ctypes binding of the C ABI in include/sd_b200.h (libsd_b200.so).

There is no CPU fallback: if the shared object is missing, or no CUDA device is usable, every entry
point raises.  torch is used by callers only for device buffers / streams / torch.distributed.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libsd_b200.so")


class SdError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"sd_b200 error {code}: {msg}")
        self.code = code


class HogParam(C.Structure):
    """rcr::HoGParam (reference include/rcr/adaptive_vlhog.hpp:41-60)."""
    _fields_ = [("variant", C.c_int32), ("num_cells", C.c_int32), ("cell_size", C.c_int32),
                ("num_bins", C.c_int32), ("relative_patch_size", C.c_float)]


class RegulariserC(C.Structure):
    _fields_ = [("type", C.c_int32), ("param", C.c_float), ("regularise_last_row", C.c_int32)]


class NormalisationC(C.Structure):
    _fields_ = [("kind", C.c_int32), ("n_right", C.c_int32), ("n_left", C.c_int32),
                ("right_idx", C.c_int32 * 4), ("left_idx", C.c_int32 * 4)]


class ImageBatchC(C.Structure):
    _fields_ = [("d_data", C.c_void_p), ("width", C.c_int32), ("height", C.c_int32), ("row_stride", C.c_int32),
                ("image_stride", C.c_int64), ("count", C.c_int32), ("d_roi", C.c_void_p), ("d_roi_miss", C.c_void_p),
                ("d_frames", C.c_void_p)]


class FrameC(C.Structure):
    """sd_frame: one frame of a batch with differently sized frames."""
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("row_stride", C.c_int32), ("reserved", C.c_int32), ("offset", C.c_int64)]


class HogImageC(C.Structure):
    """sd_hog_image: one frame of sd_hog_dense_images; offset and strides in elements."""
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("offset", C.c_int64), ("row_stride", C.c_int64),
                ("pixel_stride", C.c_int64), ("channel_stride", C.c_int64)]


class HogImagesC(C.Structure):
    """sd_hog_images: u8 or f32 frames of 1..16 channels on the device, equally sized or one descriptor per frame."""
    _fields_ = [("d_data", C.c_void_p), ("dtype", C.c_int32), ("channels", C.c_int32), ("count", C.c_int32),
                ("frame", HogImageC), ("image_stride", C.c_int64), ("d_frames", C.c_void_p)]


class HogPolarFieldsC(C.Structure):
    """sd_hog_polar_fields: f32 modulus and angle fields on the device, one descriptor placing an element in both buffers."""
    _fields_ = [("d_modulus", C.c_void_p), ("d_angle", C.c_void_p), ("count", C.c_int32), ("frame", HogImageC),
                ("image_stride", C.c_int64), ("d_frames", C.c_void_p)]


class HogGridC(C.Structure):
    """sd_hog_grid: one grid of planar features; offsets in floats."""
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("offset", C.c_int64), ("out_offset", C.c_int64)]


class HogGridsC(C.Structure):
    """sd_hog_grids: planar feature grids on the device, equally sized or one descriptor per grid."""
    _fields_ = [("d_features", C.c_void_p), ("count", C.c_int32), ("width", C.c_int32), ("height", C.c_int32),
                ("d_grids", C.c_void_p)]


class HogScoreMapC(C.Structure):
    """sd_hog_score_map: the [Q][height][width] scores of one pyramid level of one frame, at d_scores + offset (floats)."""
    _fields_ = [("frame", C.c_int32), ("level", C.c_int32), ("frame_w", C.c_int32), ("frame_h", C.c_int32), ("level_w", C.c_int32),
                ("level_h", C.c_int32), ("width", C.c_int32), ("height", C.c_int32), ("offset", C.c_int64)]


class HogDetectionC(C.Structure):
    """sd_hog_detection: a box in frame pixels (x, y, w, h), its score, filter, level and score position."""
    _fields_ = [("x", C.c_int32), ("y", C.c_int32), ("w", C.c_int32), ("h", C.c_int32), ("score", C.c_float),
                ("filter", C.c_int32), ("level", C.c_int32), ("cell_x", C.c_int32), ("cell_y", C.c_int32)]


class HogWindowC(C.Structure):
    """sd_hog_window: score position (x, y) of grid `grid`; flip = 1 reads the window of the mirrored image."""
    _fields_ = [("grid", C.c_int32), ("x", C.c_int32), ("y", C.c_int32), ("flip", C.c_int32)]


class SvmReportC(C.Structure):
    """sd_svm_report: Newton steps, final |S|, stop reason (0 converged, 1 no decrease, 2 iteration cap) and f in float64."""
    _fields_ = [("iterations", C.c_int32), ("active", C.c_int32), ("stop", C.c_int32), ("reserved", C.c_int32),
                ("objective", C.c_double)]


class HogBoxC(C.Structure):
    """sd_hog_box: a ground-truth box (x, y, w, h) in pixels of frame `frame`."""
    _fields_ = [("frame", C.c_int32), ("x", C.c_int32), ("y", C.c_int32), ("w", C.c_int32), ("h", C.c_int32)]


class HogTrainParamC(C.Structure):
    """sd_hog_train_param: the training rule's parameters (include/sd_b200.h, sd_hog_train_filter)."""
    _fields_ = [("lambda_", C.c_float), ("positive_overlap", C.c_float), ("negative_overlap", C.c_float),
                ("flip_positives", C.c_int32), ("rounds", C.c_int32), ("negatives_per_frame", C.c_int32),
                ("mine_overlap", C.c_float), ("max_negatives", C.c_int32), ("max_iterations", C.c_int32)]


class HogTrainReportC(C.Structure):
    """sd_hog_train_report: one mining round and its solve."""
    _fields_ = [("positives", C.c_int32), ("unassigned", C.c_int32), ("cache", C.c_int32), ("mined", C.c_int32),
                ("excluded", C.c_int32), ("added", C.c_int32), ("evicted", C.c_int32), ("truncated", C.c_int32),
                ("solved", C.c_int32), ("reserved", C.c_int32), ("solve", SvmReportC), ("pyramid_ms", C.c_float),
                ("scores_ms", C.c_float), ("detect_ms", C.c_float), ("host_ms", C.c_float), ("gather_ms", C.c_float),
                ("solve_ms", C.c_float), ("gathered_bytes", C.c_double)]


class HostFrameC(C.Structure):
    """sd_host_frame: one host frame of a detect call (8UC1, or 8UC3 interleaved B, G, R)."""
    _fields_ = [("h_data", C.c_void_p), ("width", C.c_int32), ("height", C.c_int32), ("row_stride", C.c_int32), ("channels", C.c_int32)]


class LevelFramesC(C.Structure):
    """sd_level_frames: where a cascade level's frames are (a device batch or host frames) and which frame each sample reads."""
    _fields_ = [("images", C.POINTER(ImageBatchC)), ("host_frames", C.POINTER(HostFrameC)), ("num_host_frames", C.c_int32),
                ("d_sample_frame", C.c_void_p), ("stage_half_bytes", C.c_size_t)]


# sd_project_fn(user, ctx, level, d_x, ldx, first_row, rows, d_out, ld) -> 0 or non-zero
ProjectFn = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.c_void_p, C.c_int64)


class LevelProjectionC(C.Structure):
    """sd_level_projection: the callback that writes a level's feature rows on the device, and its feature length."""
    _fields_ = [("fn", ProjectFn), ("user", C.c_void_p), ("level", C.c_int32), ("feature_length", C.c_int32)]


# sd_host_project_fn(user, level, h_x, ldx, first_row, rows, h_out, ld_out) -> 0 or non-zero
HostProjectFn = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.c_void_p, C.c_int64)


class LevelHostProjectionC(C.Structure):
    """sd_level_host_projection: the host callback that fills a level's feature rows in pinned staging, its feature length and
    the staging-half size (0: the library's default)."""
    _fields_ = [("fn", HostProjectFn), ("user", C.c_void_p), ("level", C.c_int32), ("feature_length", C.c_int32),
                ("stage_half_bytes", C.c_size_t)]


# every symbol declared in include/sd_b200.h (tests/test_abi.py checks the list against the header)
EXPORTS = [
    "sd_ctx_create", "sd_ctx_destroy", "sd_last_error", "sd_sync", "sd_ctx_stream", "sd_version", "sd_launch_count", "sd_roi_fallback_count",
    "sd_malloc", "sd_free", "sd_host_alloc", "sd_host_free", "sd_memcpy_h2d", "sd_memcpy_d2h", "sd_memset",
    "sd_memcpy2d_h2d", "sd_memcpy2d_d2h", "sd_memcpy2d_d2d",
    "sd_hog_feature_length", "sd_hog_batch", "sd_hog_debug", "sd_bgr2gray", "sd_upload_frames", "sd_hog_dense_shape", "sd_hog_dense",
    "sd_hog_dense_images", "sd_hog_dense_polar", "sd_hog_permutation", "sd_hog_glyphs", "sd_hog_render", "sd_hog_relayout",
    "sd_hog_pyramid_shape", "sd_hog_pyramid", "sd_hog_correlate", "sd_hog_detections",
    "sd_hog_windows", "sd_hog_box_windows", "sd_learn_squared_hinge", "sd_hog_train_filter",
    "sd_learn", "sd_centre_features", "sd_learn_centred", "sd_learn_rank_revealing", "sd_gram", "sd_solve_gram", "sd_predict", "sd_test_residual", "sd_solver_timings", "sd_set_gram_mode", "sd_set_solver", "sd_solver_iterations",
    "sd_set_rank_diagnostic", "sd_last_rank",
    "sd_comm_get_unique_id", "sd_comm_create", "sd_comm_adopt", "sd_comm_destroy", "sd_comm_rank", "sd_comm_size",
    "sd_comm_sum_int64", "sd_comm_allgather", "sd_allreduce_gram", "sd_reduce_scatter_gram", "sd_solve_gram_dist", "sd_learn_dist",
    "sd_cascade_targets", "sd_cascade_update", "sd_subtract_templates", "sd_level_chunk_rows", "sd_train_level", "sd_apply_level",
    "sd_train_level_projected", "sd_apply_level_projected", "sd_train_level_host_projected", "sd_apply_level_host_projected",
    "sd_gathered_bytes", "sd_host_frame_in_place", "sd_device_memory",
    "sd_model_load", "sd_model_save", "sd_model_create", "sd_model_destroy", "sd_model_num_levels",
    "sd_model_num_landmarks", "sd_model_hog_param", "sd_model_regulariser", "sd_model_normalisation",
    "sd_model_get_mean", "sd_model_get_weights", "sd_model_landmark_id", "sd_align_mean",
    "sd_perturb_box", "sd_normalised_landmark_errors",
    "sd_detect_batch_device", "sd_detect_batch_host", "sd_detect_faces_host", "sd_detect_faces_device",
]

_lib = None


def lib():
    """Loads libsd_b200.so; raises if it has not been built (no fallback)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise SdError(2, f"{LIB_PATH} is missing: run `python -m superviseddescent_b200.build` "
                             f"(the CUDA extension is mandatory, there is no CPU path)")
        l = C.CDLL(LIB_PATH)
        l.sd_last_error.restype = C.c_char_p
        l.sd_version.restype = C.c_char_p
        l.sd_launch_count.restype = C.c_int64
        l.sd_roi_fallback_count.restype = C.c_int64
        l.sd_roi_fallback_count.argtypes = [C.c_void_p]
        l.sd_gathered_bytes.restype = C.c_int64
        l.sd_gathered_bytes.argtypes = [C.c_void_p]
        l.sd_model_landmark_id.restype = C.c_char_p
        l.sd_last_error.argtypes = [C.c_void_p]
        l.sd_launch_count.argtypes = [C.c_void_p]
        l.sd_ctx_destroy.argtypes = [C.c_void_p]
        l.sd_model_destroy.argtypes = [C.c_void_p]
        l.sd_model_landmark_id.argtypes = [C.c_void_p, C.c_int]
        l.sd_comm_destroy.argtypes = [C.c_void_p]
        l.sd_solver_iterations.argtypes = [C.c_void_p]
        l.sd_last_rank.argtypes = [C.c_void_p]
        l.sd_comm_rank.argtypes = [C.c_void_p]
        l.sd_comm_size.argtypes = [C.c_void_p]
        l.sd_ctx_stream.restype = C.c_void_p
        l.sd_ctx_stream.argtypes = [C.c_void_p]
        l.sd_train_level_projected.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(LevelProjectionC), C.c_void_p, C.c_void_p, C.c_int,
                                               C.c_int, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int, C.c_void_p,
                                               C.c_int64, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        l.sd_apply_level_projected.argtypes = [C.c_void_p, C.POINTER(LevelProjectionC), C.c_void_p, C.c_int, C.c_int, C.c_void_p,
                                               C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p]
        l.sd_train_level_host_projected.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(LevelHostProjectionC), C.c_void_p, C.c_void_p,
                                                    C.c_int, C.c_int, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int,
                                                    C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        l.sd_apply_level_host_projected.argtypes = [C.c_void_p, C.POINTER(LevelHostProjectionC), C.c_void_p, C.c_int, C.c_int,
                                                    C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int64, C.c_int,
                                                    C.c_void_p]
        _i = C.c_int
        _ip = C.POINTER(C.c_int)
        l.sd_hog_pyramid_shape.argtypes = [_i, _i, C.c_double, _i, _i, _i, _ip, _ip, _ip, _ip, _ip]
        l.sd_hog_pyramid.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_double), _i, _i, _i, _i, C.c_void_p, C.c_void_p]
        l.sd_hog_correlate.argtypes = [C.c_void_p, C.c_void_p, _i, _i, C.c_void_p, _i, _i, _i, C.c_void_p, _i, _i, C.c_void_p]
        l.sd_hog_detections.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, _i, _i, _i, _i, _i, _i, _i, _i, C.c_float, C.c_double,
                                        _i, _i, C.c_void_p, C.c_void_p, C.c_void_p]
        l.sd_hog_windows.argtypes = [C.c_void_p, C.c_void_p, _i, _i, _i, _i, _i, _i, C.c_void_p, _i, C.c_void_p, C.c_int64]
        l.sd_hog_box_windows.argtypes = [_i, _i, C.c_void_p, _i, _i, _i, _i, _i, _i, _i, _i, C.c_double, C.c_void_p, _i,
                                         C.c_void_p, C.c_void_p]
        l.sd_learn_squared_hinge.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, _i, _i, C.c_float, _i, C.c_void_p,
                                             C.c_void_p]
        l.sd_hog_train_filter.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, _i, C.c_void_p, _i, _i, _i, _i, _i, _i, _i, _i,
                                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        _lib = l
    return _lib


def ptr(t) -> C.c_void_p:
    """Device pointer of a torch tensor (or None / int passthrough)."""
    if t is None:
        return C.c_void_p(0)
    if isinstance(t, int):
        return C.c_void_p(t)
    return C.c_void_p(t.data_ptr())
