"""The crop of sd_hog_box_scores_images (include/sd_b200.h) restated in numpy: the context rectangle of a box (track_ref), each
channel cut from it with pixels outside the frame 0 (copyMakeBorder BORDER_CONSTANT) and resized on its own, 8-bit frames by the
oracle's cv::resize INTER_LINEAR 8-bit rule and float frames by hog_resize_f32_ref's float rule.  The crop is (ch, cw) for one
channel and (ch, cw, C) for frames of C channels, channels last."""
import numpy as np

import hog_resize_f32_ref
import track_ref


def padded_roi(frame, rect):
    """The pixels of rect (x, y, w, h) of an (H, W) or (H, W, C) frame, 0 outside it."""
    a = np.asarray(frame)
    H, W = a.shape[:2]
    x, y, w, h = rect
    pad = max(0, -x, -y, x + w - W, y + h - H)
    p = np.pad(a, ((pad, pad), (pad, pad)) + ((0, 0),) * (a.ndim - 2))
    return np.ascontiguousarray(p[y + pad:y + pad + h, x + pad:x + pad + w])


def box_crop(oracle, frame, box, fw, fh, cell_size):
    """The (fh + 2) cs x (fw + 2) cs crop of box in frame (uint8 or float32, (H, W) or (H, W, C))."""
    roi = padded_roi(frame, track_ref.context_rect(box, fw, fh))
    cw, ch = (fw + 2) * cell_size, (fh + 2) * cell_size
    if roi.dtype == np.float32:
        return hog_resize_f32_ref.resize_f32(roi, cw, ch)
    if roi.ndim == 2:
        return oracle.resize_linear_u8(roi, cw, ch)
    return np.stack([oracle.resize_linear_u8(np.ascontiguousarray(roi[:, :, c]), cw, ch) for c in range(roi.shape[2])], axis=-1)
