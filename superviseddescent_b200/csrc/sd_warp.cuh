// cv::warpAffine's classic fixed-point bilinear rule (INTER_LINEAR | WARP_INVERSE_MAP, BORDER_CONSTANT 0), restated once for
// every kernel that samples a frame through an affine map M (2 x 3, row-major, destination pixel (X, Y) -> frame position):
// the face chips (sd_face_chips.cu), warped HOG samples (hog_patch_kernel, sd_hog.cu) and the host-frame gather's plan of a
// warped patch (roi_plan_kernel, sd_train.cu).  Pinned to cv2 4.13 by tests/face_chip_ref.py.
//
//   adelta[X] = cvRound(M[0] X 1024),  bdelta[X] = cvRound(M[3] X 1024)                  (per destination column)
//   X0[Y] = cvRound((M[1] Y + M[2]) 1024) + 16,  Y0[Y] = cvRound((M[4] Y + M[5]) 1024) + 16   (per destination row)
//   sx = (X0 + adelta) >> 5, sy = (Y0 + bdelta) >> 5: a position on the 1/32 px grid; taps (sx >> 5, sy >> 5) and +1 each way
//   8-bit: 15-bit integer weights (32 - fx) (32 - fy) 32, ...; sum + 2^14 >> 15, clamped to 255.  A tap outside the frame is 0.
#pragma once

#include <climits>
#include <cstdint>

#include "sd_b200.h"

// cvRound of v as an int64 when it fits int32, else false (NaN and infinities included)
__device__ __forceinline__ bool sd_round_int32(double v, long long* out)
{
    const double r = rint(v);
    if (!(r >= (double)INT32_MIN && r <= (double)INT32_MAX)) return false;
    *out = (long long)r;
    return true;
}

__device__ __forceinline__ bool sd_in_int32(long long v) { return v >= INT32_MIN && v <= INT32_MAX; }

// The per-column terms (adelta, bdelta) of destination column X and the per-row terms (X0, Y0) of destination row Y.  Only
// meaningful where sd_warp_fits holds.
__device__ __forceinline__ int2 sd_warp_col(const double* m, double X)
{
    return make_int2((int)__double2ll_rn(__dmul_rn(__dmul_rn(m[0], X), 1024.0)), (int)__double2ll_rn(__dmul_rn(__dmul_rn(m[3], X), 1024.0)));
}
__device__ __forceinline__ int2 sd_warp_row(const double* m, double Y)
{
    return make_int2((int)__double2ll_rn(__dmul_rn(__dadd_rn(__dmul_rn(m[1], Y), m[2]), 1024.0)) + 16,
                     (int)__double2ll_rn(__dmul_rn(__dadd_rn(__dmul_rn(m[4], Y), m[5]), 1024.0)) + 16);
}

// Whether every fixed-point value of the warp of a w x h destination under M fits int32 and, for a frame wider or taller than
// 32,767 px, every tap coordinate fits int16 (where cv2 saturates).  Each term is monotone in its own variable, so the corners
// X in {0, w - 1}, Y in {0, h - 1} bound them all.
__device__ inline bool sd_warp_fits(const double* m, int w, int h, bool int16_taps)
{
    long long ad[2], bd[2], x0[2], y0[2];
    for (int k = 0; k < 2; ++k) {
        const double X = k ? (double)(w - 1) : 0.0, Y = k ? (double)(h - 1) : 0.0;
        if (!sd_round_int32(__dmul_rn(__dmul_rn(m[0], X), 1024.0), &ad[k]) ||
            !sd_round_int32(__dmul_rn(__dmul_rn(m[3], X), 1024.0), &bd[k]) ||
            !sd_round_int32(__dmul_rn(__dadd_rn(__dmul_rn(m[1], Y), m[2]), 1024.0), &x0[k]) ||
            !sd_round_int32(__dmul_rn(__dadd_rn(__dmul_rn(m[4], Y), m[5]), 1024.0), &y0[k]))
            return false;
        x0[k] += 16;
        y0[k] += 16;
        if (!sd_in_int32(x0[k]) || !sd_in_int32(y0[k])) return false;
    }
    for (int i = 0; i < 2; ++i)
        for (int j = 0; j < 2; ++j) {
            const long long sx = x0[i] + ad[j], sy = y0[i] + bd[j];
            if (!sd_in_int32(sx) || !sd_in_int32(sy)) return false;
            if (int16_taps && ((sx >> 10) < -32768 || (sx >> 10) > 32767 || (sy >> 10) < -32768 || (sy >> 10) > 32767)) return false;
        }
    return true;
}

// Whether sample warp w is valid over a frame of fw x fh pixels (include/sd_b200.h): finite, V at least 1 x 1, and sd_warp_fits.
// hog_geometry_kernel (sd_hog.cu) and roi_plan_kernel (sd_train.cu) both ask here, so the gather plans exactly the warps the
// kernel reads.
__device__ inline bool sd_warp_valid(const sd_sample_warp& w, int fw, int fh)
{
    bool ok = w.width >= 1 && w.height >= 1;
    for (int k = 0; k < 6; ++k) ok = ok && isfinite(w.m[k]);
    return ok && sd_warp_fits(w.m, w.width, w.height, fw > 32767 || fh > 32767);
}

// The blend of the four taps at fractions (fx, fy) of 1/32 px: 8-bit frames by 15-bit integer weights, float frames by float
// weights summed left to right
__device__ __forceinline__ uint8_t sd_warp_blend(uint8_t s00, uint8_t s01, uint8_t s10, uint8_t s11, int fx, int fy)
{
    const int acc = (int)s00 * ((32 - fx) * (32 - fy) * 32) + (int)s01 * (fx * (32 - fy) * 32) + (int)s10 * ((32 - fx) * fy * 32) +
                    (int)s11 * (fx * fy * 32);
    return (uint8_t)min((acc + (1 << 14)) >> 15, 255);
}

__device__ __forceinline__ float sd_warp_blend(float s00, float s01, float s10, float s11, int fx, int fy)
{
    const float wx1 = fx * (1.0f / 32), wy1 = fy * (1.0f / 32), wx0 = 1.0f - wx1, wy0 = 1.0f - wy1;   // exact
    float v = __fmul_rn(s00, __fmul_rn(wx0, wy0));
    v = __fadd_rn(v, __fmul_rn(s01, __fmul_rn(wx1, wy0)));
    v = __fadd_rn(v, __fmul_rn(s10, __fmul_rn(wx0, wy1)));
    return __fadd_rn(v, __fmul_rn(s11, __fmul_rn(wx1, wy1)));
}

// The warped value at grid position (sx, sy) (1/32 px), from tap(x, y): the frame's pixel, 0 outside the frame
template <class T, class Tap>
__device__ __forceinline__ T sd_warp_sample(int sx, int sy, Tap tap)
{
    const int x = sx >> 5, y = sy >> 5;
    return sd_warp_blend(tap(x, y), tap(x + 1, y), tap(x, y + 1), tap(x + 1, y + 1), sx & 31, sy & 31);
}
