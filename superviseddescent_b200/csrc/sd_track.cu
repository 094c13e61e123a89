// Face tracking on the device: the face box of a set of landmarks (sd_track_boxes), a HOG filter's score at a box
// (sd_hog_box_scores) and one tracking step that chains them around the detect cascade (sd_track_faces) -- the loop
// apps/rcr/rcr-track.cpp:168-177 sketches (re-align the mean to the previous landmarks' box) with the end of track it leaves open.
#include "sd_internal.cuh"

#include <algorithm>
#include <cmath>
#include <vector>

namespace {

// crops, features and scores of one slice of sd_hog_box_scores stay below this many bytes (one box at least)
constexpr size_t kBoxSliceBytes = size_t(64) << 20;

struct MeanExtent {
    float x0, x1, y0, y1;
};

// Rule 1 of include/sd_b200.h (sd_track_boxes): the box of row x (2L floats).  False for a degenerate box.
__device__ __forceinline__ bool track_box(const float* __restrict__ x, int L, const MeanExtent& m, int b[4])
{
    float lx0 = x[0], lx1 = x[0], ly0 = x[L], ly1 = x[L];
    for (int i = 1; i < L; ++i) {
        lx0 = fminf(lx0, x[i]); lx1 = fmaxf(lx1, x[i]);
        ly0 = fminf(ly0, x[L + i]); ly1 = fmaxf(ly1, x[L + i]);
    }
    const double w = __ddiv_rn(__dadd_rn((double)lx1, -(double)lx0), __dadd_rn((double)m.x1, -(double)m.x0));
    const double h = __ddiv_rn(__dadd_rn((double)ly1, -(double)ly0), __dadd_rn((double)m.y1, -(double)m.y0));
    const double bx = __dadd_rn((double)lx0, -__dmul_rn(__dadd_rn((double)m.x0, 0.5), w));
    const double by = __dadd_rn((double)ly0, -__dmul_rn(__dadd_rn((double)m.y0, 0.5), h));
    const double v[4] = {bx, by, w, h};
    for (int k = 0; k < 4; ++k) {
        const double r = rint(v[k]);                        // cvRound: ties to even; NaN and inf fail the range test
        if (!(r >= -2147483648.0 && r <= 2147483647.0)) return false;
        b[k] = (int)r;
    }
    return b[2] >= 1 && b[3] >= 1;
}

// fminf / fmaxf drop a NaN operand; a NaN landmark must make the box degenerate instead
__device__ __forceinline__ bool row_finite(const float* __restrict__ x, int P)
{
    for (int i = 0; i < P; ++i)
        if (!isfinite(x[i])) return false;
    return true;
}

// sd_track_boxes (x0 == nullptr), or step 1 of sd_track_faces: the box of prev, and x0 = align_mean(mean, B) as sd_align_mean
// computes it (ax, bx in double, then an un-fused float mul and add).  A degenerate box starts its cascade from the mean aligned
// to (0, 0, 1, 1): an empty patch that ends the track anyway and costs nothing else.  fw > 0 (step 3 of sd_track_faces): a box
// whose context rectangle under an fw x fh filter does not fit in int32 (sd_box_context) is not valid either, so that it
// scores NaN instead of a stand-in crop's score.
__global__ void track_box_kernel(const float* __restrict__ x, int T, int L, MeanExtent me, const float* __restrict__ mean,
                                 int32_t* __restrict__ boxes, uint8_t* __restrict__ valid, float* __restrict__ x0,
                                 uint8_t* __restrict__ patch_flag, int fw, int fh)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= T) return;
    const float* row = x + (long long)t * 2 * L;
    int b[4], r[4];
    const bool box_ok = row_finite(row, 2 * L) && track_box(row, L, me, b);
    if (!box_ok) b[0] = b[1] = b[2] = b[3] = 0;
    const bool ok = box_ok && (fw <= 0 || sd_box_context(b[0], b[1], b[2], b[3], fw, fh, &r[0], &r[1], &r[2], &r[3]));
    if (boxes)
        for (int k = 0; k < 4; ++k) boxes[4 * t + k] = b[k];
    valid[t] = ok;
    if (!x0) return;
    patch_flag[t] = 0;
    const int bw = ok ? b[2] : 1, bh = ok ? b[3] : 1;
    const float ax = (float)(double)bw, ay = (float)(double)bh;
    const float cx = (float)__dadd_rn(__dmul_rn(0.5, (double)bw), (double)b[0]);
    const float cy = (float)__dadd_rn(__dmul_rn(0.5, (double)bh), (double)b[1]);
    float* out = x0 + (long long)t * 2 * L;
    for (int i = 0; i < L; ++i) {
        out[i] = __fadd_rn(__fmul_rn(mean[i], ax), cx);
        out[L + i] = __fadd_rn(__fmul_rn(mean[L + i], ay), cy);
    }
}

// The largest of each box's 3 x 3 scores, first in y then x order on ties; a NaN never wins.  ok (optional): a box whose byte is
// 0 scores NaN.
__global__ void box_max_kernel(const float* __restrict__ s, int n, const uint8_t* __restrict__ ok, float* __restrict__ out)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float best = __int_as_float(0x7fc00000);
    if (!ok || ok[i])
        for (int k = 0; k < 9; ++k) {
            const float v = s[9 * i + k];
            if (v == v && (best != best || v > best)) best = v;
        }
    out[i] = best;
}

// Step 3 of sd_track_faces: the outputs of every track.
__global__ void track_finish_kernel(int T, int P, const float* __restrict__ prev, const float* __restrict__ xn,
                                    const uint8_t* __restrict__ valid_prev, const uint8_t* __restrict__ patch_flag,
                                    const uint8_t* __restrict__ valid_new, const float* __restrict__ scores, float threshold,
                                    float* __restrict__ landmarks, uint8_t* __restrict__ alive)
{
    const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (e >= (long long)T * P) return;
    const int t = (int)(e / P);
    landmarks[e] = valid_prev[t] ? xn[e] : prev[e];
    if (e % P == 0) alive[t] = valid_prev[t] && !patch_flag[t] && valid_new[t] && scores[t] > threshold;
}

MeanExtent mean_extent(const sd_model* m)
{
    const int L = sd_model_num_landmarks(m);
    std::vector<float> mean(2 * L);
    sd_model_get_mean(m, mean.data());
    MeanExtent e;
    e.x0 = *std::min_element(mean.begin(), mean.begin() + L);
    e.x1 = *std::max_element(mean.begin(), mean.begin() + L);
    e.y0 = *std::min_element(mean.begin() + L, mean.end());
    e.y1 = *std::max_element(mean.begin() + L, mean.end());
    return e;
}

// The argument rules of sd_hog_box_scores that need no device data (fn names the entry point in messages).
int box_scores_check(sd_ctx* ctx, const char* fn, const sd_image_batch* images, const float* d_filter, int fw, int fh, int cs, int K,
                     int variant)
{
    if (!images || !d_filter) return sd_fail(ctx, SD_ERR_INVALID, "%s: null argument", fn);
    if (images->d_roi) return sd_fail(ctx, SD_ERR_INVALID, "%s: a batch with regions of interest has no whole frames", fn);
    if (const int rc = sd_hog_check_config(ctx, fn, variant, K, cs)) return rc;
    if (const int rc = sd_hog_check_filter(ctx, fn, fw, fh, 0, 0)) return rc;
    if ((fw + 2) * cs <= 3 || (fh + 2) * cs <= 3) return sd_fail(ctx, SD_ERR_INVALID, "%s: the crop must be wider and taller than 3 px", fn);
    if (!sd_aligned(d_filter, 4)) return sd_fail(ctx, SD_ERR_INVALID, "%s: the filter must be 4-byte aligned", fn);
    return SD_OK;
}

// sd_hog_box_scores past its checks: the boxes in slices of whole boxes whose crops, features and scores fit kBoxSliceBytes.
int box_scores_run(sd_ctx* ctx, const sd_image_batch* images, const int32_t* d_box_frame, const int32_t* d_boxes, const uint8_t* d_ok,
                   int n, const float* d_filter, int fw, int fh, float bias, int cs, int K, int variant, float* d_scores)
{
    if (n == 0) return SD_OK;
    const int cw = (fw + 2) * cs, ch = (fh + 2) * cs, pitch = (int)sd_round16(cw);
    const size_t crop = (size_t)pitch * ch, feat = (size_t)sd_hog_dd(K, variant) * (fw + 2) * (fh + 2) * sizeof(float);
    const size_t per_box = crop + feat + 9 * sizeof(float) + sizeof(int4) + 64;
    const int slice = (int)std::max<size_t>(1, std::min<size_t>((size_t)n, kBoxSliceBytes / per_box));
    const size_t crops_bytes = sd_round16(crop * slice), feat_bytes = sd_round16(feat * slice), sc_bytes = sd_round16(9 * sizeof(float) * slice);
    uint8_t* ws = static_cast<uint8_t*>(sd_workspace(ctx, SD_WS_BOXES, crops_bytes + feat_bytes + sc_bytes + sd_hog_box_table_bytes(slice) + 16));
    if (!ws) return SD_ERR_CUDA;
    uint8_t* crops = ws;
    float* features = reinterpret_cast<float*>(ws + crops_bytes);
    float* sc = reinterpret_cast<float*>(ws + crops_bytes + feat_bytes);
    float* d_bias = reinterpret_cast<float*>(ws + crops_bytes + feat_bytes + sc_bytes);
    void* tables = ws + crops_bytes + feat_bytes + sc_bytes + 16;
    SD_CUDA(ctx, cudaMemcpyAsync(d_bias, &bias, sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
    for (int b0 = 0; b0 < n; b0 += slice) {
        const int m = std::min(slice, n - b0);
        const uint8_t* ok = d_ok ? d_ok + b0 : nullptr;
        if (const int rc = sd_hog_box_crops(ctx, images, d_box_frame + b0, d_boxes + 4 * (size_t)b0, ok, m, fw, fh, cs, crops, pitch, tables))
            return rc;
        sd_image_batch cb{};
        cb.d_data = crops;
        cb.width = cw; cb.height = ch; cb.row_stride = pitch;
        cb.image_stride = (int64_t)crop;
        cb.count = m;
        if (const int rc = sd_hog_dense(ctx, &cb, cs, K, variant, features, nullptr)) return rc;
        sd_hog_grids g{};
        g.d_features = features;
        g.count = m;
        g.width = fw + 2; g.height = fh + 2;
        if (const int rc = sd_hog_correlate(ctx, &g, K, variant, d_filter, 1, fw, fh, d_bias, 0, 0, sc)) return rc;
        box_max_kernel<<<sd_div_up(m, 128), 128, 0, ctx->stream>>>(sc, m, ok, d_scores + b0);
        SD_LAUNCH_CHECK(ctx, "box_max_kernel");
    }
    return SD_OK;
}

}  // namespace

extern "C" {

int sd_track_boxes(sd_ctx* ctx, const sd_model* m, const float* d_landmarks, int T, int32_t* d_boxes, uint8_t* d_valid)
{
    if (!ctx) return SD_ERR_INVALID;
    SD_REQUIRE(ctx, m && d_landmarks && d_boxes && d_valid && T >= 0, "bad argument");
    if (T == 0) return SD_OK;
    track_box_kernel<<<sd_div_up(T, 128), 128, 0, ctx->stream>>>(d_landmarks, T, sd_model_num_landmarks(m), mean_extent(m), nullptr,
                                                                 d_boxes, d_valid, nullptr, nullptr, 0, 0);
    SD_LAUNCH_CHECK(ctx, "track_box_kernel");
    return SD_OK;
}

int sd_hog_box_scores(sd_ctx* ctx, const sd_image_batch* images, const int32_t* d_box_frame, const int32_t* d_boxes, int n,
                      const float* d_filter, int filter_w, int filter_h, float bias, int cell_size, int num_bins, int variant,
                      float* d_scores)
{
    if (!ctx) return SD_ERR_INVALID;
    if (const int rc = box_scores_check(ctx, __func__, images, d_filter, filter_w, filter_h, cell_size, num_bins, variant)) return rc;
    SD_REQUIRE(ctx, n >= 0 && d_scores && (n == 0 || (d_box_frame && d_boxes)), "bad argument");
    SD_REQUIRE(ctx, sd_aligned(d_scores, 4) && sd_aligned(d_box_frame, 4) && sd_aligned(d_boxes, 4), "pointers must be 4-byte aligned");
    if (n == 0) return SD_OK;
    SD_REQUIRE(ctx, images->d_data && images->count >= 1, "no frames");
    std::vector<int32_t> frame, box;
    if (const int rc = sd_fetch_table(ctx, d_box_frame, n, frame)) return rc;
    if (const int rc = sd_fetch_table(ctx, d_boxes, 4 * n, box)) return rc;
    std::vector<sd_frame> fr;
    if (images->d_frames) {
        if (const int rc = sd_fetch_table(ctx, images->d_frames, images->count, fr)) return rc;
    } else {
        SD_REQUIRE(ctx, images->count == 1 || images->image_stride > 0, "bad strides");
        fr.assign(1, sd_frame{images->width, images->height, images->row_stride, 0, 0});
    }
    for (const sd_frame& d : fr)
        SD_REQUIRE(ctx, d.width >= 1 && d.height >= 1 && d.row_stride >= d.width && d.offset >= 0, "a frame is smaller than 1 x 1 or has "
                   "row_stride < width or a negative offset");
    for (int i = 0; i < n; ++i) {
        if (frame[i] < 0 || frame[i] >= images->count)
            return sd_fail(ctx, SD_ERR_INVALID, "%s: box %d refers to frame %d of %d", __func__, i, frame[i], images->count);
        int rx, ry, rw, rh;
        if (!sd_box_context(box[4 * i], box[4 * i + 1], box[4 * i + 2], box[4 * i + 3], filter_w, filter_h, &rx, &ry, &rw, &rh))
            return sd_fail(ctx, SD_ERR_INVALID, "%s: box %d has w or h < 1 or a context rectangle outside int32", __func__, i);
    }
    return box_scores_run(ctx, images, d_box_frame, d_boxes, nullptr, n, d_filter, filter_w, filter_h, bias, cell_size, num_bins,
                          variant, d_scores);
}

int sd_track_faces(sd_ctx* ctx, const sd_model* m, const sd_image_batch* images, const int32_t* d_track_frame, const float* d_prev,
                   int T, const float* d_filter, int filter_w, int filter_h, float bias, int cell_size, int num_bins, int variant,
                   float threshold, float* d_landmarks, int32_t* d_boxes, float* d_scores, uint8_t* d_alive)
{
    if (!ctx) return SD_ERR_INVALID;
    SD_REQUIRE(ctx, m && T >= 0, "bad argument");
    if (const int rc = box_scores_check(ctx, __func__, images, d_filter, filter_w, filter_h, cell_size, num_bins, variant)) return rc;
    if (T == 0) return SD_OK;
    SD_REQUIRE(ctx, images->d_data && d_track_frame && d_prev && d_landmarks && d_boxes && d_scores && d_alive, "null argument");
    // The frame table (d_frames) is trusted as sd_detect_faces_device trusts it: reading it back to check it would cost the step a
    // second read-back.  sd_hog_box_scores, which reads its tables back anyway, checks it.
    const int L = sd_model_num_landmarks(m), P = 2 * L;
    // [x0 | new landmarks | B valid | patch flags | B' valid], each 16-byte aligned
    const size_t xb = sd_round16((size_t)T * P * sizeof(float)), fb = sd_round16((size_t)T);
    uint8_t* ws = static_cast<uint8_t*>(sd_workspace(ctx, SD_WS_TRACK, 2 * xb + 3 * fb));
    if (!ws) return SD_ERR_CUDA;
    float* x0 = reinterpret_cast<float*>(ws);
    float* xn = reinterpret_cast<float*>(ws + xb);
    uint8_t* valid_prev = ws + 2 * xb;
    uint8_t* patch_flag = valid_prev + fb;
    uint8_t* valid_new = patch_flag + fb;
    const MeanExtent me = mean_extent(m);
    const int blocks = sd_div_up(T, 128);
    track_box_kernel<<<blocks, 128, 0, ctx->stream>>>(d_prev, T, L, me, sd_model_device_mean(m), nullptr, valid_prev, x0, patch_flag,
                                                      0, 0);
    SD_LAUNCH_CHECK(ctx, "track_box_kernel");
    if (const int rc = sd_detect_device(ctx, m, images, d_track_frame, x0, T, xn, patch_flag)) return rc;
    // detect's one read-back: a frame index out of range refuses the call; the empty patches are per-track flags here
    int* h = reinterpret_cast<int*>(ctx->h_scratch) + 1;
    int* d = reinterpret_cast<int*>(ctx->d_scratch) + 1;
    SD_CUDA(ctx, cudaMemcpyAsync(h, d, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    SD_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    const int st = *h;
    if (st) SD_CUDA(ctx, cudaMemsetAsync(d, 0, sizeof(int), ctx->stream));
    if (st & 2) return sd_fail(ctx, SD_ERR_INVALID, "%s: frame index out of range", __func__);
    track_box_kernel<<<blocks, 128, 0, ctx->stream>>>(xn, T, L, me, nullptr, d_boxes, valid_new, nullptr, nullptr, filter_w, filter_h);
    SD_LAUNCH_CHECK(ctx, "track_box_kernel");
    if (const int rc = box_scores_run(ctx, images, d_track_frame, d_boxes, valid_new, T, d_filter, filter_w, filter_h, bias, cell_size,
                                      num_bins, variant, d_scores))
        return rc;
    track_finish_kernel<<<sd_div_up((long long)T * P, 256), 256, 0, ctx->stream>>>(T, P, d_prev, xn, valid_prev, patch_flag, valid_new,
                                                                                  d_scores, threshold, d_landmarks, d_alive);
    SD_LAUNCH_CHECK(ctx, "track_finish_kernel");
    return SD_OK;
}

}  // extern "C"
