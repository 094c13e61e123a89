// Face tracking on the device: the face box of a set of landmarks (sd_track_boxes), a HOG filter's score at a box
// (sd_hog_box_scores, and sd_hog_box_scores_images on frames that keep their channels) and one tracking step that chains
// them around the detect cascade (sd_track_faces) -- the loop apps/rcr/rcr-track.cpp:168-177 sketches (re-align the mean to
// the previous landmarks' box) with the end of track it leaves open -- and the step with the sliding-window detector inside
// it, which starts and merges tracks (sd_track_detect_faces).  The _images steps score and detect on colour or float frames
// while the cascade reads their grey.
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

// out = align_mean(mean, (bx, by, bw, bh)) at scaling 1 and translation 0, as sd_align_mean computes it (ax, bx in double, then an
// un-fused float mul and add)
__device__ __forceinline__ void align_mean_row(const float* __restrict__ mean, int L, int bx, int by, int bw, int bh, float* __restrict__ out)
{
    const float ax = (float)(double)bw, ay = (float)(double)bh;
    const float cx = (float)__dadd_rn(__dmul_rn(0.5, (double)bw), (double)bx);
    const float cy = (float)__dadd_rn(__dmul_rn(0.5, (double)bh), (double)by);
    for (int i = 0; i < L; ++i) {
        out[i] = __fadd_rn(__fmul_rn(mean[i], ax), cx);
        out[L + i] = __fadd_rn(__fmul_rn(mean[L + i], ay), cy);
    }
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
    align_mean_row(mean, L, b[0], b[1], ok ? b[2] : 1, ok ? b[3] : 1, x0 + (long long)t * 2 * L);
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

// The rules an sd_hog_images batch of the _images entry points meets before any device data is read: those of
// sd_hog_pyramid_images / sd_hog_pyramid_float (dtype, channels, orientation assignment, frame count, data, alignment).
int images_check(sd_ctx* ctx, const char* fn, const sd_hog_images* images, int bilinear_orientations)
{
    if (!images) return sd_fail(ctx, SD_ERR_INVALID, "%s: null argument", fn);
    if (images->dtype != SD_HOG_U8 && images->dtype != SD_HOG_F32)
        return sd_fail(ctx, SD_ERR_INVALID, "%s: dtype must be SD_HOG_U8 or SD_HOG_F32", fn);
    if (images->channels < 1 || images->channels > 16) return sd_fail(ctx, SD_ERR_INVALID, "%s: channels must be in [1,16]", fn);
    if (bilinear_orientations != 0 && bilinear_orientations != 1)
        return sd_fail(ctx, SD_ERR_INVALID, "%s: bilinear_orientations must be 0 or 1", fn);
    if (images->count < 0) return sd_fail(ctx, SD_ERR_INVALID, "%s: negative frame count", fn);
    if (images->count > 0 && !images->d_data) return sd_fail(ctx, SD_ERR_INVALID, "%s: null argument", fn);
    if (images->dtype == SD_HOG_F32 && !sd_aligned(images->d_data, 4))
        return sd_fail(ctx, SD_ERR_INVALID, "%s: float frames must be 4-byte aligned", fn);
    return SD_OK;
}

// The frames of a source, read on the host (the frame table read back once) by the rules of its kind.
int read_frames(sd_ctx* ctx, const char* fn, const BoxFrames& src, HogPyramidFrames* out)
{
    return src.grey ? sd_hog_read_grey_frames(ctx, fn, src.grey, out) : sd_hog_read_image_frames(ctx, fn, src.images, src.bilinear, out);
}

// sd_hog_box_scores past its checks: the boxes in slices of whole boxes whose crops, features and scores fit kBoxSliceBytes.  A
// crop holds every channel of the source at its element size, so the slices shrink as the channels and the element size grow.
int box_scores_run(sd_ctx* ctx, const BoxFrames& src, const int32_t* d_box_frame, const int32_t* d_boxes, const uint8_t* d_ok,
                   int n, const float* d_filter, int fw, int fh, float bias, int cs, int K, int variant, float* d_scores)
{
    if (n == 0) return SD_OK;
    const int C = src.channels(), es = src.dtype() == SD_HOG_F32 ? 4 : 1;
    const int cw = (fw + 2) * cs, ch = (fh + 2) * cs, pitch = (int)sd_round16((size_t)cw * C * es);
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
        if (const int rc = sd_hog_box_crops(ctx, src, d_box_frame + b0, d_boxes + 4 * (size_t)b0, ok, m, fw, fh, cs, crops, pitch, tables))
            return rc;
        // the crops, channels last; one 8-bit channel with nearest bins is sd_hog_dense's batch
        sd_hog_images cb{};
        cb.d_data = crops;
        cb.dtype = src.dtype();
        cb.channels = C;
        cb.count = m;
        cb.frame = sd_hog_image{cw, ch, 0, pitch / es, C, 1};
        cb.image_stride = (int64_t)(crop / es);
        if (const int rc = sd_hog_dense_images(ctx, &cb, cs, K, variant, src.bilinear, features, nullptr)) return rc;
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

// Step 3 of sd_track_faces for T rows whose cascade from x0 gave xn: B' = the box of xn (d_boxes) and whether it can be scored,
// its score on the frames of src (d_scores), and each row's landmarks (prev where valid_prev is 0) and alive byte.
int track_rescore(sd_ctx* ctx, const BoxFrames& src, const int32_t* d_frame, const float* prev, const float* xn, int T, int L,
                  const MeanExtent& me, const uint8_t* valid_prev, const uint8_t* patch_flag, uint8_t* valid_new, const float* d_filter,
                  int fw, int fh, float bias, int cs, int K, int variant, float threshold, float* d_landmarks, int32_t* d_boxes,
                  float* d_scores, uint8_t* d_alive)
{
    track_box_kernel<<<sd_div_up(T, 128), 128, 0, ctx->stream>>>(xn, T, L, me, nullptr, d_boxes, valid_new, nullptr, nullptr, fw, fh);
    SD_LAUNCH_CHECK(ctx, "track_box_kernel");
    if (const int rc = box_scores_run(ctx, src, d_frame, d_boxes, valid_new, T, d_filter, fw, fh, bias, cs, K, variant, d_scores))
        return rc;
    const int P = 2 * L;
    track_finish_kernel<<<sd_div_up((long long)T * P, 256), 256, 0, ctx->stream>>>(T, P, prev, xn, valid_prev, patch_flag, valid_new,
                                                                                  d_scores, threshold, d_landmarks, d_alive);
    SD_LAUNCH_CHECK(ctx, "track_finish_kernel");
    return SD_OK;
}

// ---- sd_track_detect_faces --------------------------------------------------------------------------------------------------
// Rows are grouped by frame twice: the old rows alive after step 3 (for the association) and all rows alive after it (for the
// merge).  A group is a count per frame (integer atomics), an exclusive scan and a fill whose order within a frame depends on
// the order atomics land; the association only asks whether some row of the frame overlaps, and the merge sorts each frame's
// rows on a total key first, so no result depends on that order.

constexpr size_t kDetectSliceFloats = size_t(64) << 20;   // pyramid features of one slice of the listed frames: 256 MB
constexpr int kScanThreads = 1024;
constexpr int kMergeThreads = 256;
constexpr int kMergeSmemRows = 1024;                      // a frame with more alive rows sorts and suppresses them in global scratch

// the overlap rule of sd_track_detect_faces (include/sd_b200.h) for boxes (x, y, w, h)
__device__ __forceinline__ bool boxes_overlap(int4 a, int4 b, double overlap)
{
    const long long iw = min((long long)a.x + a.z, (long long)b.x + b.z) - max(a.x, b.x);
    const long long ih = min((long long)a.y + a.w, (long long)b.y + b.w) - max(a.y, b.y);
    const long long inter = iw > 0 && ih > 0 ? iw * ih : 0;
    const long long uni = (long long)a.z * a.w + (long long)b.z * b.w - inter;
    return (double)inter > overlap * (double)uni;
}

__device__ __forceinline__ int4 row_box(const int32_t* __restrict__ boxes, int r)
{
    const int32_t* b = boxes + 4 * (long long)r;
    return make_int4(b[0], b[1], b[2], b[3]);
}

// rows r < n with alive[r], counted per frame
__global__ void group_count_kernel(const int32_t* __restrict__ frame, const uint8_t* __restrict__ alive, int n, int* __restrict__ count)
{
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r < n && alive[r]) atomicAdd(count + frame[r], 1);
}

// out[i] = in[0] + ... + in[i - 1] for i <= n, in one CTA
__global__ void __launch_bounds__(kScanThreads) scan_kernel(const int* __restrict__ in, int n, int* __restrict__ out)
{
    __shared__ int warp_sum[kScanThreads / 32];
    __shared__ int carry;
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    if (tid == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < n; base += kScanThreads) {
        const int i = base + tid;
        const int v = i < n ? in[i] : 0;
        int x = v;
        for (int d = 1; d < 32; d <<= 1) {
            const int y = __shfl_up_sync(0xFFFFFFFFu, x, d);
            if (lane >= d) x += y;
        }
        if (lane == 31) warp_sum[w] = x;
        __syncthreads();
        if (w == 0) {
            int s = warp_sum[lane];
            for (int d = 1; d < 32; d <<= 1) {
                const int y = __shfl_up_sync(0xFFFFFFFFu, s, d);
                if (lane >= d) s += y;
            }
            warp_sum[lane] = s;
        }
        __syncthreads();
        const int excl = carry + (w ? warp_sum[w - 1] : 0) + x - v;
        if (i < n) out[i] = excl;
        __syncthreads();
        if (tid == kScanThreads - 1) carry = excl + v;
        __syncthreads();
    }
    if (tid == 0) out[n] = carry;
}

// each counted row into its frame's list at offset[frame]; count runs back down to 0
__global__ void group_fill_kernel(const int32_t* __restrict__ frame, const uint8_t* __restrict__ alive, int n, const int* __restrict__ offset,
                                  int* __restrict__ count, int* __restrict__ list)
{
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n || !alive[r]) return;
    const int f = frame[r];
    list[offset[f] + atomicSub(count + f, 1) - 1] = r;
}

// Step 3: keep[s] = 1 for detection slot s (listed frame s / max_det, detection s % max_det) that holds a detection no alive old
// row of its frame overlaps.
__global__ void associate_kernel(const sd_hog_detection* __restrict__ det, const int32_t* __restrict__ det_count,
                                 const int32_t* __restrict__ det_frame, int slots, int max_det, const int32_t* __restrict__ boxes,
                                 const int* __restrict__ offset, const int* __restrict__ list, double overlap, int* __restrict__ keep)
{
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= slots) return;
    const int i = s / max_det;
    int k = 0;
    if (s - i * max_det < det_count[i]) {
        const sd_hog_detection d = det[s];
        const int4 a = make_int4(d.x, d.y, d.w, d.h);
        const int f = det_frame[i];
        k = 1;
        for (int j = offset[f]; j < offset[f + 1] && k; ++j) k = !boxes_overlap(row_box(boxes, list[j]), a, overlap);
    }
    keep[s] = k;
}

// Step 4: kept slot s becomes row T + dest[s]: its frame, and x0 = align_mean(mean, box) (row dest[s] of x0)
__global__ void new_rows_kernel(const sd_hog_detection* __restrict__ det, const int32_t* __restrict__ det_frame, int slots, int max_det,
                                const int* __restrict__ keep, const int* __restrict__ dest, const float* __restrict__ mean, int L, int T,
                                int32_t* __restrict__ frame, float* __restrict__ x0)
{
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= slots || !keep[s]) return;
    const sd_hog_detection d = det[s];
    frame[T + dest[s]] = det_frame[s / max_det];
    align_mean_row(mean, L, d.x, d.y, d.w, d.h, x0 + (long long)dest[s] * 2 * L);
}

// order-preserving: a larger float gives a larger key; -0 and +0 give one key
__device__ __forceinline__ unsigned score_key(float s)
{
    const unsigned b = __float_as_uint(s == 0.f ? 0.f : s);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

// Step 5, one CTA per frame: its alive rows sorted by the key (old row, score, -row) descending (a rank sort; keys are unique),
// then greedy suppression in that order; a suppressed row's alive byte is cleared.  Frames of more than kMergeSmemRows rows use
// the global scratch (two keys and one byte per row, at the frame's offset) instead of shared memory.
__global__ void __launch_bounds__(kMergeThreads) merge_kernel(const int* __restrict__ offset, const int* __restrict__ list, int T,
                                                              const int32_t* __restrict__ boxes, const float* __restrict__ scores,
                                                              double overlap, unsigned long long* __restrict__ g_key,
                                                              unsigned long long* __restrict__ g_sorted, uint8_t* __restrict__ g_removed,
                                                              uint8_t* __restrict__ alive)
{
    __shared__ unsigned long long s_key[kMergeSmemRows], s_sorted[kMergeSmemRows];
    __shared__ uint8_t s_removed[kMergeSmemRows];
    const int f = blockIdx.x, tid = threadIdx.x;
    const int o = offset[f], n = offset[f + 1] - o;
    if (n < 2) return;
    const bool smem = n <= kMergeSmemRows;
    unsigned long long* key = smem ? s_key : g_key + o;
    unsigned long long* sorted = smem ? s_sorted : g_sorted + o;
    uint8_t* removed = smem ? s_removed : g_removed + o;
    for (int i = tid; i < n; i += kMergeThreads) {
        const int r = list[o + i];
        key[i] = ((unsigned long long)(r < T) << 63) | ((unsigned long long)score_key(scores[r]) << 31) | (unsigned)(0x7FFFFFFF - r);
        removed[i] = 0;
    }
    __syncthreads();
    for (int i = tid; i < n; i += kMergeThreads) {
        const unsigned long long k = key[i];
        int rank = 0;
        for (int j = 0; j < n; ++j) rank += key[j] > k;
        sorted[rank] = k;
    }
    __syncthreads();
    auto row_of = [](unsigned long long k) { return 0x7FFFFFFF - (int)(k & 0x7FFFFFFFu); };
    for (int i = 0; i < n; ++i) {
        if (removed[i]) continue;                                  // uniform: written before the last barrier
        const int4 bi = row_box(boxes, row_of(sorted[i]));
        for (int j = i + 1 + tid; j < n; j += kMergeThreads)
            if (!removed[j] && boxes_overlap(bi, row_box(boxes, row_of(sorted[j])), overlap)) removed[j] = 1;
        __syncthreads();
    }
    for (int i = tid; i < n; i += kMergeThreads)
        if (removed[i]) alive[row_of(sorted[i])] = 0;
}

// The rows r < n with alive[r] grouped by their frame in [0, F): offset[F + 1], list[n]; count[F + 1] is scratch.
int group_rows(sd_ctx* ctx, const int32_t* d_frame, const uint8_t* d_alive, int n, int F, int* count, int* offset, int* list)
{
    SD_CUDA(ctx, cudaMemsetAsync(count, 0, sizeof(int) * (F + 1), ctx->stream));
    if (n > 0) {
        group_count_kernel<<<sd_div_up(n, 256), 256, 0, ctx->stream>>>(d_frame, d_alive, n, count);
        SD_LAUNCH_CHECK(ctx, "group_count_kernel");
    }
    scan_kernel<<<1, kScanThreads, 0, ctx->stream>>>(count, F, offset);
    SD_LAUNCH_CHECK(ctx, "scan_kernel");
    if (n > 0) {
        group_fill_kernel<<<sd_div_up(n, 256), 256, 0, ctx->stream>>>(d_frame, d_alive, n, offset, count, list);
        SD_LAUNCH_CHECK(ctx, "group_fill_kernel");
    }
    return SD_OK;
}

// sd_hog_box_scores and sd_hog_box_scores_images past the checks that need no device data: the frame index and box tables and the
// frame table read back once, every frame and box checked, then the scores.
int box_scores_entry(sd_ctx* ctx, const char* fn, const BoxFrames& src, const int32_t* d_box_frame, const int32_t* d_boxes, int n,
                     const float* d_filter, int fw, int fh, float bias, int cs, int K, int variant, float* d_scores)
{
    if (!(n >= 0 && d_scores && (n == 0 || (d_box_frame && d_boxes)))) return sd_fail(ctx, SD_ERR_INVALID, "%s: bad argument", fn);
    if (!(sd_aligned(d_scores, 4) && sd_aligned(d_box_frame, 4) && sd_aligned(d_boxes, 4)))
        return sd_fail(ctx, SD_ERR_INVALID, "%s: pointers must be 4-byte aligned", fn);
    if (n == 0) return SD_OK;
    if (!src.data() || src.count() < 1) return sd_fail(ctx, SD_ERR_INVALID, "%s: no frames", fn);
    std::vector<int32_t> frame, box;
    if (const int rc = sd_fetch_table(ctx, d_box_frame, n, frame)) return rc;
    if (const int rc = sd_fetch_table(ctx, d_boxes, 4 * n, box)) return rc;
    HogPyramidFrames fr;
    if (const int rc = read_frames(ctx, fn, src, &fr)) return rc;
    for (int i = 0; i < n; ++i) {
        if (frame[i] < 0 || frame[i] >= src.count())
            return sd_fail(ctx, SD_ERR_INVALID, "%s: box %d refers to frame %d of %d", fn, i, frame[i], src.count());
        int rx, ry, rw, rh;
        if (!sd_box_context(box[4 * i], box[4 * i + 1], box[4 * i + 2], box[4 * i + 3], fw, fh, &rx, &ry, &rw, &rh))
            return sd_fail(ctx, SD_ERR_INVALID, "%s: box %d has w or h < 1 or a context rectangle outside int32", fn, i);
    }
    return box_scores_run(ctx, src, d_box_frame, d_boxes, nullptr, n, d_filter, fw, fh, bias, cs, K, variant, d_scores);
}

// The rule of the _images tracking steps: frame f of src has the size of frame f of the grey batch images, for every f.  Each
// frame table is read back once; *fr receives src's frames (read by its rules) for the detector.
int match_frames(sd_ctx* ctx, const char* fn, const sd_image_batch* images, const BoxFrames& src, HogPyramidFrames* fr)
{
    const int F = images->count;
    if (src.count() != F)
        return sd_fail(ctx, SD_ERR_INVALID, "%s: filter_images has %d frames and images %d", fn, src.count(), F);
    if (F <= 0) return SD_OK;
    if (const int rc = read_frames(ctx, fn, src, fr)) return rc;
    std::vector<sd_frame> grey;
    if (images->d_frames) {
        if (const int rc = sd_fetch_table(ctx, images->d_frames, F, grey)) return rc;
    } else {
        grey.assign(1, sd_frame{images->width, images->height, images->row_stride, 0, 0});
    }
    for (int f = 0; f < F; ++f) {
        const sd_frame& g = grey[images->d_frames ? f : 0];
        const sd_hog_image& d = fr->frames[f];
        if (g.width != d.width || g.height != d.height)
            return sd_fail(ctx, SD_ERR_INVALID, "%s: frame %d of filter_images is %d x %d and of images %d x %d", fn, f, d.width, d.height,
                           g.width, g.height);
    }
    return SD_OK;
}

// sd_track_faces past its checks: the cascade on the grey batch images, the box scores on the frames of src.
int track_faces_run(sd_ctx* ctx, const char* fn, const sd_model* m, const sd_image_batch* images, const BoxFrames& src,
                    const int32_t* d_track_frame, const float* d_prev, int T, const float* d_filter, int filter_w, int filter_h,
                    float bias, int cell_size, int num_bins, int variant, float threshold, float* d_landmarks, int32_t* d_boxes,
                    float* d_scores, uint8_t* d_alive)
{
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
    track_box_kernel<<<sd_div_up(T, 128), 128, 0, ctx->stream>>>(d_prev, T, L, me, sd_model_device_mean(m), nullptr, valid_prev, x0, patch_flag,
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
    if (st & 2) return sd_fail(ctx, SD_ERR_INVALID, "%s: frame index out of range", fn);
    return track_rescore(ctx, src, d_track_frame, d_prev, xn, T, L, me, valid_prev, patch_flag, valid_new, d_filter, filter_w, filter_h,
                         bias, cell_size, num_bins, variant, threshold, d_landmarks, d_boxes, d_scores, d_alive);
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
    return box_scores_entry(ctx, __func__, BoxFrames{images, nullptr, 0}, d_box_frame, d_boxes, n, d_filter, filter_w, filter_h, bias,
                            cell_size, num_bins, variant, d_scores);
}

int sd_hog_box_scores_images(sd_ctx* ctx, const sd_hog_images* images, int bilinear_orientations, const int32_t* d_box_frame,
                             const int32_t* d_boxes, int n, const float* d_filter, int filter_w, int filter_h, float bias, int cell_size,
                             int num_bins, int variant, float* d_scores)
{
    if (!ctx) return SD_ERR_INVALID;
    const sd_image_batch none{};   // box_scores_check's batch: no regions of interest
    if (const int rc = images_check(ctx, __func__, images, bilinear_orientations)) return rc;
    if (const int rc = box_scores_check(ctx, __func__, &none, d_filter, filter_w, filter_h, cell_size, num_bins, variant)) return rc;
    return box_scores_entry(ctx, __func__, BoxFrames{nullptr, images, bilinear_orientations}, d_box_frame, d_boxes, n, d_filter, filter_w,
                            filter_h, bias, cell_size, num_bins, variant, d_scores);
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
    return track_faces_run(ctx, __func__, m, images, BoxFrames{images, nullptr, 0}, d_track_frame, d_prev, T, d_filter, filter_w, filter_h,
                           bias, cell_size, num_bins, variant, threshold, d_landmarks, d_boxes, d_scores, d_alive);
}

int sd_track_faces_images(sd_ctx* ctx, const sd_model* m, const sd_image_batch* images, const sd_hog_images* filter_images,
                          int bilinear_orientations, const int32_t* d_track_frame, const float* d_prev, int T, const float* d_filter,
                          int filter_w, int filter_h, float bias, int cell_size, int num_bins, int variant, float threshold,
                          float* d_landmarks, int32_t* d_boxes, float* d_scores, uint8_t* d_alive)
{
    if (!ctx) return SD_ERR_INVALID;
    SD_REQUIRE(ctx, m && T >= 0, "bad argument");
    if (const int rc = box_scores_check(ctx, __func__, images, d_filter, filter_w, filter_h, cell_size, num_bins, variant)) return rc;
    if (const int rc = images_check(ctx, __func__, filter_images, bilinear_orientations)) return rc;
    if (T == 0) return SD_OK;
    SD_REQUIRE(ctx, images->d_data && d_track_frame && d_prev && d_landmarks && d_boxes && d_scores && d_alive, "null argument");
    const BoxFrames src{nullptr, filter_images, bilinear_orientations};
    HogPyramidFrames fr;
    if (const int rc = match_frames(ctx, __func__, images, src, &fr)) return rc;
    return track_faces_run(ctx, __func__, m, images, src, d_track_frame, d_prev, T, d_filter, filter_w, filter_h, bias, cell_size, num_bins,
                           variant, threshold, d_landmarks, d_boxes, d_scores, d_alive);
}

}  // extern "C"

namespace {

// sd_track_detect_faces (src: the grey batch images) and sd_track_detect_faces_images (src: filter_images); fn names the entry point.
int track_detect(sd_ctx* ctx, const char* fn, const sd_model* m, const sd_image_batch* images, const BoxFrames& src,
                 const int32_t* d_track_frame, const float* d_prev, int T, const float* d_filter, int filter_w, int filter_h, float bias,
                 int cell_size, int num_bins, int variant, float threshold, const int32_t* h_detect_frames, int num_detect_frames,
                 const sd_track_detect_param* param, float* d_landmarks, int32_t* d_boxes, float* d_scores, uint8_t* d_alive,
                 int32_t* d_frame, int32_t* h_num_new)
{
#define TD_REQUIRE(cond, msg)                                                          \
    do {                                                                               \
        if (!(cond)) return sd_fail(ctx, SD_ERR_INVALID, "%s: %s", fn, msg);           \
    } while (0)
    TD_REQUIRE(m && param && h_num_new && T >= 0 && num_detect_frames >= 0, "bad argument");
    const int D = num_detect_frames, F = images->count;
    TD_REQUIRE(d_landmarks && d_boxes && d_scores && d_alive && d_frame && (D == 0 || h_detect_frames), "null argument");
    TD_REQUIRE(T == 0 || (d_track_frame && d_prev), "null argument");
    TD_REQUIRE(T + D == 0 || (images->d_data && F >= 1), "no frames");
    const sd_track_detect_param& p = *param;
    TD_REQUIRE(!std::isnan(threshold) && !std::isnan(p.detect_threshold), "threshold is NaN");
    TD_REQUIRE(p.nms_overlap >= 0.0 && p.nms_overlap <= 1.0 && p.track_overlap >= 0.0 && p.track_overlap <= 1.0,
               "overlaps must be in [0, 1]");
    TD_REQUIRE(p.max_candidates >= 1 && p.max_candidates <= SD_HOG_DETECT_MAX_CANDIDATES,
               "max_candidates must be in [1, SD_HOG_DETECT_MAX_CANDIDATES]");
    TD_REQUIRE(p.max_detections >= 1 && p.max_detections <= p.max_candidates, "max_detections must be in [1, max_candidates]");
    if (const int rc = sd_hog_check_filter(ctx, fn, filter_w, filter_h, p.pad_x, p.pad_y)) return rc;
    TD_REQUIRE(p.h_scales && p.num_scales >= 1, "num_scales must be at least 1");
    for (int s = 0; s < p.num_scales; ++s)
        TD_REQUIRE(p.h_scales[s] > 0.0 && p.h_scales[s] <= 4.0, "every scale must be finite and in (0, 4]");
    const int S = p.num_scales, max_det = p.max_detections;
    const long long slots = (long long)D * max_det;
    TD_REQUIRE(T + slots <= INT32_MAX && (long long)D * S <= INT32_MAX, "too many rows");
    {
        std::vector<char> seen(F, 0);
        for (int i = 0; i < D; ++i) {
            const int f = h_detect_frames[i];
            if (f < 0 || f >= F) return sd_fail(ctx, SD_ERR_INVALID, "%s: listed frame %d is out of range [0, %d)", fn, f, F);
            if (seen[f]) return sd_fail(ctx, SD_ERR_INVALID, "%s: frame %d is listed twice", fn, f);
            seen[f] = 1;
        }
    }
#undef TD_REQUIRE
    // frames that keep their channels: sized as the grey ones (each frame table read back once, here)
    HogPyramidFrames fr;
    if (src.images)
        if (const int rc = match_frames(ctx, fn, images, src, &fr)) return rc;

    // the listed frames (the frame table read back once) and their levels, sliced so that a slice's features fit kDetectSliceFloats
    HogPyramidFrames sel;
    struct Level {
        int lw, lh, hw, hh, ow, oh;
    };
    std::vector<Level> lv((size_t)D * S);
    std::vector<int> slice0 = {0};
    size_t max_feat = 0, max_scores = 0;
    int max_slice = 0;
    const int dd = sd_hog_dd(num_bins, variant);
    if (D > 0) {
        if (src.grey)
            if (const int rc = read_frames(ctx, fn, src, &fr)) return rc;
        sel = fr;
        for (int i = 0; i < D; ++i) sel.frames[i] = fr.frames[h_detect_frames[i]];
        sel.frames.resize(D);
        size_t feat = 0, scores = 0;
        for (int i = 0; i < D; ++i) {
            const sd_hog_image& d = sel.frames[i];
            size_t ff = 0, fs = 0;
            for (int s = 0; s < S; ++s) {
                Level& l = lv[(size_t)i * S + s];
                int hd;
                if (sd_hog_pyramid_shape(d.width, d.height, p.h_scales[s], cell_size, num_bins, variant, &l.lw, &l.lh, &l.hw, &l.hh, &hd))
                    return sd_fail(ctx, SD_ERR_INVALID, "%s: frame %d at scale %g is larger than 2^28 px per side", fn, h_detect_frames[i],
                                   p.h_scales[s]);
                l.ow = l.hw ? std::max(0, sd_score_extent(l.hw, p.pad_x, filter_w)) : 0;
                l.oh = l.hw ? std::max(0, sd_score_extent(l.hh, p.pad_y, filter_h)) : 0;
                if (!sd_window_boxes_fit_int32(l.ow, l.oh, p.pad_x, p.pad_y, filter_w, filter_h, cell_size, d.width, d.height, l.lw, l.lh))
                    return sd_fail(ctx, SD_ERR_INVALID, "%s: the boxes of frame %d do not fit in int32", fn, h_detect_frames[i]);
                ff += (size_t)dd * l.hw * l.hh;
                fs += (size_t)l.ow * l.oh;
            }
            if (fs > UINT32_MAX) return sd_fail(ctx, SD_ERR_INVALID, "%s: more than 2^32 - 1 scores in frame %d", fn, h_detect_frames[i]);
            if (i > slice0.back() && feat + ff > kDetectSliceFloats) {
                slice0.push_back(i);
                feat = scores = 0;
            }
            feat += ff;
            scores += fs;
            max_feat = std::max(max_feat, feat);
            max_scores = std::max(max_scores, scores);
        }
    }
    slice0.push_back(D);
    for (size_t i = 0; i + 1 < slice0.size(); ++i) max_slice = std::max(max_slice, slice0[i + 1] - slice0[i]);

    // workspace: the slice's features | scores | level offsets | grids | score maps | bias, the detections | counts | listed frames
    // | keep | dest, the groups' count | offset | list, the merge's keys | sorted keys | removed, and the new rows' x0 | landmarks |
    // ones | patch flags | box flags
    const int L = sd_model_num_landmarks(m), P = 2 * L;
    const long long R = T + slots;
    const size_t sizes[] = {
        sd_round16(max_feat * sizeof(float)), sd_round16(max_scores * sizeof(float)), sd_round16(sizeof(int64_t) * max_slice * S),
        sd_round16(sizeof(sd_hog_grid) * max_slice * S), sd_round16(sizeof(sd_hog_score_map) * max_slice * S), 16,
        sd_round16(sizeof(sd_hog_detection) * slots), sd_round16(sizeof(int32_t) * D), sd_round16(sizeof(int32_t) * D),
        sd_round16(sizeof(int) * slots), sd_round16(sizeof(int) * (slots + 1)),
        sd_round16(sizeof(int) * (F + 1)), sd_round16(sizeof(int) * (F + 1)), sd_round16(sizeof(int) * R),
        sd_round16(sizeof(unsigned long long) * R), sd_round16(sizeof(unsigned long long) * R), sd_round16(R),
        sd_round16(sizeof(float) * slots * P), sd_round16(sizeof(float) * slots * P), sd_round16(slots), sd_round16(slots), sd_round16(slots)};
    constexpr int kParts = sizeof(sizes) / sizeof(sizes[0]);
    size_t total = 0, at[kParts];
    for (int i = 0; i < kParts; ++i) {
        at[i] = total;
        total += sizes[i];
    }
    uint8_t* ws = static_cast<uint8_t*>(sd_workspace(ctx, SD_WS_TRACK_DETECT, total));
    if (!ws) return SD_ERR_CUDA;
    float* d_feat = reinterpret_cast<float*>(ws + at[0]);
    float* d_sc = reinterpret_cast<float*>(ws + at[1]);
    int64_t* d_off = reinterpret_cast<int64_t*>(ws + at[2]);
    sd_hog_grid* d_grids = reinterpret_cast<sd_hog_grid*>(ws + at[3]);
    sd_hog_score_map* d_maps = reinterpret_cast<sd_hog_score_map*>(ws + at[4]);
    float* d_bias = reinterpret_cast<float*>(ws + at[5]);
    sd_hog_detection* d_det = reinterpret_cast<sd_hog_detection*>(ws + at[6]);
    int32_t* d_cnt = reinterpret_cast<int32_t*>(ws + at[7]);
    int32_t* d_list_frame = reinterpret_cast<int32_t*>(ws + at[8]);
    int* d_keep = reinterpret_cast<int*>(ws + at[9]);
    int* d_dest = reinterpret_cast<int*>(ws + at[10]);
    int* g_count = reinterpret_cast<int*>(ws + at[11]);
    int* g_offset = reinterpret_cast<int*>(ws + at[12]);
    int* g_list = reinterpret_cast<int*>(ws + at[13]);
    unsigned long long* m_key = reinterpret_cast<unsigned long long*>(ws + at[14]);
    unsigned long long* m_sorted = reinterpret_cast<unsigned long long*>(ws + at[15]);
    uint8_t* m_removed = ws + at[16];
    float* x0 = reinterpret_cast<float*>(ws + at[17]);
    float* xn = reinterpret_cast<float*>(ws + at[18]);
    uint8_t* ones = ws + at[19];
    uint8_t* patch_flag = ws + at[20];
    uint8_t* valid_new = ws + at[21];

    // 1. the old rows: sd_track_faces (its status read-back refuses a frame index out of range before any output is written)
    if (T > 0) {
        if (const int rc = track_faces_run(ctx, fn, m, images, src, d_track_frame, d_prev, T, d_filter, filter_w, filter_h, bias, cell_size,
                                           num_bins, variant, threshold, d_landmarks, d_boxes, d_scores, d_alive))
            return rc;
        SD_CUDA(ctx, cudaMemcpyAsync(d_frame, d_track_frame, sizeof(int32_t) * T, cudaMemcpyDeviceToDevice, ctx->stream));
    }

    int n = 0;
    if (D > 0) {
        // 2. the detections of each slice of listed frames: pyramid, scores and sd_hog_detections, as vl_hog_detect composes them
        SD_CUDA(ctx, cudaMemcpyAsync(d_bias, &bias, sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
        SD_CUDA(ctx, cudaMemcpyAsync(d_list_frame, h_detect_frames, sizeof(int32_t) * D, cudaMemcpyHostToDevice, ctx->stream));
        for (size_t k = 0; k + 1 < slice0.size(); ++k) {
            const int i0 = slice0[k], i1 = slice0[k + 1];
            std::vector<int64_t> off((size_t)(i1 - i0) * S, 0);
            std::vector<sd_hog_grid> grids;
            std::vector<sd_hog_score_map> maps;
            int64_t fa = 0, sa = 0;
            int max_w = 0, max_h = 0;
            for (int i = i0; i < i1; ++i)
                for (int s = 0; s < S; ++s) {
                    const Level& l = lv[(size_t)i * S + s];
                    if (!l.hw) continue;
                    off[(size_t)(i - i0) * S + s] = fa;
                    grids.push_back(sd_hog_grid{l.hw, l.hh, fa, sa});
                    maps.push_back(sd_hog_score_map{i - i0, s, sel.frames[i].width, sel.frames[i].height, l.lw, l.lh, l.ow, l.oh, sa});
                    max_w = std::max(max_w, l.hw);
                    max_h = std::max(max_h, l.hh);
                    fa += (int64_t)dd * l.hw * l.hh;
                    sa += (int64_t)l.ow * l.oh;
                }
            if (!grids.empty()) {
                SD_CUDA(ctx, cudaMemcpyAsync(d_off, off.data(), sizeof(int64_t) * off.size(), cudaMemcpyHostToDevice, ctx->stream));
                SD_CUDA(ctx, cudaMemcpyAsync(d_grids, grids.data(), sizeof(sd_hog_grid) * grids.size(), cudaMemcpyHostToDevice, ctx->stream));
                SD_CUDA(ctx, cudaMemcpyAsync(d_maps, maps.data(), sizeof(sd_hog_score_map) * maps.size(), cudaMemcpyHostToDevice, ctx->stream));
                if (const int rc = sd_hog_pyramid_frames(ctx, fn, sel, i0, i1, p.h_scales, S, cell_size, num_bins, variant, d_feat, d_off))
                    return rc;
                const sd_hog_grids gs = {d_feat, (int32_t)grids.size(), 0, 0, d_grids};
                if (const int rc = sd_hog_correlate_table(ctx, &gs, grids.data(), max_w, max_h, num_bins, variant, d_filter, 1, filter_w,
                                                          filter_h, d_bias, p.pad_x, p.pad_y, d_sc))
                    return rc;
            }
            if (const int rc = sd_hog_detections_table(ctx, d_sc, d_maps, maps.data(), (int)maps.size(), i1 - i0, 1, cell_size, filter_w,
                                                       filter_h, p.pad_x, p.pad_y, p.detect_threshold, p.nms_overlap, p.max_candidates,
                                                       max_det, d_det + (size_t)i0 * max_det, d_cnt + i0, nullptr))
                return rc;
        }

        // 3. association against the alive old rows of each frame, and 4. the kept detections' rows, numbered by a scan
        if (const int rc = group_rows(ctx, d_frame, d_alive, T, F, g_count, g_offset, g_list)) return rc;
        associate_kernel<<<sd_div_up(slots, 128), 128, 0, ctx->stream>>>(d_det, d_cnt, d_list_frame, (int)slots, max_det, d_boxes, g_offset,
                                                                         g_list, p.track_overlap, d_keep);
        SD_LAUNCH_CHECK(ctx, "associate_kernel");
        scan_kernel<<<1, kScanThreads, 0, ctx->stream>>>(d_keep, (int)slots, d_dest);
        SD_LAUNCH_CHECK(ctx, "scan_kernel");
        new_rows_kernel<<<sd_div_up(slots, 128), 128, 0, ctx->stream>>>(d_det, d_list_frame, (int)slots, max_det, d_keep, d_dest,
                                                                        sd_model_device_mean(m), L, T, d_frame, x0);
        SD_LAUNCH_CHECK(ctx, "new_rows_kernel");
        int* h = reinterpret_cast<int*>(ctx->h_scratch) + 1;
        SD_CUDA(ctx, cudaMemcpyAsync(h, d_dest + slots, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
        SD_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        n = *h;
    }

    if (n > 0) {
        // the new rows' cascade; an empty patch ends its row (patch_flag), and the status flag it raises is cleared unread
        SD_CUDA(ctx, cudaMemsetAsync(patch_flag, 0, n, ctx->stream));
        SD_CUDA(ctx, cudaMemsetAsync(ones, 1, n, ctx->stream));
        if (const int rc = sd_detect_device(ctx, m, images, d_frame + T, x0, n, xn, patch_flag)) return rc;
        SD_CUDA(ctx, cudaMemsetAsync(reinterpret_cast<int*>(ctx->d_scratch) + 1, 0, sizeof(int), ctx->stream));
        if (const int rc = track_rescore(ctx, src, d_frame + T, xn, xn, n, L, mean_extent(m), ones, patch_flag, valid_new, d_filter,
                                         filter_w, filter_h, bias, cell_size, num_bins, variant, threshold, d_landmarks + (size_t)T * P,
                                         d_boxes + 4 * (size_t)T, d_scores + T, d_alive + T))
            return rc;
    }

    // 5. the merge of each frame's alive rows
    if (T + n > 1) {
        if (const int rc = group_rows(ctx, d_frame, d_alive, T + n, F, g_count, g_offset, g_list)) return rc;
        merge_kernel<<<F, kMergeThreads, 0, ctx->stream>>>(g_offset, g_list, T, d_boxes, d_scores, p.track_overlap, m_key, m_sorted, m_removed,
                                                           d_alive);
        SD_LAUNCH_CHECK(ctx, "merge_kernel");
    }
    *h_num_new = n;
    return SD_OK;
}

}  // namespace

extern "C" {

int sd_track_detect_faces(sd_ctx* ctx, const sd_model* m, const sd_image_batch* images, const int32_t* d_track_frame, const float* d_prev,
                          int T, const float* d_filter, int filter_w, int filter_h, float bias, int cell_size, int num_bins, int variant,
                          float threshold, const int32_t* h_detect_frames, int num_detect_frames, const sd_track_detect_param* param,
                          float* d_landmarks, int32_t* d_boxes, float* d_scores, uint8_t* d_alive, int32_t* d_frame, int32_t* h_num_new)
{
    if (!ctx) return SD_ERR_INVALID;
    if (const int rc = box_scores_check(ctx, __func__, images, d_filter, filter_w, filter_h, cell_size, num_bins, variant)) return rc;
    return track_detect(ctx, __func__, m, images, BoxFrames{images, nullptr, 0}, d_track_frame, d_prev, T, d_filter, filter_w, filter_h,
                        bias, cell_size, num_bins, variant, threshold, h_detect_frames, num_detect_frames, param, d_landmarks, d_boxes,
                        d_scores, d_alive, d_frame, h_num_new);
}

int sd_track_detect_faces_images(sd_ctx* ctx, const sd_model* m, const sd_image_batch* images, const sd_hog_images* filter_images,
                                 int bilinear_orientations, const int32_t* d_track_frame, const float* d_prev, int T, const float* d_filter,
                                 int filter_w, int filter_h, float bias, int cell_size, int num_bins, int variant, float threshold,
                                 const int32_t* h_detect_frames, int num_detect_frames, const sd_track_detect_param* param,
                                 float* d_landmarks, int32_t* d_boxes, float* d_scores, uint8_t* d_alive, int32_t* d_frame,
                                 int32_t* h_num_new)
{
    if (!ctx) return SD_ERR_INVALID;
    if (const int rc = box_scores_check(ctx, __func__, images, d_filter, filter_w, filter_h, cell_size, num_bins, variant)) return rc;
    if (const int rc = images_check(ctx, __func__, filter_images, bilinear_orientations)) return rc;
    return track_detect(ctx, __func__, m, images, BoxFrames{nullptr, filter_images, bilinear_orientations}, d_track_frame, d_prev, T,
                        d_filter, filter_w, filter_h, bias, cell_size, num_bins, variant, threshold, h_detect_frames, num_detect_frames,
                        param, d_landmarks, d_boxes, d_scores, d_alive, d_frame, h_num_new);
}

}  // extern "C"
