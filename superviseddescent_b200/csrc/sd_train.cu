// Cascade levels of the optimiser in chunks of rows (include/sd_b200.h, "cascade levels").
//
//   sd_level_chunk_rows       rows of one chunk that fit beside what the level's solve allocates
//   sd_train_level            superviseddescent.hpp:173-217: HOG, targets, shift, Gram accumulation, exchange, solve, update
//   sd_apply_level            superviseddescent.hpp:262-306, 323-344: HOG, templates, update
//   sd_*_level_projected      the same two levels with the feature rows from the caller's projection callback (RowSource)
//   sd_*_level_host_projected the same with a host callback, its rows uploaded through a pinned staging pair (host_rows)
//
// [A^T A | A^T b] is a sum over rows, so a level never needs all of its feature rows at once.  The rows are shifted by the column
// means of the first chunk (the pilot p, over all ranks) before they enter the Gram: with n0 rows in that chunk p is within about
// sigma / sqrt(n0) of the true mean, so the shifted Gram keeps the digits that centring saves (DESIGN 4.3), and the solve
// (solve_gram_impl) is exact for any shift -- it rebuilds the norm of the unshifted matrix from the shift, eliminates the bias
// column first (the exact centring of any shifted Gram) and shifts the bias back.  With one chunk p IS the mean and the call
// sequence is sd_train's one-shot sequence, kernel for kernel.
//
// The HOG rows come from frames resident on the device, or from frames that stay in pinned host memory, gathered batch by batch
// (gather_hog_rows); sd_level_frames says which.
#include "sd_internal.cuh"
#include "sd_warp.cuh"

#include <climits>
#include <cstring>

namespace {

constexpr int kMinChunkRows = 256;                       // below this a chunk is all launch overhead
constexpr size_t kReserveBytes = size_t(512) << 20;      // small workspaces, tile lists, allocator granularity

// The batch as seen from sample r0 on: sample i of the view reads the frame sample r0 + i reads in the whole batch.
sd_image_batch batch_from(const sd_image_batch& b, int r0)
{
    sd_image_batch v = b;
    if (r0 == 0) return v;
    v.count = b.count - r0;
    if (b.d_frames) v.d_frames = b.d_frames + r0;
    if (b.d_roi) v.d_roi = b.d_roi + r0;
    if (b.d_roi_miss) v.d_roi_miss = b.d_roi_miss + r0;
    if (!b.d_frames && !b.d_roi) v.d_data = b.d_data + (int64_t)r0 * b.image_stride;
    return v;
}

// ---- host frames: the training gather (DESIGN 4.6) ----------------------------------------------------------------------------
// At the start of a level every sample's landmarks are known, so the window each of its patches reads is known exactly.  Per
// gather batch, roi_plan_kernel merges the windows of a sample's L patches into the union slot of its frame, gather_layout_kernel
// clips every touched union to its frame, lays the unions out back to back in one staging half and writes the gather records;
// roi_gather_kernel pulls them over PCIe (samples of one frame in one batch share one region), and the unchanged HOG kernel reads
// them through per-sample sd_roi records.  The window a sample's patch reads always lies in its frame's region: a region miss
// is a bug, reported as such, never a retry.
struct FrameDev {
    const uint8_t* src;                   // device-mapped address of the frame's first pixel
    int32_t width, height, row_stride, channels;
};

struct GatherTotals {
    long long bytes;                      // grey bytes of the batch's regions in the staging half
    long long pcie;                       // bytes read from host memory (x channels)
    int n_grey, n_colour;                 // gather records of grey / colour frames
};

// The state of one level call on host frames
struct HostGather {
    int num_frames;
    const int32_t* d_sample_frame;        // the caller's index, or the identity in SD_WS_GATHER
    size_t half;                          // bytes of one staging half (the context's d_stage pair)
    // device tables (SD_WS_GATHER)
    FrameDev* d_fr;
    int2* d_lo;                           // per frame: union of the planned windows, min corner (INT_MAX = none) ...
    int2* d_hi;                           // ... and max corner, exclusive
    sd_roi* d_froi;                       // per frame: its region in the current batch
    GatherRec* d_rec;                     // grey records [0, F), colour records [F, 2F)
    sd_roi* d_roi;                        // per sample: its frame's region
    sd_frame* d_dims;                     // per sample: its frame's size
    int32_t* d_hidx;                      // per sample: its HOG index into its batch, with its mirrored bit (NULL: none is mirrored)
    const sd_sample_warp* d_warp;         // the caller's per-sample warps (NULL: none)
    uint8_t* d_miss;                      // per sample: a patch read outside the region (must never be raised)
    GatherTotals* d_tot;
    int guess = 0;                        // samples the next batch starts from (gather_hog_rows)
    int buf = 0;
};

constexpr int kPlanThreads = 128;
constexpr int kLayoutThreads = 1024;

// frame of sample s, as the HOG kernel resolves an image index: an index out of range raises the status flag and reads frame 0.
// With a warp table (warped) a mirrored bit is not decoded: the index is out of range.
__device__ __forceinline__ int sample_frame(const int32_t* __restrict__ idx, int s, int F, int* status, bool warped)
{
    int f = warped ? idx[s] : sd_sample_frame_of(idx[s]);
    if (f < 0 || f >= F) {
        if (status) atomicOr(status, 2);
        f = 0;
    }
    return f;
}

// The rectangle [x0, x1) x [y0, y1) of frame pixels that the taps of window [ua, ub) x [va, vb) of V (already clipped to V, not
// empty) read under warp m: cv::warpAffine's fixed-point terms are each monotone in their own variable, so the window's corners
// bound every tap, and each tap also reads the pixel right of and below it.
__device__ __forceinline__ void warp_window_rect(const double* m, int ua, int ub, int va, int vb, int* x0, int* y0, int* x1, int* y1)
{
    const int2 ca = sd_warp_col(m, (double)ua), cb = sd_warp_col(m, (double)(ub - 1));
    const int2 ra = sd_warp_row(m, (double)va), rb = sd_warp_row(m, (double)(vb - 1));
    const int sx[4] = {ra.x + ca.x, ra.x + cb.x, rb.x + ca.x, rb.x + cb.x}, sy[4] = {ra.y + ca.y, ra.y + cb.y, rb.y + ca.y, rb.y + cb.y};
    int xa = INT_MAX, xb = INT_MIN, ya = INT_MAX, yb = INT_MIN;
    for (int k = 0; k < 4; ++k) {
        xa = min(xa, sx[k] >> 10); xb = max(xb, sx[k] >> 10);
        ya = min(ya, sy[k] >> 10); yb = max(yb, sy[k] >> 10);
    }
    *x0 = xa; *x1 = xb + 2; *y0 = ya; *y1 = yb + 2;
}

// One block per sample: the union of the windows of its L patches in its frame, [x0, x0 + 2 half) x [cy - half, cy + half) with
// x0 = sd_window_x0 (cvRound(x_l) - half, or the frame's window of a mirrored patch), merged into its frame's slot.  A warped
// sample (warp != NULL) plans, per patch, the frame pixels its window of V reads (warp_window_rect); an invalid warp reads none
// (the HOG kernel flags it and reads no pixel).
__global__ void __launch_bounds__(kPlanThreads) roi_plan_kernel(const float* __restrict__ x, int L, const int32_t* __restrict__ idx,
                                                                int F, const FrameDev* __restrict__ fr, const sd_eyes_dev eyes,
                                                                float rel, int fixed_half, int2* __restrict__ lo, int2* __restrict__ hi,
                                                                int* status, const sd_sample_warp* __restrict__ warp)
{
    const int s = blockIdx.x;
    const float* __restrict__ row = x + (long long)s * 2 * L;
    __shared__ int s_half, s_frame, s_width, s_mirrored, s_warp_ok;
    __shared__ int s_box[4][kPlanThreads / 32];
    if (threadIdx.x == 0) {
        bool degenerate;
        s_half = sd_patch_half(row, L, eyes, rel, fixed_half, &degenerate);   // the HOG kernel flags a degenerate sample itself
        s_frame = sample_frame(idx, s, F, status, warp != nullptr);
        s_width = fr[s_frame].width;
        s_mirrored = !warp && sd_sample_is_mirrored(idx[s]);
        if (warp) {
            s_warp_ok = sd_warp_valid(warp[s], fr[s_frame].width, fr[s_frame].height);
        }
    }
    __syncthreads();
    int x0 = INT_MAX, y0 = INT_MAX, x1 = INT_MIN, y1 = INT_MIN;
    for (int l = threadIdx.x; l < L; l += kPlanThreads) {
        const int cx = __float2int_rn(row[l]), cy = __float2int_rn(row[l + L]);
        if (warp) {
            if (!s_warp_ok) continue;
            const sd_sample_warp& w = warp[s];
            const int ua = max(cx - s_half, 0), ub = min(cx + s_half, w.width), va = max(cy - s_half, 0), vb = min(cy + s_half, w.height);
            if (ua >= ub || va >= vb) continue;                   // the window lies outside V: zeros, no pixel read
            int rx0, ry0, rx1, ry1;
            warp_window_rect(w.m, ua, ub, va, vb, &rx0, &ry0, &rx1, &ry1);
            x0 = min(x0, rx0); y0 = min(y0, ry0);
            x1 = max(x1, rx1); y1 = max(y1, ry1);
            continue;
        }
        const int wx = sd_window_x0(cx, s_half, s_width, s_mirrored);
        x0 = min(x0, wx); y0 = min(y0, cy - s_half);
        x1 = max(x1, wx + 2 * s_half); y1 = max(y1, cy + s_half);
    }
    for (int o = 16; o > 0; o >>= 1) {
        x0 = min(x0, __shfl_xor_sync(0xffffffffu, x0, o)); y0 = min(y0, __shfl_xor_sync(0xffffffffu, y0, o));
        x1 = max(x1, __shfl_xor_sync(0xffffffffu, x1, o)); y1 = max(y1, __shfl_xor_sync(0xffffffffu, y1, o));
    }
    const int w = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0) { s_box[0][w] = x0; s_box[1][w] = y0; s_box[2][w] = x1; s_box[3][w] = y1; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int k = 1; k < kPlanThreads / 32; ++k) {
            x0 = min(x0, s_box[0][k]); y0 = min(y0, s_box[1][k]); x1 = max(x1, s_box[2][k]); y1 = max(y1, s_box[3][k]);
        }
        const int f = s_frame;
        if (x0 <= x1) {                                       // a warped sample may read no pixel at all
            atomicMin(&lo[f].x, x0); atomicMin(&lo[f].y, y0);
            atomicMax(&hi[f].x, x1); atomicMax(&hi[f].y, y1);
        }
    }
}

// One block over all frames: every touched union is clipped to its frame, its x aligned down to 16 pixels and its width bounded by
// row_stride / channels (as detect's face_roi does), laid out at an exclusive scan of the region bytes, given a gather record, and
// its slot emptied for the next batch.  Then each of the batch's n samples receives its frame's region and size, and, when some
// sample is mirrored (hidx), its index into the batch with its mirrored bit.
__global__ void __launch_bounds__(kLayoutThreads) gather_layout_kernel(const FrameDev* __restrict__ fr, int F, int2* __restrict__ lo,
                                                                       int2* __restrict__ hi, sd_roi* __restrict__ froi,
                                                                       GatherRec* __restrict__ rec, const int32_t* __restrict__ idx, int n,
                                                                       sd_roi* __restrict__ roi, sd_frame* __restrict__ dims,
                                                                       int32_t* __restrict__ hidx, GatherTotals* __restrict__ tot,
                                                                       bool warped)
{
    __shared__ long long s_scan[kLayoutThreads / 32];
    __shared__ long long s_base, s_pcie;
    __shared__ int s_ng, s_nc;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) { s_base = 0; s_pcie = 0; s_ng = 0; s_nc = 0; }
    __syncthreads();
    for (int f0 = 0; f0 < F; f0 += kLayoutThreads) {
        const int f = f0 + tid;
        long long bytes = 0;
        sd_roi r{};
        if (f < F) {
            const int2 a = lo[f], b = hi[f];
            if (a.x <= b.x) {                                  // touched by this batch
                lo[f] = make_int2(INT_MAX, INT_MAX);
                hi[f] = make_int2(INT_MIN, INT_MIN);
                const FrameDev d = fr[f];
                const int xa = max(a.x, 0), ya = max(a.y, 0), xb = min(b.x, d.width), yb = min(b.y, d.height);
                if (xa < xb && ya < yb) {                      // otherwise every patch lies outside the frame: zeros, no pixel read
                    r.x = xa & ~15;
                    int w = (xb - r.x + 15) & ~15;
                    const int maxw = (d.row_stride / d.channels - r.x) & ~15;
                    r.w = w < maxw ? w : maxw;
                    r.y = ya;
                    r.h = yb - ya;
                    r.row_stride = r.w;
                    bytes = (long long)r.w * r.h;
                }
            }
        }
        // block-wide exclusive scan of the region bytes
        long long v = bytes;
        for (int o = 1; o < 32; o <<= 1) {
            const long long t = __shfl_up_sync(0xffffffffu, v, o);
            if (lane >= o) v += t;
        }
        if (lane == 31) s_scan[warp] = v;
        __syncthreads();
        if (warp == 0) {
            long long w = lane < kLayoutThreads / 32 ? s_scan[lane] : 0;
            for (int o = 1; o < 32; o <<= 1) {
                const long long t = __shfl_up_sync(0xffffffffu, w, o);
                if (lane >= o) w += t;
            }
            if (lane < kLayoutThreads / 32) s_scan[lane] = w;   // inclusive per warp
        }
        __syncthreads();
        const long long excl = s_base + (warp > 0 ? s_scan[warp - 1] : 0) + v - bytes;
        if (f < F) {
            r.offset = excl;
            froi[f] = r;
            if (bytes > 0) {
                const FrameDev d = fr[f];
                const int k = d.channels == 1 ? atomicAdd(&s_ng, 1) : F + atomicAdd(&s_nc, 1);
                rec[k] = GatherRec{d.src + (long long)r.y * d.row_stride + (long long)r.x * d.channels, d.row_stride, excl, r.w >> 4, r.h};
                atomicAdd((unsigned long long*)&s_pcie, (unsigned long long)(bytes * d.channels));
            }
        }
        __syncthreads();
        if (tid == 0) s_base += s_scan[kLayoutThreads / 32 - 1];
        __syncthreads();
    }
    for (int s = tid; s < n; s += kLayoutThreads) {
        const int f = sample_frame(idx, s, F, nullptr, warped);   // roi_plan_kernel has flagged a bad index
        roi[s] = froi[f];
        dims[s] = sd_frame{fr[f].width, fr[f].height, 0, 0, 0};
        if (hidx) hidx[s] = sd_sample_is_mirrored(idx[s]) ? s | SD_SAMPLE_MIRRORED : s;
    }
    if (tid == 0) *tot = GatherTotals{s_base, s_pcie, s_ng, s_nc};
}

// bytes of one staging half: the caller's size (0 = the default), at least the largest frame's grey bytes (no region is larger)
size_t stage_half(const sd_level_frames& src, size_t largest)
{
    const size_t want = src.stage_half_bytes ? src.stage_half_bytes : SD_STAGE_HALF_BYTES;
    return sd_round16(want > largest ? want : largest);
}

// Checks the frames (SD_ERR_INVALID before any work is queued), sizes the context's staging pair and sets up the device tables.
int gather_prepare(sd_ctx* ctx, HostGather& g, const sd_level_frames& src, int N)
{
    const int F = src.num_host_frames;
    // the frames the samples refer to (an index out of range reads frame 0 and is reported by the projection's status flag)
    std::vector<int32_t> idx(N);
    if (!src.d_sample_frame)
        for (int s = 0; s < N; ++s) idx[s] = s;
    else if (N > 0) {
        SD_CUDA(ctx, cudaMemcpyAsync(idx.data(), src.d_sample_frame, (size_t)N * sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
        SD_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    std::vector<char> used(F, 0);
    bool mirrored = false;
    const bool warped = src.d_sample_warp != nullptr;            // then a mirrored bit is an index out of range
    for (int s = 0; s < N; ++s) {
        const int f = warped ? idx[s] : sd_sample_frame_of(idx[s]);
        used[f >= 0 && f < F ? f : 0] = 1;
        mirrored = mirrored || (!warped && sd_sample_is_mirrored(idx[s]));
    }
    std::vector<FrameDev> fr(F);
    PinnedRange last;
    size_t largest = 0;
    for (int f = 0; f < F; ++f) {
        if (!used[f]) { fr[f] = FrameDev{nullptr, 1, 1, 16, 1}; continue; }
        const sd_host_frame& h = src.host_frames[f];
        int rc = sd_check_host_frame(ctx, __func__, h, f);
        if (rc) return rc;
        const uint8_t* m = sd_mapped_frame(h.h_data, sd_host_frame_bytes(h), last);
        if (!m || ((reinterpret_cast<uintptr_t>(m) | (uintptr_t)h.row_stride) & 15))
            return sd_fail(ctx, SD_ERR_INVALID, "%s: frame %d is not pinned and device-mapped with a 16-byte aligned base and row_stride", __func__, f);
        // the gather moves 16 pixels at a time: every 16-pixel step of a row must lie inside the row
        if ((size_t)h.row_stride < (size_t)h.channels * sd_round16(h.width))
            return sd_fail(ctx, SD_ERR_INVALID, "%s: frame %d: row_stride < channels * (width rounded up to 16)", __func__, f);
        fr[f] = FrameDev{m, h.width, h.height, h.row_stride, h.channels};
        largest = sd_gray_bytes(h) > largest ? sd_gray_bytes(h) : largest;
    }
    g.half = stage_half(src, largest);
    int rc = sd_ensure_stage(ctx, g.half);
    if (rc) return rc;
    // device tables
    const size_t n = N > 0 ? N : 1;
    const size_t b_fr = sd_round16(F * sizeof(FrameDev)), b_lo = sd_round16(F * sizeof(int2)), b_froi = sd_round16(F * sizeof(sd_roi));
    const size_t b_rec = sd_round16(2 * F * sizeof(GatherRec)), b_roi = sd_round16(n * sizeof(sd_roi)), b_dims = sd_round16(n * sizeof(sd_frame));
    const size_t b_idx = src.d_sample_frame ? 0 : sd_round16(n * sizeof(int32_t));
    const size_t b_hidx = mirrored ? sd_round16(n * sizeof(int32_t)) : 0;
    uint8_t* t = (uint8_t*)sd_workspace(ctx, SD_WS_GATHER, b_fr + 2 * b_lo + b_froi + b_rec + b_roi + b_dims + b_idx + b_hidx +
                                                               sd_round16(n) + sizeof(GatherTotals));
    if (!t) return SD_ERR_CUDA;
    g.d_fr = (FrameDev*)t;                      t += b_fr;
    g.d_lo = (int2*)t;                          t += b_lo;
    g.d_hi = (int2*)t;                          t += b_lo;
    g.d_froi = (sd_roi*)t;                      t += b_froi;
    g.d_rec = (GatherRec*)t;                    t += b_rec;
    g.d_roi = (sd_roi*)t;                       t += b_roi;
    g.d_dims = (sd_frame*)t;                    t += b_dims;
    int32_t* d_idx = (int32_t*)t;               t += b_idx;
    g.d_hidx = b_hidx ? (int32_t*)t : nullptr;  t += b_hidx;
    g.d_miss = t;                               t += sd_round16(n);
    g.d_tot = (GatherTotals*)t;
    g.num_frames = F;
    g.d_sample_frame = b_idx ? d_idx : src.d_sample_frame;
    g.d_warp = src.d_sample_warp;
    if (b_idx && N > 0)                                                                    // no index: sample i reads frame i
        SD_CUDA(ctx, cudaMemcpyAsync(d_idx, idx.data(), (size_t)N * sizeof(int32_t), cudaMemcpyHostToDevice, ctx->stream));
    SD_CUDA(ctx, cudaMemcpyAsync(g.d_fr, fr.data(), F * sizeof(FrameDev), cudaMemcpyHostToDevice, ctx->stream));
    SD_CUDA(ctx, cudaMemsetAsync(g.d_lo, 0x7f, F * sizeof(int2), ctx->stream));          // 0x7f7f7f7f: above any coordinate
    SD_CUDA(ctx, cudaMemsetAsync(g.d_hi, 0x80, F * sizeof(int2), ctx->stream));          // 0x80808080: below any coordinate
    SD_CUDA(ctx, cudaMemsetAsync(g.d_miss, 0, n, ctx->stream));
    SD_CUDA(ctx, cudaStreamSynchronize(ctx->stream));                                      // fr and idx go out of scope
    g.guess = N > 0 ? N : 1;
    return SD_OK;
}

// A patch that read outside its planned region would mean rows computed from a partial window: fail the call.
int gather_finish(sd_ctx* ctx, const HostGather& g, int N)
{
    if (N == 0) return SD_OK;
    std::vector<uint8_t> miss(N);
    SD_CUDA(ctx, cudaMemcpyAsync(miss.data(), g.d_miss, N, cudaMemcpyDeviceToHost, ctx->stream));
    SD_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    for (int s = 0; s < N; ++s)
        if (miss[s]) return sd_fail(ctx, SD_ERR_CUDA, "internal error: sample %d read a pixel outside its planned gather region", s);
    return SD_OK;
}

// HOG rows of samples [r0, r0 + rows) from host frames, in gather batches that fit one staging half: plan, layout and gather on
// the copy stream (the gather of batch k+1 runs while the HOG of batch k does), HOG on the compute stream.
int gather_hog_rows(sd_ctx* ctx, HostGather& g, const float* d_x, int r0, int rows, int L, const sd_normalisation* eyes,
                    const sd_hog_param* p, float* d_chunk, int64_t ld)
{
    const int P = 2 * L;
    const bool fixed = !eyes || eyes->kind == 0;
    sd_eyes_dev eyes_dev;
    memset(&eyes_dev, 0, sizeof(eyes_dev));
    int rc = fixed ? SD_OK : sd_eyes_to_dev(ctx, eyes, L, &eyes_dev);
    if (rc) return rc;
    const int fixed_half = fixed ? p->num_cells * (p->cell_size / 2) : 0;
    int* status = reinterpret_cast<int*>(ctx->d_scratch) + 1;
    // the copy stream starts after everything queued so far on the compute stream: the landmarks, and every earlier reader of the
    // per-sample tables and of both staging halves
    SD_CUDA(ctx, cudaEventRecord(ctx->stage_done[0], ctx->stream));
    SD_CUDA(ctx, cudaEventRecord(ctx->stage_done[1], ctx->stream));
    SD_CUDA(ctx, cudaStreamWaitEvent(ctx->copy_stream, ctx->stage_done[0], 0));
    for (int b0 = 0; b0 < rows;) {
        const int s0 = r0 + b0;
        int nb = g.guess < rows - b0 ? g.guess : rows - b0;
        GatherTotals t;
        for (;;) {
            roi_plan_kernel<<<nb, kPlanThreads, 0, ctx->copy_stream>>>(d_x + (int64_t)s0 * P, L, g.d_sample_frame + s0, g.num_frames, g.d_fr,
                                                                       eyes_dev, p->relative_patch_size, fixed_half, g.d_lo, g.d_hi, status,
                                                                       g.d_warp ? g.d_warp + s0 : nullptr);
            SD_LAUNCH_CHECK(ctx, "roi_plan_kernel");
            gather_layout_kernel<<<1, kLayoutThreads, 0, ctx->copy_stream>>>(g.d_fr, g.num_frames, g.d_lo, g.d_hi, g.d_froi, g.d_rec,
                                                                            g.d_sample_frame + s0, nb, g.d_roi + s0, g.d_dims + s0,
                                                                            g.d_hidx ? g.d_hidx + s0 : nullptr, g.d_tot, g.d_warp != nullptr);
            SD_LAUNCH_CHECK(ctx, "gather_layout_kernel");
            SD_CUDA(ctx, cudaMemcpyAsync(&t, g.d_tot, sizeof(t), cudaMemcpyDeviceToHost, ctx->copy_stream));
            SD_CUDA(ctx, cudaStreamSynchronize(ctx->copy_stream));
            if ((size_t)t.bytes <= g.half) break;
            // too large for one staging half: fewer samples (one always fits: no region exceeds its frame's grey bytes)
            const int scaled = (int)((double)nb * (double)g.half / (double)t.bytes * 0.9);
            nb = scaled < nb - 1 ? (scaled > 1 ? scaled : 1) : nb - 1;
        }
        // the next batch starts from this size, twice it when this one filled less than half a staging half
        g.guess = (size_t)t.bytes * 2 <= g.half && nb <= INT_MAX / 2 ? 2 * nb : nb;
        const int buf = g.buf;
        g.buf ^= 1;
        uint8_t* stage = static_cast<uint8_t*>(ctx->d_stage[buf]);
        SD_CUDA(ctx, cudaStreamWaitEvent(ctx->copy_stream, ctx->stage_done[buf], 0));   // the HOG that last read this half is done
        rc = sd_roi_gather(ctx, g.d_rec, t.n_grey, g.d_rec + g.num_frames, t.n_colour, stage, ctx->copy_stream);
        if (rc) return rc;
        SD_CUDA(ctx, cudaEventRecord(ctx->stage_ev[buf], ctx->copy_stream));
        SD_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, ctx->stage_ev[buf], 0));
        sd_image_batch ib{};
        ib.d_data = stage;
        ib.count = nb;
        ib.d_roi = g.d_roi + s0;
        ib.d_roi_miss = g.d_miss + s0;
        ib.d_frames = g.d_dims + s0;
        rc = g.d_warp ? sd_hog_batch_unmirrored(ctx, &ib, nullptr, d_x + (int64_t)s0 * P, P, nb, L, eyes, p, d_chunk + (int64_t)b0 * ld, ld,
                                                nullptr, g.d_warp + s0)
                      : sd_hog_batch(ctx, &ib, g.d_hidx ? g.d_hidx + s0 : nullptr, d_x + (int64_t)s0 * P, P, nb, L, eyes, p,
                                     d_chunk + (int64_t)b0 * ld, ld);
        if (rc) return rc;
        SD_CUDA(ctx, cudaEventRecord(ctx->stage_done[buf], ctx->stream));
        ctx->gathered_bytes += t.pcie;
        b0 += nb;
    }
    return SD_OK;
}

// exactly one source of frames (SD_ERR_INVALID otherwise)
int check_frames(sd_ctx* ctx, const sd_level_frames* src)
{
    SD_REQUIRE(ctx, src && !src->images != !src->host_frames, "exactly one of frames->images and frames->host_frames");
    SD_REQUIRE(ctx, src->images || src->num_host_frames >= 1, "num_host_frames < 1");
    return SD_OK;
}

// On the host route: checks the frames and sets up the gather (SD_ERR_INVALID before any work is queued).
int frames_prepare(sd_ctx* ctx, const sd_level_frames* src, HostGather& g, int N)
{
    const int rc = check_frames(ctx, src);
    if (rc || src->images) return rc;
    return gather_prepare(ctx, g, *src, N);
}

// HOG rows of samples [r0, r0 + rows) into the chunk buffer
int hog_rows(sd_ctx* ctx, const sd_level_frames& src, HostGather& g, const float* d_x, int r0, int rows, int L,
             const sd_normalisation* eyes, const sd_hog_param* p, float* d_chunk, int64_t ld)
{
    if (!src.images) return gather_hog_rows(ctx, g, d_x, r0, rows, L, eyes, p, d_chunk, ld);
    const int P = 2 * L;
    const int32_t* idx = src.d_sample_frame;
    const sd_image_batch view = idx ? *src.images : batch_from(*src.images, r0);
    if (src.d_sample_warp)
        return sd_hog_batch_unmirrored(ctx, &view, idx ? idx + r0 : nullptr, d_x + (int64_t)r0 * P, P, rows, L, eyes, p, d_chunk, ld, nullptr,
                                       src.d_sample_warp + r0);
    return sd_hog_batch(ctx, &view, idx ? idx + r0 : nullptr, d_x + (int64_t)r0 * P, P, rows, L, eyes, p, d_chunk, ld);
}

size_t round_up(size_t v, size_t m) { return (v + m - 1) / m * m; }

// ---- rows from a host projection: the copy pipeline (DESIGN 4.8) --------------------------------------------------------------
// The callback fills one pinned staging half on the calling thread while the other half's rows go up on the copy stream; one event
// per half tells the host when it may refill that half.  The first upload of a chunk waits for the chunk buffer's last reader on
// the stream, and the stream waits for the chunk's last upload, so the host fills chunk k + 1 while the GPU works on chunk k.
struct HostRows {
    const float* h_x = nullptr;          // pinned copy of this rank's parameter rows (the context's host_x)
    int64_t ld_out = 0;                  // floats between staged rows: roundup4(D)
    int per_half = 1;                    // rows of one batch: what the requested staging half holds, at least one
    int buf = 0;                         // the half the next batch fills
};

// the context's pinned buffer *p holds at least `bytes` (grow-only; the old one is freed once no upload reads it)
int ensure_pinned(sd_ctx* ctx, void** p, size_t* have, size_t bytes)
{
    if (*have >= bytes) return SD_OK;
    if (*p) {
        SD_CUDA(ctx, cudaStreamSynchronize(ctx->copy_stream));
        SD_CUDA(ctx, cudaFreeHost(*p));
        *p = nullptr;
        *have = 0;
    }
    SD_CUDA(ctx, cudaMallocHost(p, bytes));
    *have = bytes;
    return SD_OK;
}

// Sizes the staging pair from the descriptor and copies d_x (N x P) into pinned memory once for the level call.
int host_prepare(sd_ctx* ctx, const sd_level_host_projection& hp, HostRows& h, const float* d_x, int N, int P)
{
    h.ld_out = (int64_t)round_up(hp.feature_length, 4);
    const size_t row = (size_t)h.ld_out * sizeof(float);
    const size_t fit = (hp.stage_half_bytes ? hp.stage_half_bytes : SD_STAGE_HALF_BYTES) / row;
    h.per_half = fit < 1 ? 1 : (fit > INT_MAX ? INT_MAX : (int)fit);
    h.buf = 0;
    if (N == 0) return SD_OK;                                        // a rank without samples: no callback, no copy
    const size_t half = (size_t)(h.per_half < N ? h.per_half : N) * row;    // no batch is longer than the level
    for (int b = 0; b < 2; ++b) {
        const int rc = ensure_pinned(ctx, &ctx->host_stage[b], &ctx->host_stage_bytes[b], half);
        if (rc) return rc;
    }
    const size_t xbytes = (size_t)N * P * sizeof(float);
    const int rc = ensure_pinned(ctx, &ctx->host_x, &ctx->host_x_bytes, xbytes);
    if (rc) return rc;
    SD_CUDA(ctx, cudaMemcpyAsync(ctx->host_x, d_x, xbytes, cudaMemcpyDeviceToHost, ctx->stream));
    SD_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    h.h_x = static_cast<const float*>(ctx->host_x);
    return SD_OK;
}

// feature rows of samples [r0, r0 + rows) into columns [0, D) of the chunk buffer, batch by batch through the staging pair
int host_rows(sd_ctx* ctx, const sd_level_host_projection& hp, HostRows& h, int P, int r0, int rows, float* d_chunk, int64_t ld)
{
    SD_CUDA(ctx, cudaEventRecord(ctx->host_chunk_free, ctx->stream));                 // after the previous chunk's last reader
    SD_CUDA(ctx, cudaStreamWaitEvent(ctx->copy_stream, ctx->host_chunk_free, 0));
    int rc = SD_OK, last = -1;
    for (int b0 = 0; b0 < rows;) {
        const int nb = rows - b0 < h.per_half ? rows - b0 : h.per_half;
        const int buf = h.buf;
        h.buf ^= 1;
        SD_CUDA(ctx, cudaEventSynchronize(ctx->host_stage_ev[buf]));                  // the upload that last read this half is done
        float* out = static_cast<float*>(ctx->host_stage[buf]);
        const int64_t first = (int64_t)r0 + b0;
        const int cb = hp.fn(hp.user, hp.level, h.h_x + first * P, P, first, nb, out, h.ld_out);
        if (cb) {
            rc = sd_fail(ctx, SD_ERR_INVALID, "projection callback returned %d", cb);
            break;
        }
        SD_CUDA(ctx, cudaMemcpy2DAsync(d_chunk + (int64_t)b0 * ld, (size_t)ld * sizeof(float), out, (size_t)h.ld_out * sizeof(float),
                                       (size_t)hp.feature_length * sizeof(float), nb, cudaMemcpyHostToDevice, ctx->copy_stream));
        SD_CUDA(ctx, cudaEventRecord(ctx->host_stage_ev[buf], ctx->copy_stream));
        last = buf;
        b0 += nb;
    }
    // what reads the chunk (templates, targets, centring, Gram, update) waits for its uploads; after a failure too, so that the
    // caller may free the buffer in stream order
    if (last >= 0) SD_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, ctx->host_stage_ev[last], 0));
    return rc;
}

// ---- the row source of a level (DESIGN 4.7, 4.8) ------------------------------------------------------------------------------
// A level's feature rows come from the HOG of its frames (sd_train_level / sd_apply_level), from the caller's device projection
// (sd_train_level_projected / sd_apply_level_projected) or from the caller's host projection (sd_*_level_host_projected).
// Everything after the rows -- templates, targets, shift, Gram, exchange, solve, update -- is one loop (train_rows, apply_rows)
// whichever the source.
struct RowSource {
    const sd_level_projection* proj = nullptr;        // the caller's device projection ...
    const sd_level_host_projection* hproj = nullptr;  // ... or host projection; both NULL: HOG of the frames below
    HostRows h{};
    const sd_level_frames* frames = nullptr;
    HostGather g{};
    int L = 0;
    const sd_normalisation* hog_eyes = nullptr;
    const sd_hog_param* p = nullptr;
    void use(const sd_level_projection* d) { proj = d; }
    void use(const sd_level_host_projection* d) { hproj = d; }
    bool callback() const { return proj || hproj; }
};

// On the HOG source: checks the frames and sets up a host-frame gather (SD_ERR_INVALID before any work is queued).  On a host
// projection: the staging pair and the pinned copy of d_x.
int source_prepare(sd_ctx* ctx, RowSource& s, const float* d_x, int P, int N)
{
    if (s.hproj) return host_prepare(ctx, *s.hproj, s.h, d_x, N, P);
    return s.proj ? SD_OK : frames_prepare(ctx, s.frames, s.g, N);
}

// feature rows of samples [r0, r0 + rows) into columns [0, D) of the chunk buffer; P = the parameter width
int source_rows(sd_ctx* ctx, RowSource& s, const float* d_x, int P, int r0, int rows, float* d_chunk, int64_t ld)
{
    if (!s.callback()) return hog_rows(ctx, *s.frames, s.g, d_x, r0, rows, s.L, s.hog_eyes, s.p, d_chunk, ld);
    if (rows == 0) return SD_OK;                                     // a rank without samples
    if (s.hproj) return host_rows(ctx, *s.hproj, s.h, P, r0, rows, d_chunk, ld);
    const int rc = s.proj->fn(s.proj->user, ctx, s.proj->level, d_x + (int64_t)r0 * P, P, r0, rows, d_chunk, ld);
    return rc ? sd_fail(ctx, SD_ERR_INVALID, "projection callback returned %d", rc) : SD_OK;
}

// the end of a level on host frames: no patch may have read outside its planned region
int source_finish(sd_ctx* ctx, const RowSource& s, int N)
{
    return s.callback() || s.frames->images ? SD_OK : gather_finish(ctx, s.g, N);
}

// The rules of a caller's projection, device or host (SD_ERR_INVALID before any work is queued): a callback, D >= 1, and a
// normalisation that can read the parameter rows -- inter-eye distance needs [x.., y..] rows (even P) with its eye indices below
// P / 2.
template <class Desc>
int check_projection(sd_ctx* ctx, const char* fn, const Desc* proj, int P, const sd_normalisation* norm)
{
    if (!proj || !proj->fn || proj->feature_length < 1)
        return sd_fail(ctx, SD_ERR_INVALID, "%s: the projection needs a callback and feature_length >= 1", fn);
    if (P < 1) return sd_fail(ctx, SD_ERR_INVALID, "%s: P < 1", fn);
    if (norm && norm->kind == 1) {
        sd_eyes_dev eyes;
        if (P % 2 || sd_eyes_to_dev(ctx, norm, P / 2, &eyes))
            return sd_fail(ctx, SD_ERR_INVALID, "%s: inter-eye distance normalisation needs an even P and eye indices below P / 2", fn);
    } else if (norm && norm->kind != 0) {
        return sd_fail(ctx, SD_ERR_INVALID, "%s: unknown normalisation kind %d", fn, norm->kind);
    }
    return SD_OK;
}

// Several ranks on a caller's projection: a callback that fails on one rank must not leave the others waiting in a collective.  The
// failing rank still takes part in every collective up to the exchange (the centring's without rows), and the ranks agree on a
// failure -- one host integer -- before the exchange and at the end of the level, so either every rank fails the level or none.
int agree_on_failure(sd_ctx* ctx, const char* fn, const RowSource& s, sd_comm* c, int failed)
{
    if (!s.callback() || !c) return failed;
    int64_t any = failed != 0;
    const int rc = sd_comm_sum_int64(ctx, c, &any);
    if (failed) return failed;                                       // keeps its own message
    if (rc) return rc;
    return any ? sd_fail(ctx, SD_ERR_INVALID, "%s: the projection callback failed on another rank", fn) : SD_OK;
}

// One training level of D features on P parameters from the row source s (sd_train_level, sd_train_level_*projected); the caller
// has checked the arguments.
int train_rows(sd_ctx* ctx, const char* fn, sd_comm* comm, RowSource& s, int D, const float* d_x, const float* d_x_gt, int N_local,
               int P, int64_t n_global, const sd_normalisation* norm, const float* d_templates, int64_t ldt, const sd_regulariser* reg,
               int route, float* d_chunk, int64_t ld, int chunk_rows, float* d_X, float* d_x_next, float* lambda_out)
{
    int rc = source_prepare(ctx, s, d_x, P, N_local);
    if (rc) return rc;
    float* mu = (float*)sd_workspace(ctx, SD_WS_LEVEL, (size_t)D * (P + 1) * sizeof(float));
    if (!mu) return SD_ERR_CUDA;
    float* Xc = mu + D;                                   // weights for the shifted rows: what the update multiplies them with
    sd_comm* c = sd_comm_size_of(comm) > 1 ? comm : nullptr;
    float* B = d_chunk + D;                               // [A | b] side by side: the Gram reads both in one pass
    const int chunks = N_local > 0 ? sd_div_up(N_local, chunk_rows) : 1;
    // the pilot shift is the mean of every rank's first chunk (sd_centre_features also checks the all-ones bias column there)
    int64_t n0 = N_local < chunk_rows ? N_local : chunk_rows;
    rc = c ? sd_comm_sum_int64(ctx, c, &n0) : SD_OK;
    if (rc) return rc;
    if (n0 < 1) return sd_fail(ctx, SD_ERR_INVALID, "%s: no samples on any rank", fn);
    const bool shifted = D > SD_LU_MAX_DIM && !reg->regularise_last_row;     // otherwise sd_centre_features leaves mu = 0
    int failed = SD_OK;
    for (int k = 0; k < chunks; ++k) {
        const int r0 = k * chunk_rows, rows = N_local - r0 < chunk_rows ? N_local - r0 : chunk_rows;
        rc = source_rows(ctx, s, d_x, P, r0, rows, d_chunk, ld);                                                      // :173-189
        if (rc && s.callback() && c) {                    // agree_on_failure: the centring's collective without rows, then stop
            failed = rc;
            rc = k == 0 ? sd_centre_features(ctx, c, d_chunk, ld, 0, D, (int)n0, reg, mu) : SD_OK;
            if (rc) return rc;
            break;
        }
        if (!rc && d_templates) rc = sd_subtract_templates(ctx, d_chunk, ld, d_templates, ldt, rows, D);             // :191-197
        if (!rc) rc = sd_cascade_targets(ctx, d_x + (int64_t)r0 * P, d_x_gt + (int64_t)r0 * P, rows, P, norm, B, ld); // :199-205
        if (!rc) rc = k == 0 ? sd_centre_features(ctx, c, d_chunk, ld, rows, D, (int)n0, reg, mu)
                             : (shifted ? sd_shift_rows(ctx, d_chunk, ld, rows, D, mu) : SD_OK);
        if (!rc) rc = sd_learn_gram(ctx, d_chunk, ld, B, ld, rows, true, D, P, k > 0);
        if (rc) return rc;
    }
    rc = agree_on_failure(ctx, fn, s, c, failed);
    if (rc) return rc;
    rc = sd_learn_centred_solve(ctx, c, D, P, reg, (int)n_global, route, mu, d_X, Xc, lambda_out);                    // :207
    if (rc) return rc;
    // :209-215 -- the last chunk is still in the buffer; the others are projected and shifted again
    const int last = (chunks - 1) * chunk_rows;
    rc = sd_cascade_update(ctx, d_chunk, ld, N_local - last, D, Xc, P, d_x + (int64_t)last * P, norm, d_x_next + (int64_t)last * P);
    for (int k = 0; !rc && k + 1 < chunks; ++k) {
        const int r0 = k * chunk_rows;
        rc = source_rows(ctx, s, d_x, P, r0, chunk_rows, d_chunk, ld);
        if (!rc && shifted) rc = sd_shift_rows(ctx, d_chunk, ld, chunk_rows, D, mu);
        if (!rc) rc = sd_cascade_update(ctx, d_chunk, ld, chunk_rows, D, Xc, P, d_x + (int64_t)r0 * P, norm, d_x_next + (int64_t)r0 * P);
    }
    if (!rc) rc = source_finish(ctx, s, N_local);
    return agree_on_failure(ctx, fn, s, c, rc);
}

// One test / predict level of D features on P parameters from the row source s (sd_apply_level, sd_apply_level_*projected); the
// caller has checked the arguments.
int apply_rows(sd_ctx* ctx, RowSource& s, int D, const float* d_x, int N, int P, const sd_normalisation* norm, const float* d_templates,
               int64_t ldt, const float* d_X, float* d_chunk, int64_t ld, int chunk_rows, float* d_x_next)
{
    int rc = source_prepare(ctx, s, d_x, P, N);
    for (int r0 = 0; !rc && r0 < N; r0 += chunk_rows) {
        const int rows = N - r0 < chunk_rows ? N - r0 : chunk_rows;
        rc = source_rows(ctx, s, d_x, P, r0, rows, d_chunk, ld);
        if (!rc && d_templates) rc = sd_subtract_templates(ctx, d_chunk, ld, d_templates + (int64_t)r0 * ldt, ldt, rows, D);
        if (!rc) rc = sd_cascade_update(ctx, d_chunk, ld, rows, D, d_X, P, d_x + (int64_t)r0 * P, norm, d_x_next + (int64_t)r0 * P);
    }
    if (!rc) rc = source_finish(ctx, s, N);
    return rc;
}

// SD_REQUIRE for the projected levels, which name the entry point `fn` in their messages
#define SD_REQUIRE_IN(ctx, fn, cond, msg)                                                      \
    do {                                                                                       \
        if (!(cond)) return sd_fail((ctx), SD_ERR_INVALID, "%s: %s", (fn), msg);               \
    } while (0)

// sd_train_level_projected / sd_train_level_host_projected: the argument checks, then the level from the caller's projection
template <class Desc>
int train_projected(sd_ctx* ctx, const char* fn, sd_comm* comm, const Desc* proj, const float* d_x, const float* d_x_gt, int N_local,
                    int P, int64_t n_global, const sd_normalisation* norm, const float* d_templates, int64_t ldt, const sd_regulariser* reg,
                    int route, float* d_chunk, int64_t ld, int chunk_rows, float* d_X, float* d_x_next, float* lambda_out)
{
    if (!ctx) return SD_ERR_INVALID;
    SD_REQUIRE_IN(ctx, fn, d_x && d_x_gt && reg && d_chunk && d_X && d_x_next, "null argument");
    SD_REQUIRE_IN(ctx, fn, N_local >= 0 && n_global >= 1 && n_global <= INT_MAX, "bad sample count");
    SD_REQUIRE_IN(ctx, fn, chunk_rows >= 1, "chunk_rows must be >= 1");
    SD_REQUIRE_IN(ctx, fn, reg->type == 0 || reg->type == 1, "unknown regularisation type");
    const int rc = check_projection(ctx, fn, proj, P, norm);
    if (rc) return rc;
    const int D = proj->feature_length;
    SD_REQUIRE_IN(ctx, fn, ld >= (int64_t)D + P, "ld < D + P");
    SD_REQUIRE_IN(ctx, fn, !d_templates || (chunk_rows >= N_local && ldt >= D), "templates need one chunk (chunk_rows >= N_local) and ldt >= D");
    SD_REQUIRE_IN(ctx, fn, d_x_next != d_x, "x_next must not alias x");
    RowSource s;
    s.use(proj);
    return train_rows(ctx, fn, comm, s, D, d_x, d_x_gt, N_local, P, n_global, norm, d_templates, ldt, reg, route, d_chunk, ld,
                      chunk_rows, d_X, d_x_next, lambda_out);
}

// sd_apply_level_projected / sd_apply_level_host_projected
template <class Desc>
int apply_projected(sd_ctx* ctx, const char* fn, const Desc* proj, const float* d_x, int N, int P, const sd_normalisation* norm,
                    const float* d_templates, int64_t ldt, const float* d_X, float* d_chunk, int64_t ld, int chunk_rows, float* d_x_next)
{
    if (!ctx) return SD_ERR_INVALID;
    SD_REQUIRE_IN(ctx, fn, d_x && d_X && d_chunk && d_x_next, "null argument");
    SD_REQUIRE_IN(ctx, fn, N >= 0, "bad sample count");
    SD_REQUIRE_IN(ctx, fn, chunk_rows >= 1, "chunk_rows must be >= 1");
    const int rc = check_projection(ctx, fn, proj, P, norm);
    if (rc) return rc;
    const int D = proj->feature_length;
    SD_REQUIRE_IN(ctx, fn, ld >= D, "ld < D");
    SD_REQUIRE_IN(ctx, fn, !d_templates || ldt >= D, "ldt < D");
    SD_REQUIRE_IN(ctx, fn, d_x_next != d_x, "x_next must not alias x");
    RowSource s;
    s.use(proj);
    return apply_rows(ctx, s, D, d_x, N, P, norm, d_templates, ldt, d_X, d_chunk, ld, chunk_rows, d_x_next);
}

#undef SD_REQUIRE_IN

}  // namespace

extern "C" {

int sd_train_level(sd_ctx* ctx, sd_comm* comm, const sd_level_frames* frames, const float* d_x, const float* d_x_gt, int N_local, int L,
                   int64_t n_global, const sd_normalisation* hog_eyes, const sd_hog_param* p, const sd_normalisation* norm,
                   const float* d_templates, int64_t ldt, const sd_regulariser* reg, int route, float* d_chunk, int64_t ld, int chunk_rows,
                   float* d_X, float* d_x_next, float* lambda_out)
{
    if (!ctx) return SD_ERR_INVALID;
    SD_REQUIRE(ctx, d_x && d_x_gt && p && reg && d_chunk && d_X && d_x_next, "null argument");
    SD_REQUIRE(ctx, N_local >= 0 && L >= 1 && n_global >= 1 && n_global <= INT_MAX, "bad sample / landmark count");
    SD_REQUIRE(ctx, chunk_rows >= 1, "chunk_rows must be >= 1");
    SD_REQUIRE(ctx, reg->type == 0 || reg->type == 1, "unknown regularisation type");
    const int D = sd_hog_feature_length(L, p), P = 2 * L;
    SD_REQUIRE(ctx, D >= 2, "bad HOG parameters");
    SD_REQUIRE(ctx, ld >= (int64_t)D + P, "ld < D + 2L");
    SD_REQUIRE(ctx, !d_templates || (chunk_rows >= N_local && ldt >= D), "templates need one chunk (chunk_rows >= N_local) and ldt >= D");
    SD_REQUIRE(ctx, d_x_next != d_x, "x_next must not alias x");
    RowSource s;
    s.frames = frames;
    s.L = L;
    s.hog_eyes = hog_eyes;
    s.p = p;
    return train_rows(ctx, __func__, comm, s, D, d_x, d_x_gt, N_local, P, n_global, norm, d_templates, ldt, reg, route, d_chunk, ld,
                      chunk_rows, d_X, d_x_next, lambda_out);
}

int sd_apply_level(sd_ctx* ctx, const sd_level_frames* frames, const float* d_x, int N, int L, const sd_normalisation* hog_eyes,
                   const sd_hog_param* p, const sd_normalisation* norm, const float* d_templates, int64_t ldt, const float* d_X,
                   float* d_chunk, int64_t ld, int chunk_rows, float* d_x_next)
{
    if (!ctx) return SD_ERR_INVALID;
    SD_REQUIRE(ctx, d_x && p && d_X && d_chunk && d_x_next, "null argument");
    SD_REQUIRE(ctx, N >= 0 && L >= 1, "bad sample / landmark count");
    SD_REQUIRE(ctx, chunk_rows >= 1, "chunk_rows must be >= 1");
    const int D = sd_hog_feature_length(L, p), P = 2 * L;
    SD_REQUIRE(ctx, D >= 2, "bad HOG parameters");
    SD_REQUIRE(ctx, ld >= D, "ld < D");
    SD_REQUIRE(ctx, !d_templates || ldt >= D, "ldt < D");
    SD_REQUIRE(ctx, d_x_next != d_x, "x_next must not alias x");
    RowSource s;
    s.frames = frames;
    s.L = L;
    s.hog_eyes = hog_eyes;
    s.p = p;
    return apply_rows(ctx, s, D, d_x, N, P, norm, d_templates, ldt, d_X, d_chunk, ld, chunk_rows, d_x_next);
}

int sd_train_level_projected(sd_ctx* ctx, sd_comm* comm, const sd_level_projection* proj, const float* d_x, const float* d_x_gt,
                             int N_local, int P, int64_t n_global, const sd_normalisation* norm, const float* d_templates, int64_t ldt,
                             const sd_regulariser* reg, int route, float* d_chunk, int64_t ld, int chunk_rows, float* d_X,
                             float* d_x_next, float* lambda_out)
{
    return train_projected(ctx, __func__, comm, proj, d_x, d_x_gt, N_local, P, n_global, norm, d_templates, ldt, reg, route, d_chunk, ld,
                           chunk_rows, d_X, d_x_next, lambda_out);
}

int sd_apply_level_projected(sd_ctx* ctx, const sd_level_projection* proj, const float* d_x, int N, int P, const sd_normalisation* norm,
                             const float* d_templates, int64_t ldt, const float* d_X, float* d_chunk, int64_t ld, int chunk_rows,
                             float* d_x_next)
{
    return apply_projected(ctx, __func__, proj, d_x, N, P, norm, d_templates, ldt, d_X, d_chunk, ld, chunk_rows, d_x_next);
}

int sd_train_level_host_projected(sd_ctx* ctx, sd_comm* comm, const sd_level_host_projection* proj, const float* d_x, const float* d_x_gt,
                                  int N_local, int P, int64_t n_global, const sd_normalisation* norm, const float* d_templates,
                                  int64_t ldt, const sd_regulariser* reg, int route, float* d_chunk, int64_t ld, int chunk_rows,
                                  float* d_X, float* d_x_next, float* lambda_out)
{
    return train_projected(ctx, __func__, comm, proj, d_x, d_x_gt, N_local, P, n_global, norm, d_templates, ldt, reg, route, d_chunk, ld,
                           chunk_rows, d_X, d_x_next, lambda_out);
}

int sd_apply_level_host_projected(sd_ctx* ctx, const sd_level_host_projection* proj, const float* d_x, int N, int P,
                                  const sd_normalisation* norm, const float* d_templates, int64_t ldt, const float* d_X, float* d_chunk,
                                  int64_t ld, int chunk_rows, float* d_x_next)
{
    return apply_projected(ctx, __func__, proj, d_x, N, P, norm, d_templates, ldt, d_X, d_chunk, ld, chunk_rows, d_x_next);
}

int sd_level_chunk_rows(sd_ctx* ctx, sd_comm* comm, const sd_level_frames* frames, int64_t N_local, int D, int M, int route,
                        size_t free_bytes, int* rows_out)
{
    if (!ctx) return SD_ERR_INVALID;
    SD_REQUIRE(ctx, rows_out && N_local >= 0 && D >= 1 && M >= 1, "bad argument");
    int rc = frames ? check_frames(ctx, frames) : SD_OK;
    if (rc) return rc;
    if (free_bytes == 0) {
        size_t total = 0;
        SD_CUDA(ctx, cudaSetDevice(ctx->device));
        SD_CUDA(ctx, cudaMemGetInfo(&free_bytes, &total));
    }
    const int64_t ld = sd_learn_ldg(D, M);
    const int nranks = sd_comm_size_of(comm);
    // what the level's solve will still allocate with the context's settings, less what the context already holds
    size_t need = 0;
    auto add = [&](int slot, size_t bytes) { if (bytes > ctx->ws_bytes[slot]) need += bytes - ctx->ws_bytes[slot]; };
    const size_t gram = (size_t)D * ld * sizeof(float);
    add(SD_WS_SCRATCH, gram);
    add(SD_WS_LEVEL, (size_t)D * (M + 1) * sizeof(float));
    if (nranks > 1) add(SD_WS_GRAM_EXT, gram);                                          // band buffer of the exchange (at most G)
    if (ctx->rank_diagnostic && !(nranks > 1 && route == 1))                            // the rank's copy of the system
        add(SD_WS_RANK, (size_t)(D + 130) * round_up(D, 4) * sizeof(float) + 4096);
    if (D > SD_LU_MAX_DIM) {
        const size_t n = (size_t)D - 1;
        add(SD_WS_BIAS, (size_t)(D + M) * sizeof(double) + n * (M + 1) * sizeof(float));
        add(SD_WS_DIAGINV2, round_up(n, 128) / 128 * 2 * 128 * 128 * sizeof(float));    // the Cholesky's inverse diagonal blocks
        if (ctx->solver_mode == 1 || (nranks > 1 && route == 2))                        // CG's strip-major copy of the system
            add(SD_WS_CGMAT, round_up(n, 128) * round_up(n, 16) * sizeof(float));
    }
    if (frames && frames->host_frames) {                                                // the staging pair of the gather
        size_t largest = 0;
        for (int f = 0; f < frames->num_host_frames; ++f)
            largest = sd_gray_bytes(frames->host_frames[f]) > largest ? sd_gray_bytes(frames->host_frames[f]) : largest;
        const size_t half = stage_half(*frames, largest);
        for (int b = 0; b < 2; ++b)
            if (half > ctx->stage_bytes[b]) need += half - ctx->stage_bytes[b];
    }
    // per row: the caller's chunk row and the update's partial sums (sd_cascade_update)
    const size_t per_row = (size_t)ld * sizeof(float) + (size_t)M * sizeof(double);
    const size_t fixed = need + kReserveBytes;
    const int64_t fit = free_bytes > fixed ? (int64_t)((free_bytes - fixed) / per_row) : 0;
    const int64_t least = N_local < kMinChunkRows ? N_local : kMinChunkRows;
    if (fit < least)
        return sd_fail(ctx, SD_ERR_CUDA, "sd_level_chunk_rows: D = %d: the solve needs %.2f GB and %lld rows of %.1f KB do not fit beside it "
                       "in %.2f GB", D, need / 1e9, (long long)least, per_row / 1e3, free_bytes / 1e9);
    int64_t rows = fit < N_local ? fit : N_local;
    if (rows > INT_MAX) rows = INT_MAX;
    *rows_out = rows < 1 ? 1 : (int)rows;
    return SD_OK;
}

int64_t sd_gathered_bytes(const sd_ctx* ctx) { return ctx ? ctx->gathered_bytes : 0; }

int sd_host_frame_in_place(sd_ctx* ctx, const sd_host_frame* frame, int* in_place)
{
    if (!ctx) return SD_ERR_INVALID;
    SD_REQUIRE(ctx, frame && in_place, "null argument");
    const int rc = sd_check_host_frame(ctx, __func__, *frame, 0);
    if (rc) return rc;
    PinnedRange last;
    const uint8_t* m = sd_mapped_frame(frame->h_data, sd_host_frame_bytes(*frame), last);
    *in_place = m && ((reinterpret_cast<uintptr_t>(m) | (uintptr_t)frame->row_stride) & 15) == 0 &&
                (size_t)frame->row_stride >= (size_t)frame->channels * sd_round16(frame->width);
    return SD_OK;
}

int sd_device_memory(sd_ctx* ctx, size_t* free_bytes, size_t* total_bytes)
{
    if (!ctx) return SD_ERR_INVALID;
    SD_REQUIRE(ctx, free_bytes && total_bytes, "null argument");
    SD_CUDA(ctx, cudaSetDevice(ctx->device));
    SD_CUDA(ctx, cudaMemGetInfo(free_bytes, total_bytes));
    return SD_OK;
}

}  // extern "C"
