// Training HOG filters for the sliding-window detector (sd_hog_windows, sd_hog_box_windows, sd_learn_squared_hinge,
// sd_hog_train_filter): the feature rows of score positions, the window that covers a ground-truth box, a squared-hinge
// linear SVM on the learn path, and the hard-negative mining loop that composes them with the pyramid routine
// (sd_hog_pyramid_frames), sd_hog_correlate and sd_hog_detections.
//
// The window gather is one CTA per row: its threads walk the row's columns in order, so the stores of a row are coalesced and
// the loads of one (channel, dy) run of fw cells are consecutive floats of the map.  The SVM's kernels are the margins (one
// warp per row, a float64 dot product in a fixed lane order and a fixed shuffle tree) and the active-row compaction (one CTA
// per row of a host-built index list in row order); neither uses atomics, so every result is the same in every run.
#include "sd_internal.cuh"

#include <algorithm>
#include <chrono>
#include <cfloat>
#include <cmath>
#include <cstring>
#include <set>
#include <tuple>
#include <vector>

namespace {

constexpr int kGatherThreads = 256;
constexpr int kMaxDd = 4 * SD_MAX_BINS;          // the largest dd (Dalal-Triggs at K = 16)
constexpr size_t kSliceFloats = size_t(64) << 20; // pyramid features of one slice of the trainer's frames: 256 MB

struct WindowArgs {
    const float* maps;
    const sd_hog_grid* grids;    // per-grid descriptors, or null: equally sized grids
    int width, height;           // equally sized grids
    long long in_stride;
    const sd_hog_window* windows;
    const int* dest;             // row of window r in d_rows, or null: row r
    int count, dd, fw, fh, pad_x, pad_y, D;
    long long ldr;
    float* rows;
    int perm[kMaxDd];            // sd_hog_permutation: plane c of a flipped window reads plane perm[c]
};

__global__ void __launch_bounds__(kGatherThreads) hog_windows_kernel(const __grid_constant__ WindowArgs a)
{
    const int taps = a.fh * a.fw;
    for (int r = blockIdx.x; r < a.count; r += gridDim.x) {
        const sd_hog_window win = a.windows[r];
        int W, H;
        const float* __restrict__ M;
        if (a.grids) {
            const sd_hog_grid d = a.grids[win.grid];
            W = d.width; H = d.height;
            M = a.maps + d.offset;
        } else {
            W = a.width; H = a.height;
            M = a.maps + (long long)win.grid * a.in_stride;
        }
        const long long plane = (long long)W * H;
        float* __restrict__ out = a.rows + (long long)(a.dest ? a.dest[r] : r) * a.ldr;
        for (int j = threadIdx.x; j < a.D; j += kGatherThreads) {
            float v = 1.0f;                                          // column D - 1: the bias
            if (j < a.D - 1) {
                const int c = j / taps, t = j - c * taps;
                const int dy = t / a.fw, dx = t - dy * a.fw;
                // a flipped window is sd_hog_relayout(flip = 1) of the block it reads: plane perm[c], columns mirrored
                const int src_c = win.flip ? a.perm[c] : c;
                const int gx = win.x - a.pad_x + (win.flip ? a.fw - 1 - dx : dx);
                const int gy = win.y - a.pad_y + dy;
                v = (unsigned)gx < (unsigned)W && (unsigned)gy < (unsigned)H ? __ldg(M + src_c * plane + (long long)gy * W + gx) : 0.f;
            }
            out[j] = v;
        }
    }
}

// o[i] = a_i . w in float64, products and sums in a fixed order: lane l sums columns l, l + 32, ..., then a fixed shuffle tree
__global__ void __launch_bounds__(256) svm_margins_kernel(const float* __restrict__ A, long long lda, int N, int D,
                                                          const float* __restrict__ w, double* __restrict__ o)
{
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    const int warps = (gridDim.x * blockDim.x) >> 5;
    for (int i = warp; i < N; i += warps) {
        const float* row = A + (long long)i * lda;
        double s = 0.0;
        for (int j = lane; j < D; j += 32) s = fma((double)__ldg(row + j), (double)__ldg(w + j), s);
#pragma unroll
        for (int k = 16; k > 0; k >>= 1) s += __shfl_xor_sync(0xffffffffu, s, k);
        if (lane == 0) o[i] = s;
    }
}

// row r of S = [row idx[r] of A | y[idx[r]]]: the active rows in row order with their labels beside them (the Gram reads
// [A_S | y_S] as one matrix)
__global__ void __launch_bounds__(256) svm_compact_kernel(const float* __restrict__ A, long long lda, const float* __restrict__ y,
                                                          const int* __restrict__ idx, int n, int D, float* __restrict__ S, long long lds)
{
    for (int r = blockIdx.x; r < n; r += gridDim.x) {
        const int i = idx[r];
        const float* src = A + (long long)i * lda;
        float* dst = S + (long long)r * lds;
        for (int j = threadIdx.x; j < D; j += blockDim.x) dst[j] = __ldg(src + j);
        if (threadIdx.x == 0) dst[D] = __ldg(y + i);
    }
}

int launch_windows(sd_ctx* ctx, const float* maps, const sd_hog_grid* d_grids, int width, int height, int num_bins, int variant,
                   int fw, int fh, int pad_x, int pad_y, const sd_hog_window* d_windows, const int* d_dest, int count, float* d_rows,
                   int64_t ldr)
{
    if (count == 0) return SD_OK;
    WindowArgs a;
    memset(&a, 0, sizeof(a));
    a.maps = maps; a.grids = d_grids; a.width = width; a.height = height;
    a.dd = sd_hog_dd(num_bins, variant);
    a.in_stride = (long long)a.dd * width * height;
    a.windows = d_windows; a.dest = d_dest; a.count = count;
    a.fw = fw; a.fh = fh; a.pad_x = pad_x; a.pad_y = pad_y;
    a.D = a.dd * fw * fh + 1;
    a.ldr = ldr; a.rows = d_rows;
    int64_t perm[kMaxDd];
    sd_hog_permutation(num_bins, variant, perm);
    for (int c = 0; c < a.dd; ++c) a.perm[c] = (int)perm[c];
    const int blocks = std::min(count, 16 * ctx->sm_count);
    hog_windows_kernel<<<blocks, kGatherThreads, 0, ctx->stream>>>(a);
    SD_LAUNCH_CHECK(ctx, "hog_windows_kernel");
    return SD_OK;
}

// ---- exact IoU of detection boxes ------------------------------------------------------------------------------------------
// intersection and union of two boxes in int64 pixel areas
void inter_union(const sd_box64& a, const sd_box64& b, int64_t* inter, int64_t* uni)
{
    const int64_t iw = std::min(a.x1, b.x1) - std::max(a.x0, b.x0), ih = std::min(a.y1, b.y1) - std::max(a.y0, b.y0);
    *inter = iw > 0 && ih > 0 ? iw * ih : 0;
    *uni = (a.x1 - a.x0) * (a.y1 - a.y0) + (b.x1 - b.x0) * (b.y1 - b.y0) - *inter;
}

struct Level { int level_w, level_h, hog_w, hog_h; };

// sd_hog_box_windows for one box over a frame's level table (levels with hog_w = 0 are empty)
void best_window(const std::vector<Level>& lv, int frame_w, int frame_h, int cell_size, int fw, int fh, int pad_x, int pad_y,
                 double positive_overlap, const sd_box64& box, sd_hog_window* out, double* iou)
{
    int64_t bi = 0, bu = 1;                           // best IoU so far as a rational, -1 / 1 before the first candidate
    bool any = false;
    sd_hog_window best = {-1, 0, 0, 0};
    for (int s = 0; s < (int)lv.size(); ++s) {
        if (!lv[s].hog_w) continue;
        const int oh = sd_score_extent(lv[s].hog_h, pad_y, fh), ow = sd_score_extent(lv[s].hog_w, pad_x, fw);
        for (int y = 0; y < oh; ++y)
            for (int x = 0; x < ow; ++x) {
                const sd_box64 b = sd_window_box(x, y, pad_x, pad_y, fw, fh, cell_size, frame_w, frame_h, lv[s].level_w, lv[s].level_h);
                int64_t in, un;
                inter_union(box, b, &in, &un);
                // in / un > bi / bu, exactly (both unions are positive)
                if (!any || (__int128)in * bu > (__int128)bi * un) {
                    any = true;
                    bi = in; bu = un;
                    best = {s, x, y, 0};
                }
            }
    }
    *iou = any ? (double)bi / (double)bu : 0.0;
    if (!any || !((double)bi >= positive_overlap * (double)bu)) best = {-1, 0, 0, 0};
    *out = best;
}

int level_table(int frame_w, int frame_h, const double* scales, int num_scales, int cell_size, int num_bins, int variant,
                std::vector<Level>* lv)
{
    lv->resize(num_scales);
    for (int s = 0; s < num_scales; ++s) {
        int dd;
        Level& l = (*lv)[s];
        if (sd_hog_pyramid_shape(frame_w, frame_h, scales[s], cell_size, num_bins, variant, &l.level_w, &l.level_h, &l.hog_w, &l.hog_h, &dd))
            return SD_ERR_INVALID;
    }
    return SD_OK;
}

// ---- the squared-hinge SVM -----------------------------------------------------------------------------------------------
// f(w) from the margins o_i = a_i . w, in float64
double svm_objective(const std::vector<double>& o, const std::vector<float>& y, const float* w, int D, double lambda)
{
    double reg = 0.0, loss = 0.0;
    for (int j = 0; j < D - 1; ++j) reg += (double)w[j] * (double)w[j];
    for (size_t i = 0; i < o.size(); ++i) {
        const double r = 1.0 - (double)y[i] * o[i];
        if (r > 0) loss += r * r;
    }
    return 0.5 * lambda * reg + 0.5 * loss;
}

// The exact minimiser t >= 0 of phi(t) = f(w + t d), a convex piecewise quadratic: phi'(t) = b + a t between breakpoints, where
// row i is active while alpha_i - t beta_i > 0 (alpha_i = 1 - y_i o_i, beta_i = y_i delta_i, delta_i = a_i . d).
double line_search(const std::vector<double>& o, const std::vector<double>& z, const std::vector<float>& y, const float* w,
                   const float* wn, int D, double lambda)
{
    double dd = 0.0, wd = 0.0;
    for (int j = 0; j < D - 1; ++j) {
        const double d = (double)wn[j] - (double)w[j];
        dd += d * d;
        wd += (double)w[j] * d;
    }
    double a = lambda * dd, b = lambda * wd;
    std::vector<std::pair<double, int>> brk;
    for (size_t i = 0; i < o.size(); ++i) {
        const double al = 1.0 - (double)y[i] * o[i], be = (double)y[i] * (z[i] - o[i]);
        if (al > 0 || (al == 0 && be < 0)) {          // active just after t = 0
            a += be * be;
            b -= be * al;
            if (be > 0) brk.push_back({al / be, (int)i});   // leaves at al / be
        } else if (be < 0) {
            brk.push_back({al / be, (int)i});               // enters at al / be (> 0)
        }
    }
    std::sort(brk.begin(), brk.end());
    double t0 = 0.0;
    for (const auto& e : brk) {
        if (a > 0 && -b / a <= e.first) return std::max(t0, -b / a);
        const int i = e.second;
        const double al = 1.0 - (double)y[i] * o[i], be = (double)y[i] * (z[i] - o[i]);
        const double sgn = be > 0 ? -1.0 : 1.0;       // leaves or enters
        a += sgn * be * be;
        b -= sgn * be * al;
        t0 = e.first;
    }
    return a > 0 ? std::max(t0, -b / a) : 1.0;
}

int svm_margins(sd_ctx* ctx, const float* d_A, int64_t lda, int N, int D, const float* d_w, double* d_o, std::vector<double>& o)
{
    const int blocks = std::min(sd_div_up((int64_t)N * 32, 256), 8 * ctx->sm_count);
    svm_margins_kernel<<<blocks, 256, 0, ctx->stream>>>(d_A, lda, N, D, d_w, d_o);
    SD_LAUNCH_CHECK(ctx, "svm_margins_kernel");
    o.resize(N);
    SD_CUDA(ctx, cudaMemcpyAsync(o.data(), d_o, sizeof(double) * N, cudaMemcpyDeviceToHost, ctx->stream));
    SD_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return SD_OK;
}

std::vector<int> active_rows(const std::vector<double>& o, const std::vector<float>& y)
{
    std::vector<int> s;
    for (size_t i = 0; i < o.size(); ++i)
        if ((double)y[i] * o[i] < 1.0) s.push_back((int)i);
    return s;
}

// the solve behind sd_learn_squared_hinge, arguments checked; h_y: the labels on the host as well
int squared_hinge(sd_ctx* ctx, const float* d_A, int64_t lda, const float* d_y, const std::vector<float>& y, int N, int D, float lambda,
                  int max_iterations, float* d_w, sd_svm_report* report)
{
    const int64_t lds = ((int64_t)D + 1 + 3) / 4 * 4;       // [A_S | y_S], 16-byte rows for the tensor-core Gram
    const size_t s_bytes = (size_t)N * lds * sizeof(float);
    const size_t o_bytes = (size_t)N * sizeof(double);
    const size_t v_bytes = (size_t)(2 * D + 2) * sizeof(float);
    unsigned char* ws = static_cast<unsigned char*>(sd_workspace(ctx, SD_WS_SVM, s_bytes + o_bytes + v_bytes + (size_t)N * sizeof(int) + 64));
    if (!ws) return SD_ERR_CUDA;
    float* S = reinterpret_cast<float*>(ws);
    double* d_o = reinterpret_cast<double*>(ws + s_bytes);
    float* d_mu = reinterpret_cast<float*>(ws + s_bytes + o_bytes);
    float* d_wn = d_mu + D + 1;                              // the Newton point of the current step
    int* d_idx = reinterpret_cast<int*>(ws + s_bytes + o_bytes + v_bytes);

    sd_regulariser reg = {0, lambda, 0};
    std::vector<float> w(D, 0.f), wn(D);
    std::vector<double> o(N, 0.0), z;
    SD_CUDA(ctx, cudaMemsetAsync(d_w, 0, sizeof(float) * D, ctx->stream));
    double f = svm_objective(o, y, w.data(), D, lambda);
    std::vector<int> act(N);                                 // at w = 0 every row is active
    for (int i = 0; i < N; ++i) act[i] = i;
    int stop = SD_SVM_ITERATION_CAP, it = 0;
    for (it = 1; it <= max_iterations; ++it) {
        const int n = (int)act.size();
        int rc = SD_OK;
        if (n == 0) {
            // no active row: f = lambda / 2 |w'|^2 near w, whose Newton point is w' = 0 with the bias unchanged (the bias has no
            // curvature there)
            for (int j = 0; j < D - 1; ++j) wn[j] = 0.f;
            wn[D - 1] = w[D - 1];
            SD_CUDA(ctx, cudaMemcpyAsync(d_wn, wn.data(), sizeof(float) * D, cudaMemcpyHostToDevice, ctx->stream));
        } else {
            SD_CUDA(ctx, cudaMemcpyAsync(d_idx, act.data(), sizeof(int) * n, cudaMemcpyHostToDevice, ctx->stream));
            svm_compact_kernel<<<std::min(n, 16 * ctx->sm_count), 256, 0, ctx->stream>>>(d_A, lda, d_y, d_idx, n, D, S, lds);
            SD_LAUNCH_CHECK(ctx, "svm_compact_kernel");
            // one column shift for the whole solve, the means of all rows (every row is active in the first step); the bias is
            // not regularised, so each step on shifted rows is the same least-squares problem (sd_centre_features)
            rc = it == 1 ? sd_centre_features(ctx, nullptr, S, lds, n, D, n, &reg, d_mu)
                         : D > SD_LU_MAX_DIM ? sd_shift_rows(ctx, S, lds, n, D, d_mu) : SD_OK;   // small systems: mu = 0
            if (rc) return rc;
            rc = sd_learn_centred(ctx, nullptr, S, lds, S + D, lds, n, D, 1, &reg, n, 0, d_mu, d_wn, nullptr, nullptr);
            if (rc) return rc;
            SD_CUDA(ctx, cudaMemcpyAsync(wn.data(), d_wn, sizeof(float) * D, cudaMemcpyDeviceToHost, ctx->stream));
        }
        if ((rc = svm_margins(ctx, d_A, lda, N, D, d_wn, d_o, z))) return rc;
        std::vector<int> act_n = active_rows(z, y);
        std::vector<float> wt;
        std::vector<double>* ot = &z;
        if (act_n == act) {
            wt = wn;                                         // the Newton point keeps its active set: the optimum
        } else {
            const double t = line_search(o, z, y, w.data(), wn.data(), D, lambda);
            wt.resize(D);
            for (int j = 0; j < D; ++j) wt[j] = (float)((double)w[j] + t * ((double)wn[j] - (double)w[j]));
            if (wt != wn) {
                SD_CUDA(ctx, cudaMemcpyAsync(d_wn, wt.data(), sizeof(float) * D, cudaMemcpyHostToDevice, ctx->stream));
                if ((rc = svm_margins(ctx, d_A, lda, N, D, d_wn, d_o, z))) return rc;
                act_n = active_rows(z, y);
            }
        }
        const double fn = svm_objective(*ot, y, wt.data(), D, lambda);
        if (!(fn < f)) {                                     // keep the last point that decreased f
            stop = SD_SVM_NO_DECREASE;
            break;
        }
        f = fn;
        w = wt;
        o = *ot;
        SD_CUDA(ctx, cudaMemcpyAsync(d_w, d_wn, sizeof(float) * D, cudaMemcpyDeviceToDevice, ctx->stream));
        const bool same = act_n == act;
        act.swap(act_n);
        if (same) {
            stop = SD_SVM_CONVERGED;
            break;
        }
    }
    SD_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (report) {
        report->iterations = std::min(it, max_iterations);
        report->active = (int)active_rows(o, y).size();
        report->stop = stop;
        report->reserved = 0;
        report->objective = f;
    }
    return SD_OK;
}

// ---- the trainer ---------------------------------------------------------------------------------------------------------
struct Win { int frame, level, x, y; };
bool operator<(const Win& a, const Win& b) { return std::tie(a.frame, a.level, a.x, a.y) < std::tie(b.frame, b.level, b.x, b.y); }

}  // namespace

extern "C" {

int sd_hog_windows(sd_ctx* ctx, const sd_hog_grids* maps, int num_bins, int variant, int filter_w, int filter_h, int pad_x, int pad_y,
                   const sd_hog_window* d_windows, int count, float* d_rows, int64_t ldr)
{
    if (!ctx) return SD_ERR_INVALID;
    SD_REQUIRE(ctx, maps && d_windows && d_rows, "null argument");
    if (const int rc = sd_hog_check_config(ctx, __func__, variant, num_bins)) return rc;
    if (const int rc = sd_hog_check_filter(ctx, __func__, filter_w, filter_h, pad_x, pad_y)) return rc;
    SD_REQUIRE(ctx, sd_aligned(d_windows, 4) && sd_aligned(d_rows, 4), "windows and rows must be 4-byte aligned");
    SD_REQUIRE(ctx, count >= 0 && maps->count >= 0, "negative count");
    const int64_t D = (int64_t)sd_hog_dd(num_bins, variant) * filter_w * filter_h + 1;
    SD_REQUIRE(ctx, ldr >= D, "ldr must be at least dd * filter_h * filter_w + 1");
    if (count == 0) return SD_OK;
    SD_REQUIRE(ctx, maps->count >= 1 && maps->d_features && sd_aligned(maps->d_features, 4), "maps must be non-null and 4-byte aligned");
    int max_w = 0, max_h = 0;
    std::vector<sd_hog_grid> table;
    if (const int rc = sd_read_hog_grids(ctx, __func__, maps, &max_w, &max_h, &table)) return rc;
    std::vector<sd_hog_window> win;
    if (const int rc = sd_fetch_table(ctx, d_windows, count, win)) return rc;
    for (int r = 0; r < count; ++r) {
        const sd_hog_window& v = win[r];
        if (v.grid < 0 || v.grid >= maps->count || (v.flip != 0 && v.flip != 1))
            return sd_fail(ctx, SD_ERR_INVALID, "%s: window %d: grid %d out of [0, %d) or flip %d not 0 or 1", __func__, r, v.grid,
                           maps->count, v.flip);
        const int w = maps->d_grids ? table[v.grid].width : max_w, h = maps->d_grids ? table[v.grid].height : max_h;
        const int ow = sd_score_extent(w, pad_x, filter_w), oh = sd_score_extent(h, pad_y, filter_h);
        if (v.x < 0 || v.x >= ow || v.y < 0 || v.y >= oh)
            return sd_fail(ctx, SD_ERR_INVALID, "%s: window %d: (%d, %d) is not a score position of grid %d (%d x %d)", __func__, r, v.x,
                           v.y, v.grid, ow > 0 ? ow : 0, oh > 0 ? oh : 0);
    }
    return launch_windows(ctx, maps->d_features, maps->d_grids, max_w, max_h, num_bins, variant, filter_w, filter_h, pad_x, pad_y,
                          d_windows, nullptr, count, d_rows, ldr);
}

int sd_hog_box_windows(int frame_w, int frame_h, const double* scales, int num_scales, int cell_size, int num_bins, int variant,
                       int filter_w, int filter_h, int pad_x, int pad_y, double positive_overlap, const int32_t* boxes, int num_boxes,
                       sd_hog_window* out, double* iou)
{
    if (!scales || num_scales < 1 || num_boxes < 0 || (num_boxes > 0 && (!boxes || !out || !iou))) return SD_ERR_INVALID;
    if (frame_w < 1 || frame_h < 1 || !(positive_overlap >= 0.0 && positive_overlap <= 1.0)) return SD_ERR_INVALID;
    if (sd_hog_check_filter(nullptr, __func__, filter_w, filter_h, pad_x, pad_y)) return SD_ERR_INVALID;
    std::vector<Level> lv;
    if (level_table(frame_w, frame_h, scales, num_scales, cell_size, num_bins, variant, &lv)) return SD_ERR_INVALID;
    for (int b = 0; b < num_boxes; ++b)
        if (boxes[4 * b + 2] < 1 || boxes[4 * b + 3] < 1) return SD_ERR_INVALID;
    for (int b = 0; b < num_boxes; ++b) {
        const int32_t* q = boxes + 4 * b;
        const sd_box64 box = {q[0], q[1], (int64_t)q[0] + q[2], (int64_t)q[1] + q[3]};
        best_window(lv, frame_w, frame_h, cell_size, filter_w, filter_h, pad_x, pad_y, positive_overlap, box, out + b, iou + b);
    }
    return SD_OK;
}

int sd_learn_squared_hinge(sd_ctx* ctx, const float* d_A, int64_t lda, const float* d_y, int N, int D, float lambda, int max_iterations,
                           float* d_w, sd_svm_report* report)
{
    if (!ctx) return SD_ERR_INVALID;
    SD_REQUIRE(ctx, d_A && d_y && d_w, "null argument");
    SD_REQUIRE(ctx, N >= 1 && D >= 2 && lda >= D, "N must be >= 1, D >= 2 and lda >= D");
    SD_REQUIRE(ctx, lambda > 0.f && std::isfinite(lambda), "lambda must be positive and finite");
    SD_REQUIRE(ctx, max_iterations >= 1, "max_iterations must be >= 1");
    SD_REQUIRE(ctx, sd_aligned(d_A, 4) && sd_aligned(d_y, 4) && sd_aligned(d_w, 4), "A, y and w must be 4-byte aligned");
    std::vector<float> y(N);
    SD_CUDA(ctx, cudaMemcpyAsync(y.data(), d_y, sizeof(float) * N, cudaMemcpyDeviceToHost, ctx->stream));
    SD_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    for (int i = 0; i < N; ++i)
        if (y[i] != 1.f && y[i] != -1.f) return sd_fail(ctx, SD_ERR_INVALID, "%s: label %d is %g, not +1 or -1", __func__, i, (double)y[i]);
    return squared_hinge(ctx, d_A, lda, d_y, y, N, D, lambda, max_iterations, d_w, report);
}

}  // extern "C"

namespace {

#define TRAIN_REQUIRE(cond, msg)                                                   \
    do {                                                                           \
        if (!(cond)) return sd_fail(ctx, SD_ERR_INVALID, "%s: %s", fn, msg);       \
    } while (0)

// sd_hog_train_filter's rule (include/sd_b200.h) on the 8-bit grey frames of grey (sd_hog_train_filter), or else on those of
// images with bilinear_orientations (sd_hog_train_filter_images, sd_hog_train_filter_float); fn names the entry point in messages
int train_filter(sd_ctx* ctx, const char* fn, const sd_image_batch* grey, const sd_hog_images* images, int bilinear_orientations,
                 const sd_hog_box* h_boxes, int num_boxes, const double* h_scales, int num_scales, int cell_size, int num_bins, int variant,
                 int filter_w, int filter_h, int pad_x, int pad_y, const sd_hog_train_param* p, float* d_filter, float* h_bias,
                 sd_hog_train_report* h_rounds, sd_hog_window* h_negatives, int* h_num_negatives)
{
    if (const int rc = sd_hog_check_config(ctx, fn, variant, num_bins, cell_size)) return rc;
    if (const int rc = sd_hog_check_filter(ctx, fn, filter_w, filter_h, pad_x, pad_y)) return rc;
    TRAIN_REQUIRE(sd_aligned(d_filter, 4), "the filter must be 4-byte aligned");
    const int F = grey ? grey->count : images->count, S = num_scales;
    TRAIN_REQUIRE(num_scales >= 1 && F >= 1 && num_boxes >= 0, "need at least one scale and one frame");
    for (int s = 0; s < num_scales; ++s)
        TRAIN_REQUIRE(h_scales[s] > 0.0 && h_scales[s] <= 4.0, "every scale must be finite and in (0, 4]");
    TRAIN_REQUIRE(p->lambda > 0.f && std::isfinite(p->lambda), "lambda must be positive and finite");
    TRAIN_REQUIRE(p->positive_overlap >= 0.f && p->positive_overlap <= 1.f && p->negative_overlap >= 0.f && p->negative_overlap <= 1.f &&
                      p->mine_overlap >= 0.f && p->mine_overlap <= 1.f, "overlaps must be in [0, 1]");
    TRAIN_REQUIRE(p->flip_positives == 0 || p->flip_positives == 1, "flip_positives must be 0 or 1");
    TRAIN_REQUIRE(p->rounds >= 0 && p->max_iterations >= 1 && p->max_negatives >= 1, "rounds >= 0, max_iterations >= 1, max_negatives >= 1");
    TRAIN_REQUIRE(p->negatives_per_frame >= 1 && p->negatives_per_frame <= SD_HOG_DETECT_MAX_CANDIDATES,
                  "negatives_per_frame must be in [1, SD_HOG_DETECT_MAX_CANDIDATES]");
    const int dd = sd_hog_dd(num_bins, variant);
    const int D = dd * filter_w * filter_h + 1;
    TRAIN_REQUIRE(D <= SD_HOG_TRAIN_MAX_DIM, "dd * filter_h * filter_w + 1 exceeds SD_HOG_TRAIN_MAX_DIM");

    // the frames, read once, and their level tables
    HogPyramidFrames fr;
    if (const int rc = grey ? sd_hog_read_grey_frames(ctx, fn, grey, &fr) : sd_hog_read_image_frames(ctx, fn, images, bilinear_orientations, &fr))
        return rc;
    const std::vector<sd_hog_image>& frames = fr.frames;
    std::vector<std::vector<Level>> lv(F);
    for (int f = 0; f < F; ++f) {
        if (level_table(frames[f].width, frames[f].height, h_scales, S, cell_size, num_bins, variant, &lv[f]))
            return sd_fail(ctx, SD_ERR_INVALID, "%s: invalid pyramid level", fn);
    }
    std::vector<std::vector<int>> frame_boxes(F);
    for (int b = 0; b < num_boxes; ++b) {
        const sd_hog_box& q = h_boxes[b];
        if (q.frame < 0 || q.frame >= F || q.w < 1 || q.h < 1)
            return sd_fail(ctx, SD_ERR_INVALID, "%s: box %d: frame %d out of [0, %d) or an empty box", fn, b, q.frame, F);
        frame_boxes[q.frame].push_back(b);
    }

    // positives: the window of every box (sd_hog_box_windows), then its mirror
    std::vector<Win> pos;
    std::vector<int> pos_flip;
    int unassigned = 0;
    for (int b = 0; b < num_boxes; ++b) {
        const sd_hog_box& q = h_boxes[b];
        const sd_hog_image& d = frames[q.frame];
        sd_hog_window wv;
        double iou;
        best_window(lv[q.frame], d.width, d.height, cell_size, filter_w, filter_h, pad_x, pad_y, p->positive_overlap,
                    sd_box64{q.x, q.y, (int64_t)q.x + q.w, (int64_t)q.y + q.h}, &wv, &iou);
        if (wv.grid < 0) {
            ++unassigned;
            continue;
        }
        for (int fl = 0; fl <= p->flip_positives; ++fl) {
            pos.push_back({q.frame, wv.grid, wv.x, wv.y});
            pos_flip.push_back(fl);
        }
    }
    const int npos = (int)pos.size();
    TRAIN_REQUIRE(npos >= 1, "no box is covered by a window at positive_overlap: nothing to train on");

    // memory: the rows of the solve, the SVM's compacted copy, the Gram, one slice of pyramid features
    const int64_t ld = ((int64_t)D + 3) / 4 * 4;
    const int64_t nrows = (int64_t)npos + p->max_negatives;
    TRAIN_REQUIRE(nrows <= INT32_MAX / 2, "too many rows");
    const size_t rows_bytes = (size_t)nrows * ld * sizeof(float) + (size_t)nrows * sizeof(float);
    const size_t need = 2 * rows_bytes + (size_t)D * sd_learn_ldg(D, 1) * sizeof(float) + kSliceFloats * sizeof(float) * 2;
    size_t free_b = 0, total_b = 0;
    SD_CUDA(ctx, cudaMemGetInfo(&free_b, &total_b));
    size_t held = 0;
    for (int s = 0; s < SD_WS_COUNT; ++s) held += ctx->ws_bytes[s];
    if (need > free_b + held)
        return sd_fail(ctx, SD_ERR_CUDA, "%s: D = %d with %lld rows needs about %zu MB of device memory, %zu MB available", fn, D,
                       (long long)nrows, need >> 20, (free_b + held) >> 20);

    // slices of frames whose pyramids fit kSliceFloats (at least one frame each)
    std::vector<int> slice0 = {0};
    std::vector<size_t> frame_floats(F, 0);
    for (int f = 0; f < F; ++f)
        for (int s = 0; s < S; ++s) frame_floats[f] += (size_t)dd * lv[f][s].hog_w * lv[f][s].hog_h;
    size_t max_slice = 0;
    {
        size_t acc = 0;
        for (int f = 0; f < F; ++f) {
            if (f > slice0.back() && acc + frame_floats[f] > kSliceFloats) {
                slice0.push_back(f);
                acc = 0;
            }
            acc += frame_floats[f];
            max_slice = std::max(max_slice, acc);
        }
        slice0.push_back(F);
    }
    int max_slice_frames = 0;
    for (size_t i = 0; i + 1 < slice0.size(); ++i) max_slice_frames = std::max(max_slice_frames, slice0[i + 1] - slice0[i]);

    // workspace: [rows (nrows x ld) | labels (nrows)] ; the slice: features, scores, grid / map / offset / window tables, detections
    unsigned char* rws = static_cast<unsigned char*>(sd_workspace(ctx, SD_WS_TRAIN_ROWS, rows_bytes + 64));
    if (!rws) return SD_ERR_CUDA;
    float* d_rows = reinterpret_cast<float*>(rws);
    float* d_lab = d_rows + nrows * ld;
    size_t max_scores = 0;
    for (size_t i = 0; i + 1 < slice0.size(); ++i) {
        size_t sc = 0;
        for (int f = slice0[i]; f < slice0[i + 1]; ++f)
            for (int s = 0; s < S; ++s)
                if (lv[f][s].hog_w) {
                    const int64_t oh = sd_score_extent(lv[f][s].hog_h, pad_y, filter_h), ow = sd_score_extent(lv[f][s].hog_w, pad_x, filter_w);
                    if (oh > 0 && ow > 0) sc += (size_t)(oh * ow);
                }
        max_scores = std::max(max_scores, sc);
    }
    const int max_levels = max_slice_frames * S;
    const int64_t slice_dets = (int64_t)max_slice_frames * p->negatives_per_frame;
    TRAIN_REQUIRE(slice_dets <= INT32_MAX / (int64_t)sizeof(sd_hog_detection), "too many detections per slice: lower negatives_per_frame");
    const int max_win = (int)std::max<int64_t>(npos, std::max<int64_t>(p->max_negatives, slice_dets));
    const size_t feat_b = sd_round16(max_slice * sizeof(float)), score_b = sd_round16(max_scores * sizeof(float) + 4);
    const size_t off_b = sd_round16(sizeof(int64_t) * max_levels), grid_b = sd_round16(sizeof(sd_hog_grid) * max_levels);
    const size_t map_b = sd_round16(sizeof(sd_hog_score_map) * max_levels), win_b = sd_round16(sizeof(sd_hog_window) * max_win);
    const size_t dest_b = sd_round16(sizeof(int) * max_win);
    const size_t det_b = sd_round16(sizeof(sd_hog_detection) * (size_t)slice_dets);
    const size_t cnt_b = sd_round16(sizeof(int32_t) * max_slice_frames), filt_b = sd_round16(sizeof(float) * (D + 1));
    const size_t marg_b = sd_round16(sizeof(double) * p->max_negatives);
    unsigned char* sws = static_cast<unsigned char*>(
        sd_workspace(ctx, SD_WS_TRAIN_SLICE, feat_b + score_b + off_b + grid_b + map_b + win_b + dest_b + det_b + cnt_b + filt_b + marg_b));
    if (!sws) return SD_ERR_CUDA;
    double* d_marg = reinterpret_cast<double*>(sws + feat_b + score_b + off_b + grid_b + map_b + win_b + dest_b + det_b + cnt_b + filt_b);
    float* d_feat = reinterpret_cast<float*>(sws);
    float* d_scores = reinterpret_cast<float*>(sws + feat_b);
    int64_t* d_off = reinterpret_cast<int64_t*>(sws + feat_b + score_b);
    sd_hog_grid* d_grids = reinterpret_cast<sd_hog_grid*>(sws + feat_b + score_b + off_b);
    sd_hog_score_map* d_maps = reinterpret_cast<sd_hog_score_map*>(sws + feat_b + score_b + off_b + grid_b);
    sd_hog_window* d_win = reinterpret_cast<sd_hog_window*>(sws + feat_b + score_b + off_b + grid_b + map_b);
    int* d_dest = reinterpret_cast<int*>(sws + feat_b + score_b + off_b + grid_b + map_b + win_b);
    sd_hog_detection* d_det = reinterpret_cast<sd_hog_detection*>(sws + feat_b + score_b + off_b + grid_b + map_b + win_b + dest_b);
    int32_t* d_cnt = reinterpret_cast<int32_t*>(sws + feat_b + score_b + off_b + grid_b + map_b + win_b + dest_b + det_b);
    float* d_fb = reinterpret_cast<float*>(sws + feat_b + score_b + off_b + grid_b + map_b + win_b + dest_b + det_b + cnt_b);  // F | b

    // CUDA events around each phase of a round (the trainer synchronises after each phase anyway); host phases on the host clock
    struct Events {
        cudaEvent_t a = nullptr, b = nullptr;
        ~Events() { if (a) cudaEventDestroy(a); if (b) cudaEventDestroy(b); }
    } ev;
    SD_CUDA(ctx, cudaEventCreate(&ev.a));
    SD_CUDA(ctx, cudaEventCreate(&ev.b));
    sd_hog_train_report* cur = &h_rounds[0];
    memset(h_rounds, 0, sizeof(sd_hog_train_report) * (size_t)(p->rounds + 1));
    auto timed = [&](float sd_hog_train_report::*field, auto&& fn) -> int {
        SD_CUDA(ctx, cudaEventRecord(ev.a, ctx->stream));
        const int rc = fn();
        if (rc) return rc;
        SD_CUDA(ctx, cudaEventRecord(ev.b, ctx->stream));
        SD_CUDA(ctx, cudaEventSynchronize(ev.b));
        float ms = 0.f;
        SD_CUDA(ctx, cudaEventElapsedTime(&ms, ev.a, ev.b));
        cur->*field += ms;
        return SD_OK;
    };

    // one slice resident: its pyramid, and per (frame, level) its grid index in the slice's table (-1: empty level)
    std::vector<int> grid_of;
    std::vector<sd_hog_grid> grids;
    auto load_slice = [&](int f0, int f1) -> int {
        std::vector<int64_t> off((size_t)(f1 - f0) * S, 0);
        grid_of.assign((size_t)(f1 - f0) * S, -1);
        grids.clear();
        int64_t acc = 0;
        for (int f = f0; f < f1; ++f)
            for (int s = 0; s < S; ++s) {
                const Level& l = lv[f][s];
                if (!l.hog_w) continue;
                off[(size_t)(f - f0) * S + s] = acc;
                grid_of[(size_t)(f - f0) * S + s] = (int)grids.size();
                grids.push_back(sd_hog_grid{l.hog_w, l.hog_h, acc, 0});
                acc += (int64_t)dd * l.hog_w * l.hog_h;
            }
        if (grids.empty()) return SD_OK;
        SD_CUDA(ctx, cudaMemcpyAsync(d_off, off.data(), sizeof(int64_t) * off.size(), cudaMemcpyHostToDevice, ctx->stream));
        return timed(&sd_hog_train_report::pyramid_ms, [&] {
            return sd_hog_pyramid_frames(ctx, fn, fr, f0, f1, h_scales, S, cell_size, num_bins, variant, d_feat, d_off);
        });
    };
    // gather windows (frame, level, x, y, flip) of the resident slice into rows dest[i] of d_rows
    auto gather = [&](int f0, const std::vector<sd_hog_window>& w, const std::vector<int>& dest) -> int {
        if (w.empty()) return SD_OK;
        std::vector<sd_hog_window> local(w);
        for (auto& v : local) v.grid = grid_of[(size_t)(v.grid / S - f0) * S + v.grid % S];
        SD_CUDA(ctx, cudaMemcpyAsync(d_grids, grids.data(), sizeof(sd_hog_grid) * grids.size(), cudaMemcpyHostToDevice, ctx->stream));
        SD_CUDA(ctx, cudaMemcpyAsync(d_win, local.data(), sizeof(sd_hog_window) * local.size(), cudaMemcpyHostToDevice, ctx->stream));
        SD_CUDA(ctx, cudaMemcpyAsync(d_dest, dest.data(), sizeof(int) * dest.size(), cudaMemcpyHostToDevice, ctx->stream));
        const int rc = timed(&sd_hog_train_report::gather_ms, [&] {
            return launch_windows(ctx, d_feat, d_grids, 0, 0, num_bins, variant, filter_w, filter_h, pad_x, pad_y, d_win, d_dest,
                                  (int)local.size(), d_rows, ld);
        });
        if (rc) return rc;
        cur->gathered_bytes += 2.0 * (double)local.size() * D * sizeof(float);
        return sd_check_cuda(ctx, cudaStreamSynchronize(ctx->stream), "gather");   // the host tables are reused
    };

    // the positive rows, in box order (each row followed by its mirror), and their labels
    for (size_t i = 0; i + 1 < slice0.size(); ++i) {
        const int f0 = slice0[i], f1 = slice0[i + 1];
        std::vector<sd_hog_window> w;
        std::vector<int> dest;
        for (int r = 0; r < npos; ++r)
            if (pos[r].frame >= f0 && pos[r].frame < f1) {
                w.push_back({pos[r].frame * S + pos[r].level, pos[r].x, pos[r].y, pos_flip[r]});
                dest.push_back(r);
            }
        if (w.empty()) continue;
        int rc = load_slice(f0, f1);
        if (!rc) rc = gather(f0, w, dest);
        if (rc) return rc;
    }
    std::vector<float> lab(nrows, -1.f);
    std::fill(lab.begin(), lab.begin() + npos, 1.f);
    SD_CUDA(ctx, cudaMemcpyAsync(d_lab, lab.data(), sizeof(float) * nrows, cudaMemcpyHostToDevice, ctx->stream));

    // round 0's filter: the mean of the unflipped positive rows minus its own scalar mean, in float64 rounded to float
    std::vector<float> hpos((size_t)npos * ld);
    SD_CUDA(ctx, cudaMemcpyAsync(hpos.data(), d_rows, sizeof(float) * hpos.size(), cudaMemcpyDeviceToHost, ctx->stream));
    SD_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    std::vector<float> fb(D + 1, 0.f);               // the current filter (D - 1 weights) and bias, then one spare
    {
        std::vector<double> sum(D - 1, 0.0);
        int n = 0;
        for (int r = 0; r < npos; ++r) {
            if (pos_flip[r]) continue;
            ++n;
            for (int j = 0; j < D - 1; ++j) sum[j] += hpos[(size_t)r * ld + j];
        }
        double total = 0.0;
        for (int j = 0; j < D - 1; ++j) {
            fb[j] = (float)(sum[j] / n);
            total += fb[j];
        }
        const float m = (float)(total / (D - 1));
        for (int j = 0; j < D - 1; ++j) fb[j] = fb[j] - m;
        fb[D - 1] = 0.f;
    }

    std::vector<Win> cache;                          // slot order
    std::set<Win> cached;
    float* d_w = d_fb;                               // the SVM writes [filter | bias] here
    std::vector<double> margins;
    for (int round = 0; round <= p->rounds; ++round) {
        sd_hog_train_report& rep = h_rounds[round];
        cur = &rep;
        rep.positives = npos;
        rep.unassigned = unassigned;
        SD_CUDA(ctx, cudaMemcpyAsync(d_fb, fb.data(), sizeof(float) * D, cudaMemcpyHostToDevice, ctx->stream));
        // inactive cached negatives under the current filter (margin >= 1): the slots that new windows may take, in cache order
        std::vector<int> free_slots;
        if (!cache.empty()) {
            if (const int rc = svm_margins(ctx, d_rows + (int64_t)npos * ld, ld, (int)cache.size(), D, d_fb, d_marg, margins)) return rc;
            for (size_t k = 0; k < cache.size(); ++k)
                if (-margins[k] >= 1.0) free_slots.push_back(npos + (int)k);
        }
        size_t next_free = 0;
        const float threshold = round == 0 ? -FLT_MAX : -1.f;
        for (size_t i = 0; i + 1 < slice0.size(); ++i) {
            const int f0 = slice0[i], f1 = slice0[i + 1], nf = f1 - f0;
            int rc = load_slice(f0, f1);
            if (rc) return rc;
            if (grids.empty()) continue;
            // scores of the filter on every non-empty level, and their score maps
            std::vector<sd_hog_grid> g(grids);
            std::vector<sd_hog_score_map> maps;
            int64_t acc = 0;
            for (int f = f0; f < f1; ++f)
                for (int s = 0; s < S; ++s) {
                    const int gi = grid_of[(size_t)(f - f0) * S + s];
                    if (gi < 0) continue;
                    const int oh = std::max(0, sd_score_extent(lv[f][s].hog_h, pad_y, filter_h)),
                              ow = std::max(0, sd_score_extent(lv[f][s].hog_w, pad_x, filter_w));
                    g[gi].out_offset = acc;
                    maps.push_back(sd_hog_score_map{f - f0, s, frames[f].width, frames[f].height, lv[f][s].level_w, lv[f][s].level_h, ow, oh, acc});
                    acc += (int64_t)oh * ow;
                }
            SD_CUDA(ctx, cudaMemcpyAsync(d_grids, g.data(), sizeof(sd_hog_grid) * g.size(), cudaMemcpyHostToDevice, ctx->stream));
            SD_CUDA(ctx, cudaMemcpyAsync(d_maps, maps.data(), sizeof(sd_hog_score_map) * maps.size(), cudaMemcpyHostToDevice, ctx->stream));
            sd_hog_grids gs = {d_feat, (int32_t)g.size(), 0, 0, d_grids};
            if ((rc = timed(&sd_hog_train_report::scores_ms, [&] {
                     return sd_hog_correlate(ctx, &gs, num_bins, variant, d_fb, 1, filter_w, filter_h, d_fb + (D - 1), pad_x, pad_y, d_scores);
                 })))
                return rc;
            if ((rc = timed(&sd_hog_train_report::detect_ms, [&] {
                     return sd_hog_detections(ctx, d_scores, d_maps, (int)maps.size(), nf, 1, cell_size, filter_w, filter_h, pad_x, pad_y,
                                              threshold, p->mine_overlap, SD_HOG_DETECT_MAX_CANDIDATES, p->negatives_per_frame, d_det,
                                              d_cnt, nullptr);
                 })))
                return rc;
            const auto host0 = std::chrono::steady_clock::now();
            std::vector<sd_hog_detection> det((size_t)nf * p->negatives_per_frame);
            std::vector<int32_t> cnt(nf);
            SD_CUDA(ctx, cudaMemcpyAsync(det.data(), d_det, sizeof(sd_hog_detection) * det.size(), cudaMemcpyDeviceToHost, ctx->stream));
            SD_CUDA(ctx, cudaMemcpyAsync(cnt.data(), d_cnt, sizeof(int32_t) * nf, cudaMemcpyDeviceToHost, ctx->stream));
            SD_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
            // the slice's new negatives, in (frame, rule order) order
            std::vector<sd_hog_window> w;
            std::vector<int> dest;
            for (int f = f0; f < f1; ++f)
                for (int k = 0; k < cnt[f - f0]; ++k) {
                    const sd_hog_detection& d = det[(size_t)(f - f0) * p->negatives_per_frame + k];
                    const sd_box64 db = {d.x, d.y, (int64_t)d.x + d.w, (int64_t)d.y + d.h};
                    bool near_box = false;
                    for (int b : frame_boxes[f]) {
                        const sd_hog_box& q = h_boxes[b];
                        int64_t in, un;
                        inter_union(db, sd_box64{q.x, q.y, (int64_t)q.x + q.w, (int64_t)q.y + q.h}, &in, &un);
                        if ((double)in > (double)p->negative_overlap * (double)un) near_box = true;
                    }
                    if (near_box) {
                        ++rep.excluded;
                        continue;
                    }
                    ++rep.mined;
                    const Win v = {f, d.level, d.cell_x, d.cell_y};
                    if (cached.count(v)) continue;
                    ++rep.added;
                    int slot;
                    if ((int)cache.size() < p->max_negatives) {
                        slot = npos + (int)cache.size();
                        cache.push_back(v);
                    } else if (next_free < free_slots.size()) {
                        slot = free_slots[next_free++];
                        cached.erase(cache[slot - npos]);
                        cache[slot - npos] = v;
                        ++rep.evicted;
                    } else {
                        --rep.added;
                        ++rep.truncated;
                        continue;
                    }
                    cached.insert(v);
                    w.push_back({f * S + d.level, d.cell_x, d.cell_y, 0});
                    dest.push_back(slot);
                }
            rep.host_ms += std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - host0).count();
            if ((rc = gather(f0, w, dest))) return rc;
        }
        rep.cache = (int)cache.size();
        if (round > 0 && rep.added == 0) break;      // nothing new: the last solve stands
        const int N = npos + (int)cache.size();
        std::vector<float> y(lab.begin(), lab.begin() + N);
        const auto solve0 = std::chrono::steady_clock::now();
        if (const int rc = squared_hinge(ctx, d_rows, ld, d_lab, y, N, D, p->lambda, p->max_iterations, d_w, &rep.solve)) return rc;
        rep.solve_ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - solve0).count();   // ends synchronised
        rep.solved = 1;
        SD_CUDA(ctx, cudaMemcpyAsync(fb.data(), d_w, sizeof(float) * D, cudaMemcpyDeviceToHost, ctx->stream));
        SD_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    SD_CUDA(ctx, cudaMemcpyAsync(d_filter, fb.data(), sizeof(float) * (D - 1), cudaMemcpyHostToDevice, ctx->stream));
    SD_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    *h_bias = fb[D - 1];
    *h_num_negatives = (int)cache.size();
    if (h_negatives)
        for (size_t k = 0; k < cache.size(); ++k) h_negatives[k] = {cache[k].frame * S + cache[k].level, cache[k].x, cache[k].y, 0};
    return SD_OK;
}

#undef TRAIN_REQUIRE

}  // namespace

extern "C" {

int sd_hog_train_filter(sd_ctx* ctx, const sd_image_batch* images, const sd_hog_box* h_boxes, int num_boxes, const double* h_scales,
                        int num_scales, int cell_size, int num_bins, int variant, int filter_w, int filter_h, int pad_x, int pad_y,
                        const sd_hog_train_param* p, float* d_filter, float* h_bias, sd_hog_train_report* h_rounds,
                        sd_hog_window* h_negatives, int* h_num_negatives)
{
    if (!ctx) return SD_ERR_INVALID;
    SD_REQUIRE(ctx, images && h_scales && p && d_filter && h_bias && h_rounds && h_num_negatives && (num_boxes == 0 || h_boxes),
               "null argument");
    SD_REQUIRE(ctx, !images->d_roi, "a batch with regions of interest has no whole frames");
    SD_REQUIRE(ctx, images->count < 1 || images->d_data, "null argument");
    return train_filter(ctx, __func__, images, nullptr, 0, h_boxes, num_boxes, h_scales, num_scales, cell_size, num_bins, variant,
                        filter_w, filter_h, pad_x, pad_y, p, d_filter, h_bias, h_rounds, h_negatives, h_num_negatives);
}

int sd_hog_train_filter_images(sd_ctx* ctx, const sd_hog_images* images, int bilinear_orientations, const sd_hog_box* h_boxes,
                               int num_boxes, const double* h_scales, int num_scales, int cell_size, int num_bins, int variant,
                               int filter_w, int filter_h, int pad_x, int pad_y, const sd_hog_train_param* p, float* d_filter,
                               float* h_bias, sd_hog_train_report* h_rounds, sd_hog_window* h_negatives, int* h_num_negatives)
{
    if (!ctx) return SD_ERR_INVALID;
    SD_REQUIRE(ctx, images && h_scales && p && d_filter && h_bias && h_rounds && h_num_negatives && (num_boxes == 0 || h_boxes),
               "null argument");
    SD_REQUIRE(ctx, images->dtype == SD_HOG_U8, "dtype must be SD_HOG_U8: the levels are resized by the 8-bit rule");
    SD_REQUIRE(ctx, images->channels >= 1 && images->channels <= 16, "channels must be in [1,16]");
    SD_REQUIRE(ctx, bilinear_orientations == 0 || bilinear_orientations == 1, "bilinear_orientations must be 0 or 1");
    SD_REQUIRE(ctx, images->count < 1 || images->d_data, "null argument");
    return train_filter(ctx, __func__, nullptr, images, bilinear_orientations, h_boxes, num_boxes, h_scales, num_scales, cell_size,
                        num_bins, variant, filter_w, filter_h, pad_x, pad_y, p, d_filter, h_bias, h_rounds, h_negatives,
                        h_num_negatives);
}

int sd_hog_train_filter_float(sd_ctx* ctx, const sd_hog_images* images, int bilinear_orientations, const sd_hog_box* h_boxes,
                              int num_boxes, const double* h_scales, int num_scales, int cell_size, int num_bins, int variant,
                              int filter_w, int filter_h, int pad_x, int pad_y, const sd_hog_train_param* p, float* d_filter,
                              float* h_bias, sd_hog_train_report* h_rounds, sd_hog_window* h_negatives, int* h_num_negatives)
{
    if (!ctx) return SD_ERR_INVALID;
    SD_REQUIRE(ctx, images && h_scales && p && d_filter && h_bias && h_rounds && h_num_negatives && (num_boxes == 0 || h_boxes),
               "null argument");
    SD_REQUIRE(ctx, images->dtype == SD_HOG_F32, "dtype must be SD_HOG_F32: the levels are resized by the float rule");
    SD_REQUIRE(ctx, (reinterpret_cast<uintptr_t>(images->d_data) & 3) == 0, "float frames must be 4-byte aligned");
    SD_REQUIRE(ctx, images->channels >= 1 && images->channels <= 16, "channels must be in [1,16]");
    SD_REQUIRE(ctx, bilinear_orientations == 0 || bilinear_orientations == 1, "bilinear_orientations must be 0 or 1");
    SD_REQUIRE(ctx, images->count < 1 || images->d_data, "null argument");
    return train_filter(ctx, __func__, nullptr, images, bilinear_orientations, h_boxes, num_boxes, h_scales, num_scales, cell_size,
                        num_bins, variant, filter_w, filter_h, pad_x, pad_y, p, d_filter, h_bias, h_rounds, h_negatives,
                        h_num_negatives);
}

}  // extern "C"
