// HOG filters (sd_hog_correlate): a bank of Q templates of fw x fh cells correlated with every grid of a batch of planar HOG
// features, the score maps of a sliding-window detector (DPM root filters, exemplar SVMs, a linear template of HOG windows).
//
// One CTA per tile of kTileW x kTileH output positions of one grid, for a group of QF filters (blockIdx.y).  Channel chunk by
// channel chunk it stages in shared memory the zero-padded map window its tile reads, (kTileH + fh - 1) x (kTileW + fw - 1)
// cells of each channel, and the group's filter values [c][dy][dx][QF]; each thread keeps a register tile of kRun
// consecutive positions of one output row x QF filters.  Per (channel, dy) a thread holds a window of kRun map values and
// slides it along dx, so each staged map value is read once per dx run rather than once per position.  Every score is one
// float32 FMA chain from 0 over (channel, dy, dx) in ascending order, the bias added last, whatever the chunk, tile, group
// or batch: the result depends on the grid, the filter and the bias alone.
//
// Grids of different sizes are one launch: the descriptor table is read back once, a host prefix sum gives each grid's first
// CTA, and a CTA finds its grid by binary search over those.
#include "sd_internal.cuh"

#include <algorithm>
#include <climits>
#include <cstring>
#include <vector>

namespace {

constexpr int kThreads = 128;
constexpr int kRun = 4;                          // consecutive output positions of a thread
constexpr int kColumns = 8;                      // threads per output row of the tile
constexpr int kTileW = kColumns * kRun;          // 32 positions
constexpr int kTileH = kThreads / kColumns;      // 16 rows
constexpr int kSmemBudget = 24 * 1024;           // staged channels per chunk: as many as fit (one at least)

struct CorrArgs {
    const float* maps;
    const sd_hog_grid* grids;    // per-grid descriptors, or null: equally sized grids
    const int* tile0;            // per grid: its first CTA (grids only)
    int count;
    int width, height;           // equally sized grids
    long long in_stride, out_stride;
    int tiles_x, tiles;          // equally sized grids: CTAs per row of tiles, per grid
    const float* filters;        // [Q][dd][fh][fw]
    const float* bias;           // Q floats or null
    int Q, fw, fh, pad_x, pad_y, dd;
    int chunk;                   // channels staged at once
    int pitch;                   // floats per staged map row: odd, so that a warp's 8 x 4 runs hit 32 different banks
    int map_floats;              // staged map floats per chunk, rounded up to 4 (the filter values follow, 16-byte aligned)
    float* scores;
};

__host__ __device__ inline int corr_pitch(int fw) { return (kTileW + fw - 1) | 1; }

// shared floats of one staged channel: its map window and a group's filter values
__host__ __device__ inline int corr_channel_floats(int fw, int fh, int QF) { return (kTileH + fh - 1) * corr_pitch(fw) + fh * fw * QF; }

template <int QF>
__device__ __forceinline__ void load_filters(const float* p, float (&f)[QF])
{
    if constexpr (QF % 4 == 0) {
#pragma unroll
        for (int q = 0; q < QF; q += 4) {
            const float4 v = *reinterpret_cast<const float4*>(p + q);
            f[q] = v.x; f[q + 1] = v.y; f[q + 2] = v.z; f[q + 3] = v.w;
        }
    } else if constexpr (QF == 2) {
        const float2 v = *reinterpret_cast<const float2*>(p);
        f[0] = v.x; f[1] = v.y;
    } else {
        f[0] = *p;
    }
}

template <int QF>
__global__ void __launch_bounds__(kThreads, 4) hog_correlate_kernel(const __grid_constant__ CorrArgs a)
{
    extern __shared__ __align__(16) float smem[];
    const int tid = threadIdx.x;
    const int b = blockIdx.x;

    // the CTA's grid and tile
    int W, H, t, tiles_x;
    const float* __restrict__ M;
    float* __restrict__ out;
    const int fw = a.fw, fh = a.fh;
    if (a.grids) {
        const int g = sd_find_last_le(0, a.count - 1, b, [&](int i) { return a.tile0[i]; });   // the grid of CTA b
        const sd_hog_grid d = a.grids[g];
        W = d.width; H = d.height;
        M = a.maps + d.offset;
        out = a.scores + d.out_offset;
        tiles_x = (sd_score_extent(W, a.pad_x, fw) + kTileW - 1) / kTileW;
        t = b - a.tile0[g];
    } else {
        const int g = b / a.tiles;
        W = a.width; H = a.height;
        M = a.maps + (long long)g * a.in_stride;
        out = a.scores + (long long)g * a.out_stride;
        tiles_x = a.tiles_x;
        t = b - g * a.tiles;
    }
    const int oh = sd_score_extent(H, a.pad_y, fh), ow = sd_score_extent(W, a.pad_x, fw);
    const int tr = t / tiles_x;
    const int x0 = (t - tr * tiles_x) * kTileW, y0 = tr * kTileH;
    const int q0 = blockIdx.y * QF;
    const int sw = kTileW + fw - 1, sh = kTileH + fh - 1, pitch = a.pitch;
    const int gx0 = x0 - a.pad_x, gy0 = y0 - a.pad_y;          // grid cell of staged (0, 0)
    const long long plane = (long long)W * H;
    float* s_map = smem;                                          // [chunk][sh][pitch]
    float* s_f = smem + a.map_floats;                             // [chunk][fh][fw][QF]
    const int tx = tid % kColumns, ty = tid / kColumns;

    float acc[QF][kRun];
#pragma unroll
    for (int q = 0; q < QF; ++q)
#pragma unroll
        for (int p = 0; p < kRun; ++p) acc[q][p] = 0.f;

    for (int c0 = 0; c0 < a.dd; c0 += a.chunk) {
        const int nc = min(a.chunk, a.dd - c0);
        __syncthreads();                                          // the previous chunk is consumed
        // one warp per staged row, its lanes along the row: no index division per element
        const int warp = tid >> 5, lane = tid & 31;
        for (int row = warp; row < nc * sh; row += kThreads / 32) {
            const int c = row / sh, r = row - c * sh;
            const int gy = gy0 + r;
            const float* src = M + (c0 + c) * plane + (long long)gy * W;
            float* dst = s_map + (c * sh + r) * pitch;
            const bool in_rows = (unsigned)gy < (unsigned)H;
            for (int col = lane; col < sw; col += 32) {
                const int gx = gx0 + col;
                dst[col] = in_rows && (unsigned)gx < (unsigned)W ? __ldg(src + gx) : 0.f;   // M is 0 outside the grid
            }
        }
        const int taps = fh * fw;
        for (int i = tid; i < nc * taps * QF; i += kThreads) {
            const int q = i % QF, k = i / QF;                     // k = c * taps + dy * fw + dx
            const int c = k / taps, tap = k - c * taps;
            float v = 0.f;                                        // filters past Q score nothing and are not stored
            if (q0 + q < a.Q) v = __ldg(a.filters + ((long long)(q0 + q) * a.dd + c0 + c) * taps + tap);
            s_f[i] = v;
        }
        __syncthreads();

        for (int c = 0; c < nc; ++c) {
            for (int dy = 0; dy < fh; ++dy) {
                const float* mrow = s_map + (c * sh + ty + dy) * pitch + tx * kRun;
                const float* frow = s_f + (c * fh + dy) * fw * QF;
                float m[kRun];
#pragma unroll
                for (int p = 0; p < kRun; ++p) m[p] = mrow[p];
                for (int dx = 0; dx < fw; ++dx) {
                    float f[QF];
                    load_filters<QF>(frow + dx * QF, f);
#pragma unroll
                    for (int q = 0; q < QF; ++q)
#pragma unroll
                        for (int p = 0; p < kRun; ++p) acc[q][p] = __fmaf_rn(f[q], m[p], acc[q][p]);
                    if (dx + 1 < fw) {
#pragma unroll
                        for (int p = 0; p + 1 < kRun; ++p) m[p] = m[p + 1];
                        m[kRun - 1] = mrow[kRun + dx];
                    }
                }
            }
        }
    }

    const int y = y0 + ty;
    if (y >= oh) return;
#pragma unroll
    for (int q = 0; q < QF; ++q) {
        if (q0 + q >= a.Q) break;
        const float bq = a.bias ? __ldg(a.bias + q0 + q) : 0.f;
        float* o = out + ((long long)(q0 + q) * oh + y) * ow;
#pragma unroll
        for (int p = 0; p < kRun; ++p) {
            const int x = x0 + tx * kRun + p;
            if (x < ow) o[x] = a.bias ? __fadd_rn(acc[q][p], bq) : acc[q][p];
        }
    }
}

typedef void (*CorrKernel)(CorrArgs);

// filters per CTA: the smallest of 1, 2, 4, 8 that holds the bank, 8 for larger banks
int group_of(int Q) { return Q <= 1 ? 1 : Q <= 2 ? 2 : Q <= 4 ? 4 : 8; }

CorrKernel corr_kernel(int QF)
{
    return QF == 1 ? hog_correlate_kernel<1> : QF == 2 ? hog_correlate_kernel<2> : QF == 4 ? hog_correlate_kernel<4> : hog_correlate_kernel<8>;
}

}  // namespace

extern "C" {

int sd_hog_correlate(sd_ctx* ctx, const sd_hog_grids* maps, int num_bins, int variant, const float* d_filters, int num_filters,
                     int filter_w, int filter_h, const float* d_bias, int pad_x, int pad_y, float* d_scores)
{
    if (!ctx) return SD_ERR_INVALID;
    SD_REQUIRE(ctx, maps && d_filters && d_scores, "null argument");
    if (const int rc = sd_hog_check_config(ctx, __func__, variant, num_bins)) return rc;
    SD_REQUIRE(ctx, num_filters >= 1 && num_filters <= SD_HOG_FILTER_MAX_BANK, "num_filters must be in [1, SD_HOG_FILTER_MAX_BANK]");
    if (const int rc = sd_hog_check_filter(ctx, __func__, filter_w, filter_h, pad_x, pad_y)) return rc;
    SD_REQUIRE(ctx, sd_aligned(d_filters, 4) && sd_aligned(d_scores, 4) && sd_aligned(d_bias, 4),
               "filters, bias and scores must be 4-byte aligned");
    SD_REQUIRE(ctx, maps->count >= 0, "negative grid count");
    const int count = maps->count;
    if (count == 0) return SD_OK;
    SD_REQUIRE(ctx, maps->d_features && sd_aligned(maps->d_features, 4), "maps must be non-null and 4-byte aligned");

    int max_w = 0, max_h = 0;
    std::vector<sd_hog_grid> table;
    if (const int rc = sd_read_hog_grids(ctx, __func__, maps, &max_w, &max_h, &table)) return rc;
    return sd_hog_correlate_table(ctx, maps, table.data(), max_w, max_h, num_bins, variant, d_filters, num_filters, filter_w, filter_h,
                                  d_bias, pad_x, pad_y, d_scores);
}

}  // extern "C"

int sd_hog_correlate_table(sd_ctx* ctx, const sd_hog_grids* maps, const sd_hog_grid* table, int max_w, int max_h, int num_bins,
                           int variant, const float* d_filters, int num_filters, int filter_w, int filter_h, const float* d_bias,
                           int pad_x, int pad_y, float* d_scores)
{
    const int count = maps->count;
    const int dd = sd_hog_dd(num_bins, variant);
    const int QF = group_of(num_filters);

    CorrArgs a;
    memset(&a, 0, sizeof(a));
    a.maps = maps->d_features;
    a.grids = maps->d_grids;
    a.count = count;
    a.filters = d_filters;
    a.bias = d_bias;
    a.Q = num_filters; a.fw = filter_w; a.fh = filter_h; a.pad_x = pad_x; a.pad_y = pad_y; a.dd = dd;
    a.scores = d_scores;
    a.pitch = corr_pitch(filter_w);
    const int per_channel = corr_channel_floats(filter_w, filter_h, QF);
    a.chunk = std::max(1, std::min(dd, (int)(kSmemBudget / sizeof(float)) / per_channel));
    a.map_floats = (a.chunk * (kTileH + filter_h - 1) * a.pitch + 3) / 4 * 4;
    const int smem = (a.map_floats + a.chunk * filter_h * filter_w * QF) * (int)sizeof(float);

    long long total = 0;                             // CTAs per filter group
    if (maps->d_grids) {
        std::vector<int> tile0(count);
        for (int i = 0; i < count; ++i) {
            tile0[i] = (int)total;
            const int oh = sd_score_extent(table[i].height, pad_y, filter_h), ow = sd_score_extent(table[i].width, pad_x, filter_w);
            if (oh > 0 && ow > 0) total += (long long)sd_div_up(ow, kTileW) * sd_div_up(oh, kTileH);
            if (total > INT_MAX) return sd_fail(ctx, SD_ERR_INVALID, "sd_hog_correlate: too many score tiles");
        }
        if (total == 0) return SD_OK;
        int* d_tile0 = static_cast<int*>(sd_workspace(ctx, SD_WS_FILTERS, sizeof(int) * count));
        if (!d_tile0) return SD_ERR_CUDA;
        SD_CUDA(ctx, cudaMemcpyAsync(d_tile0, tile0.data(), sizeof(int) * count, cudaMemcpyHostToDevice, ctx->stream));
        a.tile0 = d_tile0;
    } else {
        const int oh = sd_score_extent(max_h, pad_y, filter_h), ow = sd_score_extent(max_w, pad_x, filter_w);
        if (oh <= 0 || ow <= 0) return SD_OK;
        a.width = max_w; a.height = max_h;
        a.in_stride = (long long)dd * max_w * max_h;
        a.out_stride = (long long)num_filters * oh * ow;
        a.tiles_x = sd_div_up(ow, kTileW);
        a.tiles = a.tiles_x * sd_div_up(oh, kTileH);
        total = (long long)a.tiles * count;
        if (total > INT_MAX) return sd_fail(ctx, SD_ERR_INVALID, "sd_hog_correlate: too many score tiles");
    }

    const CorrKernel kern = corr_kernel(QF);
    SD_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    kern<<<dim3((unsigned)total, (unsigned)sd_div_up(num_filters, QF)), kThreads, smem, ctx->stream>>>(a);
    SD_LAUNCH_CHECK(ctx, "hog_correlate_kernel");
    return SD_OK;
}
