// The rest of VLFeat's HOG object API on planar features [dd][h][w] (x fastest), batched over grids of cells:
//   sd_hog_render      vl_hog_render (reference include/rcr/hog.c:428-495): one 21 x 21 glyph tile per cell
//   sd_hog_relayout    left-right flip by vl_hog_get_permutation (hog.c:225-268, :371-380) and / or a transpose of every plane
//   sd_hog_permutation, sd_hog_glyphs   the host tables of vl_hog_new (hog.c:225-312)
// Both kernels are pure reads and writes: no reduction crosses a thread, so every result is the same in any batch and run.
#include "sd_internal.cuh"

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>
#include <vector>

namespace {

constexpr int kGlyph = SD_HOG_GLYPH_SIZE;
constexpr int kGlyphPixels = kGlyph * kGlyph;
constexpr int kRenderThreads = 256;
constexpr int kRenderCells = 12;                  // cells of one cell row per CTA: 12 * 21 = 252 image columns, one per thread
constexpr int kTile = 32;                         // relayout: 32 x 32 elements per CTA, 32 x 8 threads

// ---- host tables ------------------------------------------------------------------------------------------------------------

// vl_hog_new's permutation (hog.c:225-268): flipped[i] = features[perm[i]].  Orientation o (pointing at angle o pi / K) maps to
// K - o, the mirror image about the vertical axis; the directed half adds K modulo 2K; the undirected and Dalal-Triggs blocks
// fold modulo K.  The four blocks around a cell (x offset bx, y offset by, index bx + 2 by) swap left and right.
void permutation(int K, int variant, int64_t* perm)
{
    auto mirrored_block = [](int q) { return (1 - q % 2) + (q / 2) * 2; };
    if (variant == 1) {
        for (int o = 0; o < K; ++o) {
            const int m = K - o;
            perm[o] = m;
            perm[K + o] = (m + K) % (2 * K);
            perm[2 * K + o] = 2 * K + m % K;
        }
        for (int q = 0; q < 4; ++q) perm[3 * K + q] = 3 * K + mirrored_block(q);
    } else {
        for (int q = 0; q < 4; ++q)
            for (int o = 0; o < K; ++o) perm[q * K + o] = (K - o) % K + mirrored_block(q) * K;
    }
}

// vl_hog_new's glyphs (hog.c:276-312): glyph o is a bar orthogonal to orientation o through the tile's centre, one pixel per
// column (a bar within 45 degrees of horizontal) or per row, rounded with lround.  The arithmetic follows hog.c step by step in
// double, so each pixel lands where hog.c puts it.  Element (x, y) of glyph o is glyphs[o * 441 + y * 21 + x]; transposed
// tables store (x, y) at (y, x).
void glyphs(int K, bool transposed, float* g)
{
    const double pi = 3.141592653589793;
    const double size = kGlyph;
    std::memset(g, 0, sizeof(float) * kGlyphPixels * K);
    for (int o = 0; o < K; ++o) {
        float* t = g + o * kGlyphPixels;
        auto set = [&](long x, long y) { t[transposed ? x * kGlyph + y : y * kGlyph + x] = 1.f; };
        const double angle = std::fmod((double)o * pi / (double)K + pi / 2, pi);
        const double x2 = size * std::cos(angle) / 2, y2 = size * std::sin(angle) / 2;
        const bool along_x = angle <= pi / 4 || angle >= pi * 3 / 4;
        const double slope = along_x ? y2 / x2 : x2 / y2;
        const double offset = (1 - slope) * (size - 1) / 2;
        const long skip = (long)((1 - (along_x ? std::fabs(std::cos(angle)) : std::sin(angle))) / 2 * size);   // truncates
        for (long i = skip; i < kGlyph - skip; ++i) {
            const long j = std::lround(slope * (double)i + offset);
            if (along_x) set(i, j);
            else set(j, i);
        }
    }
}

// ---- render ---------------------------------------------------------------------------------------------------------------

struct RenderArgs {
    const float* features;
    float* image;
    int width, height;                    // equally sized grids (grids == nullptr), packed: grid i at i * dd * h * w floats,
    long long in_stride, out_stride;      // its image at i * h * w * 441 floats
    const sd_hog_grid* grids;
    int frame0;
    int K, terms;                         // terms: 3 (UoCTTI) or 4 (Dalal-Triggs) planes summed per orientation
    int tiles_x;                          // CTAs per cell row of the widest grid
    uint16_t mask[kGlyphPixels];          // bit k of mask[y * 21 + x]: glyph k is 1 at (x, y); every glyph value is 0 or 1
};

// One CTA per run of kRenderCells cells of one cell row of one grid; thread t owns image column t of the run (cell t / 21,
// glyph column t % 21) and walks its 21 rows.  Per cell (hog.c:443-490): weight k = d[k] + d[k + K] + d[k + 2K] (+ d[k + 3K]),
// left to right in float; min and max weight start at 0 and are updated by hog.c's VL_MIN / VL_MAX comparisons; every
// pixel is v += weight_k * glyph_k, k ascending, each product and sum rounded to float (no FMA), then clamped as
// VL_MAX(min, VL_MIN(max, v)).  A NaN pixel or weight therefore propagates exactly as in hog.c.
__global__ void __launch_bounds__(kRenderThreads) hog_render_kernel(const __grid_constant__ RenderArgs a)
{
    __shared__ uint16_t s_mask[kGlyphPixels];
    __shared__ float s_w[kRenderCells][SD_MAX_BINS];
    const int tid = threadIdx.x;
    const int g = a.frame0 + blockIdx.z;
    int W = a.width, H = a.height;
    const float* in;
    float* img;
    if (a.grids) {
        const sd_hog_grid d = a.grids[g];
        W = d.width; H = d.height;
        in = a.features + d.offset;
        img = a.image + d.out_offset;
    } else {
        in = a.features + (long long)g * a.in_stride;
        img = a.image + (long long)g * a.out_stride;
    }
    const int cy = blockIdx.x / a.tiles_x, cx0 = (blockIdx.x - cy * a.tiles_x) * kRenderCells;
    if (cy >= H || cx0 >= W) return;                 // the launch covers the largest grid of the batch
    const int nc = min(kRenderCells, W - cx0);
    const int K = a.K;
    const long long plane = (long long)W * H;

    for (int i = tid; i < kGlyphPixels; i += kRenderThreads) s_mask[i] = a.mask[i];
    if (tid < nc * K) {
        const int c = tid / K, k = tid - c * K;
        const float* p = in + (long long)cy * W + cx0 + c + (long long)k * plane;
        float w = p[0];
        for (int t = 1; t < a.terms; ++t) w = __fadd_rn(w, p[(long long)t * K * plane]);
        s_w[c][k] = w;
    }
    __syncthreads();

    const int cols = nc * kGlyph;
    if (tid >= cols) return;
    const int c = tid / kGlyph, gx = tid - c * kGlyph;
    float w[SD_MAX_BINS];
    float lo = 0.f, hi = 0.f;
#pragma unroll
    for (int k = 0; k < SD_MAX_BINS; ++k)
        if (k < K) {
            w[k] = s_w[c][k];
            hi = w[k] > hi ? w[k] : hi;
            lo = w[k] < lo ? w[k] : lo;
        }
    const long long row = (long long)W * kGlyph;     // image row stride in floats
    float* p = img + (long long)cy * kGlyph * row + (long long)cx0 * kGlyph + tid;
    for (int gy = 0; gy < kGlyph; ++gy, p += row) {
        const unsigned m = s_mask[gy * kGlyph + gx];
        float v = *p;
#pragma unroll
        for (int k = 0; k < SD_MAX_BINS; ++k)
            if (k < K) v = __fadd_rn(v, __fmul_rn(w[k], (m >> k) & 1u ? 1.f : 0.f));
        const float t = hi < v ? hi : v;
        *p = lo > t ? lo : t;
    }
}

// ---- relayout ---------------------------------------------------------------------------------------------------------------

struct RelayoutArgs {
    const float* in;
    float* out;
    int width, height;                    // equally sized grids, packed: grid i at i * dd * h * w floats in both buffers
    long long stride;
    const sd_hog_grid* grids;
    int frame0;
    int flip;
    int tiles_x;                          // 32-wide tiles per row of the widest grid
    int8_t perm[4 * SD_MAX_BINS];         // the flip permutation (dd <= 4 * 16)
};

// One CTA per 32 x 32 tile of one plane of one grid.  Plane d of the result is plane perm[d] (flip) or d of the input, with
// columns mirrored (flip: x -> w - 1 - x); TRANSPOSE then stores the plane as [w][h] through a padded shared-memory tile, so
// that both the reads and the writes of a warp are runs of consecutive floats.
template <bool TRANSPOSE>
__global__ void __launch_bounds__(kTile * 8) hog_relayout_kernel(const __grid_constant__ RelayoutArgs a)
{
    __shared__ float s[kTile][kTile + 1];
    const int g = a.frame0 + blockIdx.z, d = blockIdx.y;
    int W = a.width, H = a.height;
    const float* in;
    float* out;
    if (a.grids) {
        const sd_hog_grid e = a.grids[g];
        W = e.width; H = e.height;
        in = a.in + e.offset;
        out = a.out + e.out_offset;
    } else {
        in = a.in + (long long)g * a.stride;
        out = a.out + (long long)g * a.stride;
    }
    const int ty0 = blockIdx.x / a.tiles_x, x0 = (blockIdx.x - ty0 * a.tiles_x) * kTile, y0 = ty0 * kTile;
    if (x0 >= W || y0 >= H) return;
    const long long plane = (long long)W * H;
    const float* src = in + (a.flip ? a.perm[d] : d) * plane;
    float* dst = out + d * plane;
    const int tx = threadIdx.x, ty = threadIdx.y;
    const int x = x0 + tx;
#pragma unroll
    for (int j = 0; j < kTile; j += 8) {
        const int y = y0 + ty + j;
        if (x < W && y < H) {
            const float v = src[(long long)y * W + (a.flip ? W - 1 - x : x)];
            if constexpr (TRANSPOSE) s[ty + j][tx] = v;
            else dst[(long long)y * W + x] = v;
        }
    }
    if constexpr (TRANSPOSE) {
        __syncthreads();
        const int y = y0 + tx;                       // output column
#pragma unroll
        for (int j = 0; j < kTile; j += 8) {
            const int xr = x0 + ty + j;              // output row
            if (xr < W && y < H) dst[(long long)xr * H + y] = s[tx][ty + j];
        }
    }
}

// ---- shared by both entry points ----------------------------------------------------------------------------------------------

int check_config(sd_ctx* ctx, const sd_hog_grids* grids, int num_bins, int variant)
{
    SD_REQUIRE(ctx, grids, "null argument");
    if (const int rc = sd_hog_check_config(ctx, __func__, variant, num_bins)) return rc;
    SD_REQUIRE(ctx, grids->count >= 0, "negative grid count");
    return SD_OK;
}

}  // namespace

// The grids of a call: equally sized (packed, max_w x max_h cells), or the descriptor table read back once (the launch covers
// the largest grid; *table, if given, receives it).  Returns SD_OK, or an sd_fail status before anything is queued.
int sd_read_hog_grids(sd_ctx* ctx, const char* fn, const sd_hog_grids* grids, int* max_w, int* max_h, std::vector<sd_hog_grid>* table)
{
    const int count = grids->count;
    if (!grids->d_grids) {
        if (grids->width < 1 || grids->height < 1)
            return sd_fail(ctx, SD_ERR_INVALID, "%s: grids must be at least 1 x 1 cells (got %d x %d)", fn, grids->width, grids->height);
        *max_w = grids->width;
        *max_h = grids->height;
        return SD_OK;
    }
    std::vector<sd_hog_grid> t;
    if (const int rc = sd_fetch_table(ctx, grids->d_grids, count, t)) return rc;
    for (int i = 0; i < count; ++i) {
        const sd_hog_grid& d = t[i];
        if (d.width < 1 || d.height < 1 || d.offset < 0 || d.out_offset < 0)
            return sd_fail(ctx, SD_ERR_INVALID, "%s: grid %d (%d x %d cells, offsets %lld / %lld) must be at least 1 x 1 with "
                           "non-negative offsets", fn, i, d.width, d.height, (long long)d.offset, (long long)d.out_offset);
        *max_w = std::max(*max_w, (int)d.width);
        *max_h = std::max(*max_h, (int)d.height);
    }
    if (table) table->swap(t);
    return SD_OK;
}

extern "C" {

int sd_hog_permutation(int num_bins, int variant, int64_t* perm)
{
    if (!perm || sd_hog_check_config(nullptr, __func__, variant, num_bins)) return SD_ERR_INVALID;
    permutation(num_bins, variant, perm);
    return SD_OK;
}

int sd_hog_glyphs(int num_bins, int transposed, float* out)
{
    if (!out || num_bins < 1 || num_bins > SD_MAX_BINS || (transposed != 0 && transposed != 1)) return SD_ERR_INVALID;
    glyphs(num_bins, transposed != 0, out);
    return SD_OK;
}

int sd_hog_render(sd_ctx* ctx, const sd_hog_grids* grids, int num_bins, int variant, int transposed, float* d_image)
{
    if (!ctx) return SD_ERR_INVALID;
    if (const int rc = check_config(ctx, grids, num_bins, variant)) return rc;
    SD_REQUIRE(ctx, d_image, "null argument");
    SD_REQUIRE(ctx, transposed == 0 || transposed == 1, "transposed must be 0 or 1");
    const int count = grids->count;
    if (count == 0) return SD_OK;
    SD_REQUIRE(ctx, grids->d_features, "null argument");
    int max_w = 0, max_h = 0;
    if (const int rc = sd_read_hog_grids(ctx, __func__, grids, &max_w, &max_h, nullptr)) return rc;
    const int tiles_x = sd_div_up(max_w, kRenderCells);
    SD_REQUIRE(ctx, (long long)tiles_x * max_h <= INT_MAX, "grid too large");

    RenderArgs a;
    memset(&a, 0, sizeof(a));
    a.features = grids->d_features;
    a.image = d_image;
    a.width = grids->width; a.height = grids->height;
    a.in_stride = (long long)sd_hog_dd(num_bins, variant) * a.width * a.height;
    a.out_stride = (long long)a.width * a.height * kGlyphPixels;
    a.grids = grids->d_grids;
    a.K = num_bins;
    a.terms = variant == 1 ? 3 : 4;
    a.tiles_x = tiles_x;
    std::vector<float> table(static_cast<size_t>(num_bins) * kGlyphPixels);
    glyphs(num_bins, transposed != 0, table.data());
    for (int k = 0; k < num_bins; ++k)
        for (int p = 0; p < kGlyphPixels; ++p)
            if (table[k * kGlyphPixels + p] != 0.f) a.mask[p] |= (uint16_t)(1u << k);
    for (int f0 = 0; f0 < count; f0 += 65535) {
        a.frame0 = f0;
        hog_render_kernel<<<dim3((unsigned)(tiles_x * max_h), 1, (unsigned)std::min(count - f0, 65535)), kRenderThreads, 0, ctx->stream>>>(a);
        SD_LAUNCH_CHECK(ctx, "hog_render_kernel");
    }
    return SD_OK;
}

int sd_hog_relayout(sd_ctx* ctx, const sd_hog_grids* grids, int num_bins, int variant, int flip, int transpose, float* d_out)
{
    if (!ctx) return SD_ERR_INVALID;
    if (const int rc = check_config(ctx, grids, num_bins, variant)) return rc;
    SD_REQUIRE(ctx, d_out, "null argument");
    SD_REQUIRE(ctx, (flip == 0 || flip == 1) && (transpose == 0 || transpose == 1), "flip and transpose must be 0 or 1");
    const int count = grids->count;
    if (count == 0) return SD_OK;
    SD_REQUIRE(ctx, grids->d_features, "null argument");
    SD_REQUIRE(ctx, grids->d_features != d_out, "the relayout is out of place: d_out must not be the input");
    int max_w = 0, max_h = 0;
    if (const int rc = sd_read_hog_grids(ctx, __func__, grids, &max_w, &max_h, nullptr)) return rc;
    const int dd = sd_hog_dd(num_bins, variant);
    const int tiles_x = sd_div_up(max_w, kTile);
    SD_REQUIRE(ctx, (long long)tiles_x * sd_div_up(max_h, kTile) <= INT_MAX, "grid too large");
    if (!grids->d_grids) {
        const long long n = (long long)count * dd * max_w * max_h;
        const float *i0 = grids->d_features, *o0 = d_out;
        SD_REQUIRE(ctx, o0 + n <= i0 || i0 + n <= o0, "the relayout is out of place: d_out must not overlap the input");
    }

    RelayoutArgs a;
    memset(&a, 0, sizeof(a));
    a.in = grids->d_features;
    a.out = d_out;
    a.width = grids->width; a.height = grids->height;
    a.stride = (long long)dd * a.width * a.height;
    a.grids = grids->d_grids;
    a.flip = flip;
    a.tiles_x = tiles_x;
    int64_t perm[4 * SD_MAX_BINS];
    permutation(num_bins, variant, perm);
    for (int d = 0; d < dd; ++d) a.perm[d] = (int8_t)perm[d];
    const auto kern = transpose ? hog_relayout_kernel<true> : hog_relayout_kernel<false>;
    const unsigned gx = (unsigned)(tiles_x * sd_div_up(max_h, kTile));
    for (int f0 = 0; f0 < count; f0 += 65535) {
        a.frame0 = f0;
        kern<<<dim3(gx, (unsigned)dd, (unsigned)std::min(count - f0, 65535)), dim3(kTile, 8), 0, ctx->stream>>>(a);
        SD_LAUNCH_CHECK(ctx, "hog_relayout_kernel");
    }
    return SD_OK;
}

}  // extern "C"
