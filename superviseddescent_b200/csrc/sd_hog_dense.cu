// Dense HOG of whole 8-bit frames: VLFeat's vl_hog_put_image (one channel) followed by vl_hog_extract (reference
// include/rcr/hog.c:595-728, :857-1062) for every frame of a batch, written in VLFeat's planar layout [dd][hogH][hogW].
//
// One CTA per tile of T x T output cells of one frame.  The features of a cell need the histograms of its 3 x 3 cell
// neighbourhood, so the CTA builds the histograms of the tile plus a one-cell halo (clamped at the frame's cell grid) from the
// frame's pixels alone, and nothing leaves the CTA but the finished features:
//   stage the pixels that vote into those cells (TMA tile for equally sized frames, load loop otherwise)
//   gradient, orientation bin (hog_bin, sd_hog_common.cuh) and modulus of every interior pixel of the FRAME   hog.c:616-672
//   spatial weights per absolute coordinate, as the reference rounds them                                     hog.c:697-709
//   bilinear vote, separable: per cell, per row a sum over the row's pixels, then a sum over the rows          hog.c:713-724
//   cell energy in float, the four block factors, clamp and projection in double                              hog.c:875-1053
// Every histogram depends only on the frame's pixels and is summed in a fixed order (the order of the landmark-patch
// kernel's two vote passes), so the result does not depend on the tiling, on the batch, or on the run.  A frame of
// fs x fs pixels gives, bit for bit, the features the patch kernel computes from the same fs x fs patch.
#include "sd_internal.cuh"
#include "sd_hog_common.cuh"

#include <cuda.h>

#include <algorithm>
#include <cstring>
#include <vector>

namespace {

constexpr int kDenseThreads = 256;
constexpr int kDenseMaxCell = 32;   // largest cell size: one cell with its halo stays below 227 KB of shared memory at K = 16
constexpr int kDenseMaxTile = 14;   // (T + 2)^2 histogram cells <= kDenseThreads: one thread per histogram cell
constexpr int kDenseSpanBudget = 112;

struct DenseArgs {
    const uint8_t* images;
    int width, height, row_stride;       // equally sized frames (frames == nullptr)
    long long image_stride;
    const sd_frame* frames;              // optional: one descriptor per frame
    int frame0;                          // frame of blockIdx.z == 0
    float* out;
    const int64_t* out_offset;           // optional: first float of each frame's output
    long long out_stride;                // floats per frame when out_offset == nullptr
    int variant, cs, K, dd;
    int tile;                            // output cells per tile side
    int span;                            // staged pixels per side: cs * (tile + 4) + 2
    int pitch;                           // bytes per staged row (the TMA box width)
    int tma;                             // the staging is one TMA tile
    float ox[SD_MAX_BINS], oy[SD_MAX_BINS];
    int vbin[2];
};

// tile side in cells for a cell size: the staged region cs * (T + 4) + 2 stays near kDenseSpanBudget pixels
__host__ __device__ inline int dense_tile(int cs)
{
    const int t = (kDenseSpanBudget - 2) / cs - 4;
    return t < 1 ? 1 : (t > kDenseMaxTile ? kDenseMaxTile : t);
}

struct DenseSmem {
    int pix, g, bin, bx, wx1, wx2, by, wy1, wy2, T, hist, energy, mbar, total;
};

__host__ __device__ inline int dense_align(int v, int a) { return (v + a - 1) / a * a; }

// histogram cells of a tile with its halo, rounded up to a warp: the row stride of the per-cell vote arrays
__host__ __device__ inline int dense_cells(int tile) { return ((tile + 2) * (tile + 2) + 31) / 32 * 32; }

__host__ __device__ inline DenseSmem dense_smem_layout(int span, int pitch, int K, int hs)
{
    DenseSmem s;
    int o = 0;
    s.pix = o;    o = dense_align(o + pitch * span, 16);    // TMA destination: offset 0 of the 128-byte aligned block
    s.g = o;      o += span * span * 4;
    s.bx = o;     o += span * 4;
    s.wx1 = o;    o += span * 4;
    s.wx2 = o;    o += span * 4;
    s.by = o;     o += span * 4;
    s.wy1 = o;    o += span * 4;
    s.wy2 = o;    o += span * 4;
    s.T = o;      o += 2 * K * hs * 4;                     // [bin][histogram cell]: one column per thread, conflict free
    s.hist = o;   o += 2 * K * hs * 4;
    s.energy = o; o += hs * 4;
    s.mbar = dense_align(o, 8); o = s.mbar + 8;
    s.bin = o;    o = dense_align(o + span * span, 16);
    s.total = o;
    return s;
}

template <int KT>
__global__ void __launch_bounds__(kDenseThreads) hog_dense_kernel(const __grid_constant__ DenseArgs a, const __grid_constant__ CUtensorMap map)
{
    extern __shared__ __align__(128) unsigned char smem[];
    const int K = KT > 0 ? KT : a.K;
    const int cs = a.cs, tile = a.tile, span = a.span, pitch = a.pitch;
    const int hs = dense_cells(tile);
    const DenseSmem lay = dense_smem_layout(span, pitch, K, hs);
    uint8_t* s_pix = smem + lay.pix;
    float* s_g = reinterpret_cast<float*>(smem + lay.g);
    int8_t* s_bin = reinterpret_cast<int8_t*>(smem + lay.bin);
    int* s_bx = reinterpret_cast<int*>(smem + lay.bx);
    float* s_wx1 = reinterpret_cast<float*>(smem + lay.wx1);
    float* s_wx2 = reinterpret_cast<float*>(smem + lay.wx2);
    int* s_by = reinterpret_cast<int*>(smem + lay.by);
    float* s_wy1 = reinterpret_cast<float*>(smem + lay.wy1);
    float* s_wy2 = reinterpret_cast<float*>(smem + lay.wy2);
    float* s_T = reinterpret_cast<float*>(smem + lay.T);
    float* s_hist = reinterpret_cast<float*>(smem + lay.hist);
    float* s_energy = reinterpret_cast<float*>(smem + lay.energy);
    uint64_t* s_mbar = reinterpret_cast<uint64_t*>(smem + lay.mbar);
    const int tid = threadIdx.x;

    const int f = a.frame0 + blockIdx.z;
    int W = a.width, H = a.height, rs = a.row_stride;
    const uint8_t* __restrict__ img = a.images + (long long)f * a.image_stride;
    if (a.frames) {
        const sd_frame fr = a.frames[f];
        W = fr.width; H = fr.height; rs = fr.row_stride;
        img = a.images + fr.offset;
    }
    const int hogW = (W + cs / 2) / cs, hogH = (H + cs / 2) / cs;   // hog.c:542-543
    const int tx0 = blockIdx.x * tile, ty0 = blockIdx.y * tile;
    if (tx0 >= hogW || ty0 >= hogH) return;                           // the grid covers the largest frame of the batch
    const int tw = min(tile, hogW - tx0), th = min(tile, hogH - ty0);
    // histogram cells: the tile and a one-cell halo, clamped at the frame's cell grid (hog.c:930-933)
    const int hx0 = max(tx0 - 1, 0), hx1 = min(tx0 + tile, hogW - 1);
    const int hy0 = max(ty0 - 1, 0), hy1 = min(ty0 + tile, hogH - 1);
    const int nhx = hx1 - hx0 + 1, nhy = hy1 - hy0 + 1;
    // Staged region: pixel x votes into cells floor(hx) and floor(hx) + 1 with hx = (x + 0.5) / cs - 0.5, so the pixels of cells
    // hx0..hx1 lie in [cs hx0 - cs / 2 - 1 / 2, cs hx1 + 3 cs / 2 - 1 / 2); with their gradient neighbours they lie inside
    // [cs hx0 - cs - 1, cs hx1 + 2 cs].  Staged column i is frame column ox0 + i, at byte shift + i of its row.
    const int ox0 = cs * hx0 - cs - 1, oy0 = cs * hy0 - cs - 1;
    const int ax0 = ox0 & ~15;                                         // the TMA box starts on a 16-byte boundary
    const int shift = ox0 - ax0;

    // ---- S1: stage.  Bytes outside the frame are never read: only interior pixels of the frame vote (hog.c:616-617), and
    //      their neighbours are frame pixels.
    if (a.tma) {
        if (tid == 0) {
            const uint32_t bar = (uint32_t)__cvta_generic_to_shared(s_mbar);
            asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar));
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
            asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(pitch * span) : "memory");
            asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
                         ::"r"((uint32_t)__cvta_generic_to_shared(s_pix)), "l"(&map), "r"(bar), "r"(ax0), "r"(oy0), "r"(f)
                         : "memory");
        }
    } else {
        const int x_lo = max(ox0, 0), x_hi = min(ox0 + span, W);       // frame columns of the region
        const int y_lo = max(oy0, 0), y_hi = min(oy0 + span, H);
        const int nx = x_hi - x_lo;
        if (nx > 0)
            for (int i = tid; i < nx * (y_hi - y_lo); i += kDenseThreads) {
                const int r = i / nx, c = i - r * nx;
                const int y = y_lo + r, x = x_lo + c;
                s_pix[(y - oy0) * pitch + shift + (x - ox0)] = __ldg(img + (long long)y * rs + x);
            }
    }
    // spatial weights of every staged coordinate, exactly as hog.c:697-709 rounds them (hog_bintab_kernel's expression on the
    // absolute coordinate): b = floor(h), w2 = h - b, w1 = (float)(1.0 - w2); a pixel adds w1 to cell b and w2 to cell b + 1
    for (int i = tid; i < 2 * span; i += kDenseThreads) {
        const int t = i < span ? ox0 + i : oy0 + i - span;
        const float h = (float)__dadd_rn(__ddiv_rn((double)t + 0.5, (double)cs), -0.5);
        int b = (int)h;                                   // vl_floor_f, hog.h:52-58
        if (!(h >= 0.f || (float)b == h)) b -= 1;
        const float w2 = __fsub_rn(h, (float)b);
        const float w1 = (float)__dadd_rn(1.0, -(double)w2);
        if (i < span) { s_bx[i] = b; s_wx1[i] = w1; s_wx2[i] = w2; }
        else { s_by[i - span] = b; s_wy1[i - span] = w1; s_wy2[i - span] = w2; }
    }
    __syncthreads();
    if (a.tma) {
        const uint32_t bar = (uint32_t)__cvta_generic_to_shared(s_mbar);
        uint32_t ok = 0;
        const long long t0 = clock64();
        while (!ok) {                                      // bounded: a protocol bug must trap, never hang the GPU
            asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                         : "=r"(ok) : "r"(bar) : "memory");
            if (!ok && clock64() - t0 > 4000000000LL) __trap();
        }
    }

    // ---- S2: gradient, orientation bin and modulus of every staged pixel that is interior to the frame (hog.c:631-672): the
    //      gradient of 8-bit pixels is a pair of integers in [-255, 255], its squared modulus an exact float integer whose
    //      correctly rounded root is the reference's sqrtf
    {
        const int xa = max(1, 1 - ox0), xb = min(span - 2, W - 2 - ox0);
        const int ya = max(1, 1 - oy0), yb = min(span - 2, H - 2 - oy0);
        const int nx = xb - xa + 1;
        if (nx > 0)
            for (int i = tid; i < nx * (yb - ya + 1); i += kDenseThreads) {
                const int r = i / nx;
                const int y = ya + r, x = xa + i - r * nx;
                const uint8_t* p = s_pix + y * pitch + shift + x;
                const int gx = (int)p[1] - (int)p[-1];
                const int gy = (int)p[pitch] - (int)p[-pitch];
                const int g2 = gx * gx + gy * gy;
                const float g = __fsqrt_rn((float)g2);
                s_bin[y * span + x] = (int8_t)hog_bin(a, K, gx, gy, g2, g);
                s_g[y * span + x] = g;
            }
    }
    __syncthreads();

    // ---- S3: bilinear spatial vote (hog.c:697-724), one thread per histogram cell, in the order of the patch kernel's two
    //      passes: per interior row y of the cell, T[b] = sum over the row's voting pixels x (ascending) of g * wx; then
    //      hist[b] += T[b] * wy, rows ascending.  Votes into cells outside the grid are never formed (hog.c:713-723).
    const int ncell = nhx * nhy;
    if (tid < ncell) {
        const int cyl = tid / nhx, cxl = tid - cyl * nhx;
        const int ci = hx0 + cxl, cj = hy0 + cyl;
        // the interior pixels of the frame that vote into column ci / row cj: a contiguous run of staged coordinates
        int xlo = span, xhi = -1, ylo = span, yhi = -1;
        for (int i = max(1, 1 - ox0); i <= min(span - 2, W - 2 - ox0); ++i)
            if (s_bx[i] == ci || s_bx[i] == ci - 1) { xlo = min(xlo, i); xhi = i; }
        for (int i = max(1, 1 - oy0); i <= min(span - 2, H - 2 - oy0); ++i)
            if (s_by[i] == cj || s_by[i] == cj - 1) { ylo = min(ylo, i); yhi = i; }
        float* T = s_T + tid;
        float* hist = s_hist + tid;
        for (int b = 0; b < 2 * K; ++b) hist[b * hs] = 0.f;
        for (int y = ylo; y <= yhi; ++y) {
            for (int b = 0; b < 2 * K; ++b) T[b * hs] = 0.f;
            const int8_t* bp = s_bin + y * span;
            const float* gp = s_g + y * span;
            for (int x = xlo; x <= xhi; ++x) {
                const int b = bp[x];
                // b < 0: zero gradient (the patch kernel adds its +0 to bin 0, which changes nothing), or K = 1 on the gx = 0
                // axis, which the reference does not vote
                if (b < 0) continue;
                const float w = s_bx[x] == ci ? s_wx1[x] : s_wx2[x];
                float* q = T + b * hs;
                *q = __fadd_rn(*q, __fmul_rn(gp[x], w));
            }
            const float wy = s_by[y] == cj ? s_wy1[y] : s_wy2[y];
            for (int b = 0; b < 2 * K; ++b) {
                float* h = hist + b * hs;
                *h = __fadd_rn(*h, __fmul_rn(T[b * hs], wy));
            }
        }
        // ---- S4: undirected cell energy (hog.c:875-890)
        float e = 0.f;
        for (int k = 0; k < K; ++k) {
            const float h = __fadd_rn(hist[k * hs], hist[(k + K) * hs]);
            e = __fadd_rn(e, __fmul_rn(h, h));
        }
        s_energy[tid] = e;
    }
    __syncthreads();

    // ---- S5-S7: one thread per output cell: the four block factors in double (hog.c:930-982), normalise, clamp at 0.2 and
    //      project (hog.c:985-1044), texture dims summed in ascending k (hog.c:1046-1053).  Planar store: a warp writes runs of
    //      tw consecutive floats of each feature plane.
    if (tid < tw * th) {
        const int yl = tid / tw;
        const int x = tx0 + tid - yl * tw, y = ty0 + yl;
        const int xm = max(x - 1, 0), xp = min(x + 1, hogW - 1);
        const int ym = max(y - 1, 0), yp = min(y + 1, hogH - 1);
        double fac[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            // factor1: n1+n2+n4+n5, factor2: n2+n3+n5+n6, factor3: n4+n5+n7+n8, factor4: n5+n6+n8+n9
            const int xa = ((q & 1) ? x : xm) - hx0, xb = ((q & 1) ? xp : x) - hx0;
            const int ya = ((q & 2) ? y : ym) - hy0, yb = ((q & 2) ? yp : y) - hy0;
            double s = (double)s_energy[xa + ya * nhx];
            s = __dadd_rn(s, (double)s_energy[xb + ya * nhx]);
            s = __dadd_rn(s, (double)s_energy[xa + yb * nhx]);
            s = __dadd_rn(s, (double)s_energy[xb + yb * nhx]);
            s = __dadd_rn(s, 1e-4);
            fac[q] = __ddiv_rn(1.0, sqrt(s));
        }
        const int c = (x - hx0) + (y - hy0) * nhx;
        const long long plane = (long long)hogW * hogH;
        float* __restrict__ out = a.out + (a.out_offset ? a.out_offset[f] : (long long)f * a.out_stride) + (long long)y * hogW + x;
        double t[4] = {0.0, 0.0, 0.0, 0.0};
        for (int k = 0; k < K; ++k) {
            const double ha = (double)s_hist[k * hs + c];
            const double hb = (double)s_hist[(k + K) * hs + c];
            double sa = 0.0, sb = 0.0, sc = 0.0;
            double hcv[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                double haf = __dmul_rn(fac[q], ha);
                double hbf = __dmul_rn(fac[q], hb);
                double hcf = __dadd_rn(haf, hbf);
                haf = (0.2 < haf) ? 0.2 : haf;
                hbf = (0.2 < hbf) ? 0.2 : hbf;
                hcf = (0.2 < hcf) ? 0.2 : hcf;
                hcv[q] = hcf;
                sa = (q == 0) ? haf : __dadd_rn(sa, haf);
                sb = (q == 0) ? hbf : __dadd_rn(sb, hbf);
                sc = (q == 0) ? hcf : __dadd_rn(sc, hcf);
                t[q] = __dadd_rn(t[q], hcf);
            }
            if (a.variant == 1) {                               // UoCTTI
                out[k * plane] = (float)__dmul_rn(0.5, sa);
                out[(k + K) * plane] = (float)__dmul_rn(0.5, sb);
                out[(k + 2 * K) * plane] = (float)__dmul_rn(0.5, sc);
            } else {                                            // Dalal-Triggs
#pragma unroll
                for (int q = 0; q < 4; ++q) out[(k + q * K) * plane] = (float)hcv[q];
            }
        }
        if (a.variant == 1) {
            const float c18 = __fdiv_rn(1.0f, __fsqrt_rn(18.0f));
#pragma unroll
            for (int q = 0; q < 4; ++q) out[(3 * K + q) * plane] = (float)__dmul_rn((double)c18, t[q]);
        }
    }
}

// the rules of vl_hog_prepare_buffers (hog.c:542-548) and of this implementation's range, shared by both entry points
bool dense_shape(int width, int height, int cs, int K, int variant, int* hog_w, int* hog_h, int* dd)
{
    if (variant != 0 && variant != 1) return false;
    if (K < 1 || K > SD_MAX_BINS || cs < 1 || cs > kDenseMaxCell) return false;
    if (width <= 3 || height <= 3) return false;
    const int w = (width + cs / 2) / cs, h = (height + cs / 2) / cs;
    if (w <= 0 || h <= 0) return false;
    *hog_w = w;
    *hog_h = h;
    *dd = variant == 1 ? 3 * K + 4 : 4 * K;
    return true;
}

}  // namespace

extern "C" {

int sd_hog_dense_shape(int width, int height, int cell_size, int num_bins, int variant, int* hog_w, int* hog_h, int* dd)
{
    if (!hog_w || !hog_h || !dd) return SD_ERR_INVALID;
    int w, h, d;
    if (!dense_shape(width, height, cell_size, num_bins, variant, &w, &h, &d)) return SD_ERR_INVALID;
    *hog_w = w;
    *hog_h = h;
    *dd = d;
    return SD_OK;
}

int sd_hog_dense(sd_ctx* ctx, const sd_image_batch* images, int cell_size, int num_bins, int variant, float* d_out,
                 const int64_t* d_out_offset)
{
    if (!ctx) return SD_ERR_INVALID;
    SD_REQUIRE(ctx, images && d_out, "null argument");
    SD_REQUIRE(ctx, !images->d_roi, "a batch with regions of interest has no whole frames");
    SD_REQUIRE(ctx, variant == 0 || variant == 1, "unknown HOG variant");
    SD_REQUIRE(ctx, num_bins >= 1 && num_bins <= SD_MAX_BINS, "num_bins must be in [1,16]");
    SD_REQUIRE(ctx, cell_size >= 1 && cell_size <= kDenseMaxCell, "cell_size must be in [1,32]");
    SD_REQUIRE(ctx, images->count >= 0, "negative frame count");
    const int count = images->count;
    if (count == 0) return SD_OK;
    SD_REQUIRE(ctx, images->d_data, "null argument");

    // frame sizes: the batch's, or the descriptor table read back once (the grid covers the largest frame)
    int max_w = 0, max_h = 0, dd = 0;
    bool uniform = true;
    if (images->d_frames) {
        std::vector<sd_frame> fr(count);
        SD_CUDA(ctx, cudaMemcpyAsync(fr.data(), images->d_frames, sizeof(sd_frame) * count, cudaMemcpyDeviceToHost, ctx->stream));
        SD_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        for (int i = 0; i < count; ++i) {
            int w, h;
            if (!dense_shape(fr[i].width, fr[i].height, cell_size, num_bins, variant, &w, &h, &dd))
                return sd_fail(ctx, SD_ERR_INVALID, "%s: frame %d is %d x %d: frames must be wider and taller than 3 px and at least "
                               "half a cell", __func__, i, fr[i].width, fr[i].height);
            SD_REQUIRE(ctx, fr[i].row_stride >= fr[i].width && fr[i].offset >= 0, "bad frame descriptor");
            max_w = std::max(max_w, w);
            max_h = std::max(max_h, h);
            uniform = uniform && fr[i].width == fr[0].width && fr[i].height == fr[0].height;
        }
    } else {
        SD_REQUIRE(ctx, dense_shape(images->width, images->height, cell_size, num_bins, variant, &max_w, &max_h, &dd),
                   "frames must be wider and taller than 3 px and at least half a cell");
        SD_REQUIRE(ctx, images->row_stride >= images->width && (count == 1 || images->image_stride > 0), "bad strides");
    }
    SD_REQUIRE(ctx, d_out_offset || uniform, "frames of different sizes need one output offset per frame");

    DenseArgs a;
    memset(&a, 0, sizeof(a));
    a.images = images->d_data;
    a.width = images->width; a.height = images->height; a.row_stride = images->row_stride;
    a.image_stride = images->image_stride;
    a.frames = images->d_frames;
    a.out = d_out;
    a.out_offset = d_out_offset;
    a.out_stride = (long long)dd * max_w * max_h;
    a.variant = variant; a.cs = cell_size; a.K = num_bins; a.dd = dd;
    a.tile = dense_tile(cell_size);
    a.span = cell_size * (a.tile + 4) + 2;
    a.pitch = dense_align(a.span + 15, 16);
    hog_orientations(num_bins, a.ox, a.oy, a.vbin);   // hog.c:195-204

    // TMA staging: equally sized frames with 16-byte aligned base and pitches (a box of pitch x span bytes per CTA; bytes past
    // the frame's edge are zero-filled and never read)
    CUtensorMap map;
    memset(&map, 0, sizeof(map));
    if (!images->d_frames && (reinterpret_cast<uintptr_t>(images->d_data) & 15) == 0 && (images->row_stride % 16) == 0 &&
        (count == 1 || images->image_stride % 16 == 0)) {
        PFN_hogEncodeTiled enc = hog_encode_fn();
        if (enc) {
            cuuint64_t gdim[3] = {(cuuint64_t)images->width, (cuuint64_t)images->height, (cuuint64_t)count};
            cuuint64_t gstride[2] = {(cuuint64_t)images->row_stride,
                                     (cuuint64_t)(count > 1 ? images->image_stride : (int64_t)images->row_stride * images->height)};
            if (gstride[1] % 16) gstride[1] = (gstride[1] + 15) / 16 * 16;
            cuuint32_t box[3] = {(cuuint32_t)a.pitch, (cuuint32_t)a.span, 1};
            cuuint32_t estr[3] = {1, 1, 1};
            a.tma = enc(&map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, const_cast<uint8_t*>(images->d_data), gdim, gstride, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
        }
    }

    const DenseSmem lay = dense_smem_layout(a.span, a.pitch, num_bins, dense_cells(a.tile));
    SD_REQUIRE(ctx, lay.total <= 227 * 1024, "dense HOG configuration needs more than 227 KB of shared memory");
    auto kern = hog_dense_kernel<0>;
    if (num_bins == 4) kern = hog_dense_kernel<4>;
    else if (num_bins == 9) kern = hog_dense_kernel<9>;
    SD_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, lay.total));
    const dim3 block(kDenseThreads);
    const unsigned gx = (unsigned)sd_div_up(max_w, a.tile), gy = (unsigned)sd_div_up(max_h, a.tile);
    for (int f0 = 0; f0 < count; f0 += 65535) {
        a.frame0 = f0;
        const dim3 grid(gx, gy, (unsigned)std::min(count - f0, 65535));
        kern<<<grid, block, lay.total, ctx->stream>>>(a, map);
        SD_LAUNCH_CHECK(ctx, "hog_dense_kernel");
    }
    return SD_OK;
}

}  // extern "C"
