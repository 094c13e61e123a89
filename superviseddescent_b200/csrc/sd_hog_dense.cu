// Dense HOG of whole frames: VLFeat's vl_hog_put_image followed by vl_hog_extract (reference include/rcr/hog.c:595-728,
// :857-1062) for every frame of a batch, written in VLFeat's planar layout [dd][hogH][hogW].
//
// One CTA per tile of T x T output cells of one frame.  The features of a cell need the histograms of its 3 x 3 cell
// neighbourhood, so the CTA builds the histograms of the tile plus a one-cell halo (clamped at the frame's cell grid) from the
// frame's pixels alone, and nothing leaves the CTA but the finished features:
//   S1 stage the pixels that vote into those cells (8-bit grey: TMA tile for equally sized frames, load loop otherwise)
//   S2 gradient, orientation bin(s) (sd_hog_common.cuh) and modulus of every interior pixel of the FRAME        hog.c:616-682
//      spatial weights per absolute coordinate, as the reference rounds them                                     hog.c:697-709
//   S3 bilinear vote, separable: per cell, per row a sum over the row's pixels, then a sum over the rows          hog.c:713-724
//   S4-S7 cell energy in float, the four block factors, clamp and projection in double                          hog.c:875-1053
// Three kernels run the same CTA body (hog_dense_cta), which differs only in S1-S2:
//   hog_dense_kernel   8-bit grey frames, nearest-bin orientations (sd_hog_dense): staged pixels, the integer bin rule
//   hog_images_kernel  u8 or f32 frames of 1..16 strided channels, nearest-bin or bilinear orientations (sd_hog_dense_images):
//                      each pixel's gradient is read straight from the frame, channel by channel, and the channel with the
//                      largest squared modulus wins (hog.c:631-644); bilinear pixels keep two bins and a second weight
//   hog_polar_kernel   a caller's gradient field, modulus and angle per pixel (sd_hog_dense_polar, vl_hog_put_polar_field,
//                      hog.c:746-845): two f32 fields read in place through element strides; every pixel of the frame
//                      votes, the border included, and the bins come from the angle alone (polar_bins)
// Every histogram depends only on the frame's pixels and is summed in a fixed order (the order of the landmark-patch
// kernel's two vote passes), so the result does not depend on the tiling, on the batch, or on the run.  A frame of
// fs x fs pixels gives, bit for bit, the features the patch kernel computes from the same fs x fs patch.
//
// Pyramids (sd_hog_pyramid, sd_hog_pyramid_images, sd_hog_pyramid_float and the filter trainer's slices) are one routine,
// sd_hog_pyramid_frames, on a host list of frames that each entry point reads once by its own rules: per slice of frames, every
// level resized into scratch by hog_pyramid_resize_images_kernel, then one dense pass over the levels, hog_dense_kernel for
// batches that sd_hog_dense takes (8-bit grey, nearest bins) and hog_images_kernel for the others.
#include "sd_internal.cuh"
#include "sd_hog_common.cuh"

#include <algorithm>
#include <climits>
#include <cstring>
#include <type_traits>
#include <vector>

namespace {

constexpr int kDenseThreads = 256;
constexpr int kDenseMaxTile = 14;   // (T + 2)^2 histogram cells <= kDenseThreads: one thread per histogram cell
constexpr int kDenseSpanBudget = 112;
constexpr int kDenseMaxChannels = 16;

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
    HogOrient orient;
};

struct ImageArgs {
    const void* data;                    // uint8_t or float elements
    sd_hog_image frame;                  // equally sized frames (frames == nullptr): frame i at frame.offset + i * image_stride
    long long image_stride;
    const sd_hog_image* frames;          // optional: one descriptor per frame
    int channels;
    int frame0;
    float* out;
    const int64_t* out_offset;
    long long out_stride;
    int variant, cs, K, dd;
    int tile;
    int span;                            // pixels per side of the region that votes: cs * (tile + 3) + 4
    double pi_k;                         // pi / K (hog.c:677)
    HogOrient orient;
};

struct PolarArgs {
    const float* modulus;                // one descriptor places element e at modulus[e] and angle[e]
    const float* angle;
    sd_hog_image frame;                  // equally sized fields (frames == nullptr): field i at frame.offset + i * image_stride
    long long image_stride;
    const sd_hog_image* frames;          // optional: one descriptor per field
    int directed;                        // the bin period is 2K (directed) or K
    int frame0;
    float* out;
    const int64_t* out_offset;
    long long out_stride;
    int variant, cs, K, dd;
    int tile;
    int span;                            // pixels per side of the region that votes: cs * (tile + 3) + 4
    double pi_k;                         // pi / K (hog.c:756)
};

// tile side in cells for a cell size: the staged region cs * (T + 4) + 2 stays near kDenseSpanBudget pixels
__host__ __device__ inline int dense_tile(int cs)
{
    const int t = (kDenseSpanBudget - 2) / cs - 4;
    return t < 1 ? 1 : (t > kDenseMaxTile ? kDenseMaxTile : t);
}

struct DenseSmem {
    int pix, g, bin, bx, wx1, wx2, by, wy1, wy2, T, hist, energy, mbar, bin1, w1, total;
};

__host__ __device__ inline int dense_align(int v, int a) { return (v + a - 1) / a * a; }

// histogram cells of a tile with its halo, rounded up to a warp: the row stride of the per-cell vote arrays
__host__ __device__ inline int dense_cells(int tile) { return ((tile + 2) * (tile + 2) + 31) / 32 * 32; }

// pitch 0: no staged pixels.  bilinear: a second bin and the second orientation weight per pixel, after everything else.
__host__ __device__ inline DenseSmem dense_smem_layout(int span, int pitch, int K, int hs, bool bilinear = false)
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
    s.bin1 = s.w1 = o;
    if (bilinear) {
        s.bin1 = o; o = dense_align(o + span * span, 16);
        s.w1 = o;   o += span * span * 4;
    }
    s.total = o;
    return s;
}

// spatial weights of every staged coordinate (columns ox0.., rows oy0..) by their absolute coordinate (hog_spatial_weight)
__device__ __forceinline__ void dense_weights(int tid, int cs, int span, int ox0, int oy0, int* s_bx, float* s_wx1, float* s_wx2,
                                              int* s_by, float* s_wy1, float* s_wy2)
{
    for (int i = tid; i < 2 * span; i += kDenseThreads) {
        int b;
        float w1, w2;
        hog_spatial_weight(i < span ? ox0 + i : oy0 + i - span, cs, &b, &w1, &w2);
        if (i < span) { s_bx[i] = b; s_wx1[i] = w1; s_wx2[i] = w2; }
        else { s_by[i - span] = b; s_wy1[i - span] = w1; s_wy2[i - span] = w2; }
    }
}

// the staged pitch of a configuration: 8-bit grey frames are staged in shared memory, strided frames are read in place
__device__ __forceinline__ int dense_pitch(const DenseArgs& a) { return a.pitch; }
__device__ __forceinline__ int dense_pitch(const ImageArgs&) { return 0; }
__device__ __forceinline__ int dense_pitch(const PolarArgs&) { return 0; }

// ---- orientation bins of a polar-field pixel (hog.c:784-800) without the reference's loop.  ho = (float)(angle / (pi / K)) in
//      double as there, bino = floor(ho), wo2 = ho - bino and wo1 = 1 - wo2 in float.  hog.c adds 2K to bino until it is
//      non-negative and then takes it modulo period (K, or 2K when directed); period divides 2K, so that is the Euclidean
//      residue of bino, which floorf and fmodf give exactly for every finite ho, with no bound on |ho|.  Nearest-bin: bino + 1
//      when wo1 > wo2 fails (a tie included), modulo period; bilinear: bins bino and bino + 1 modulo period, *w1 = wo2 the
//      weight of the second (S3 forms wo1 = 1 - wo2 as hog.c does).  A pixel whose ho is not finite (a non-finite angle, or
//      one whose quotient overflows float; hog.c's floor is undefined there) gets bin -1 and does not vote.  Every other bin
//      is in [0, period).
template <bool BIL>
__device__ __forceinline__ int polar_bins(float angle, double pi_k, int period, int* b1, float* w1)
{
    const float ho = (float)__ddiv_rn((double)angle, pi_k);
    if (!isfinite(ho)) return -1;
    const float bino = floorf(ho);
    const float wo2 = __fsub_rn(ho, bino), wo1 = __fsub_rn(1.f, wo2);
    float r = fmodf(bino, (float)period);            // exact: an integer in (-period, period)
    if (r < 0.f) r += (float)period;
    const int b = (int)r;
    if constexpr (BIL) {
        *b1 = b + 1 == period ? 0 : b + 1;
        *w1 = wo2;
        return b;
    } else {
        const int n = b + (wo1 > wo2 ? 0 : 1);
        return n == period ? 0 : n;
    }
}

// One CTA of any of the three kernels.  STAGED (DenseArgs): 8-bit grey frames, staged by TMA or a load loop, nearest-bin
// orientations from the integer rule.  POLAR (PolarArgs): a modulus and an angle field read in place, nearest-bin or (BIL)
// bilinear bins from the angle.  Otherwise (ImageArgs): Pix frames of C strided channels read in place, nearest-bin or (BIL)
// bilinear orientations.  The weights and S3-S7 are the same code for all three.
template <int KT, bool STAGED, class Pix, bool BIL, class Args>
__device__ __forceinline__ void hog_dense_cta(const Args& a, const CUtensorMap* map)
{
    // The pixels that vote: those in [E, W - 1 - E] x [E, H - 1 - E].  A gradient needs its neighbours, so only interior pixels
    // vote (hog.c:616-617); a polar field votes at every pixel of the frame (hog.c:770-780).
    constexpr bool POLAR = std::is_same<Args, PolarArgs>::value;
    constexpr int E = POLAR ? 0 : 1;
    extern __shared__ __align__(128) unsigned char smem[];
    const int K = KT > 0 ? KT : a.K;
    const int cs = a.cs, tile = a.tile, span = a.span, pitch = dense_pitch(a);
    const int hs = dense_cells(tile);
    const DenseSmem lay = dense_smem_layout(span, pitch, K, hs, BIL);
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
    int8_t* s_bin1 = reinterpret_cast<int8_t*>(smem + lay.bin1);   // BIL: second bin and weight of each pixel
    float* s_w1 = reinterpret_cast<float*>(smem + lay.w1);
    const int tid = threadIdx.x;

    const int f = a.frame0 + blockIdx.z;
    int W, H, rs;                                    // STAGED: the frame's size and row stride in bytes
    const uint8_t* __restrict__ img;
    sd_hog_image fr;                                 // otherwise: the frame's descriptor
    const Pix* __restrict__ pimg;
    const float* __restrict__ pmod;                  // POLAR: the frame's modulus and angle fields
    const float* __restrict__ pang;
    if constexpr (POLAR) {
        fr = a.frames ? a.frames[f] : a.frame;
        const long long e0 = a.frames ? fr.offset : fr.offset + (long long)f * a.image_stride;
        pmod = a.modulus + e0;
        pang = a.angle + e0;
        W = fr.width; H = fr.height;
    } else if constexpr (STAGED) {
        W = a.width; H = a.height; rs = a.row_stride;
        img = a.images + (long long)f * a.image_stride;
        if (a.frames) {
            const sd_frame d = a.frames[f];
            W = d.width; H = d.height; rs = d.row_stride;
            img = a.images + d.offset;
        }
    } else {
        fr = a.frames ? a.frames[f] : a.frame;
        pimg = static_cast<const Pix*>(a.data) + (a.frames ? fr.offset : fr.offset + (long long)f * a.image_stride);
        W = fr.width; H = fr.height;
    }
    const int hogW = (W + cs / 2) / cs, hogH = (H + cs / 2) / cs;   // hog.c:542-543
    const int tx0 = blockIdx.x * tile, ty0 = blockIdx.y * tile;
    if (tx0 >= hogW || ty0 >= hogH) return;                           // the grid covers the largest frame of the batch
    const int tw = min(tile, hogW - tx0), th = min(tile, hogH - ty0);
    // histogram cells: the tile and a one-cell halo, clamped at the frame's cell grid (hog.c:930-933)
    const int hx0 = max(tx0 - 1, 0), hx1 = min(tx0 + tile, hogW - 1);
    const int hy0 = max(ty0 - 1, 0), hy1 = min(ty0 + tile, hogH - 1);
    const int nhx = hx1 - hx0 + 1, nhy = hy1 - hy0 + 1;
    // Region: pixel x votes into cells floor(hx) and floor(hx) + 1 with hx = (x + 0.5) / cs - 0.5, so the pixels of cells
    // hx0..hx1 lie in [cs hx0 - cs / 2 - 1 / 2, cs hx1 + 3 cs / 2 - 1 / 2); with their gradient neighbours they lie inside
    // [cs hx0 - cs / 2 - 3 / 2, cs hx1 + 3 cs / 2 + 1 / 2].  STAGED stages [cs hx0 - cs - 1, cs hx1 + 2 cs] (span
    // cs (tile + 4) + 2); staged column i is frame column ox0 + i, at byte shift + i of its row.  Frames read in place keep per-pixel
    // values for the tightest region, ox0 = cs hx0 - floor(cs / 2) - 2 with span cs (tile + 3) + 4: 132 wide at cs 32.
    // A polar field needs no neighbours, so the same region holds every pixel that votes into hx0..hx1, border pixels included:
    // since hx1 <= hx0 + tile + 1, the voting pixels lie in [cs hx0 - cs / 2 - 1 / 2, cs hx0 + cs tile + 5 cs / 2 - 1 / 2), and
    // [ox0, ox0 + span - 1] = [cs hx0 - floor(cs / 2) - 2, cs hx0 + cs tile + 3 cs - floor(cs / 2) + 1] contains it with at least
    // one pixel to spare on each side.  Region columns outside the frame (x < 0 or x > W - 1) are left out by the voting range.
    const int ox0 = STAGED ? cs * hx0 - cs - 1 : cs * hx0 - cs / 2 - 2, oy0 = STAGED ? cs * hy0 - cs - 1 : cs * hy0 - cs / 2 - 2;

    if constexpr (STAGED) {
        const int ax0 = ox0 & ~15;                                     // the TMA box starts on a 16-byte boundary
        const int shift = ox0 - ax0;

        // ---- S1: stage.  Bytes outside the frame are never read: only interior pixels of the frame vote (hog.c:616-617), and
        //      their neighbours are frame pixels.
        if (a.tma) {
            if (tid == 0) hog_tma_load(s_mbar, s_pix, map, ax0, oy0, f, pitch * span);
        } else {
            const int x_lo = max(ox0, 0), x_hi = min(ox0 + span, W);   // frame columns of the region
            const int y_lo = max(oy0, 0), y_hi = min(oy0 + span, H);
            const int nx = x_hi - x_lo;
            if (nx > 0)
                for (int i = tid; i < nx * (y_hi - y_lo); i += kDenseThreads) {
                    const int r = i / nx, c = i - r * nx;
                    const int y = y_lo + r, x = x_lo + c;
                    s_pix[(y - oy0) * pitch + shift + (x - ox0)] = __ldg(img + (long long)y * rs + x);
                }
        }
        dense_weights(tid, cs, span, ox0, oy0, s_bx, s_wx1, s_wx2, s_by, s_wy1, s_wy2);
        __syncthreads();
        if (a.tma) hog_tma_wait(s_mbar);

        // ---- S2: gradient, orientation bin and modulus of every staged pixel that is interior to the frame (hog.c:631-672):
        //      the gradient of 8-bit pixels is a pair of integers in [-255, 255], its squared modulus an exact float integer
        //      whose correctly rounded root is the reference's sqrtf
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
                    s_bin[y * span + x] = (int8_t)hog_bin(a.orient, K, gx, gy, g);
                    s_g[y * span + x] = g;
                }
        }
    } else if constexpr (POLAR) {
        dense_weights(tid, cs, span, ox0, oy0, s_bx, s_wx1, s_wx2, s_by, s_wy1, s_wy2);
        // ---- S2 (hog.c:770-800): per pixel of the frame, the modulus and the bin(s) of the angle (polar_bins); a modulus <= 0
        //      does not vote (a NaN modulus does, as in hog.c)
        const long long prs = fr.row_stride, pps = fr.pixel_stride;
        const int period = a.directed ? 2 * K : K;
        const int xa = max(E, E - ox0), xb = min(span - 1 - E, W - 1 - E - ox0);
        const int ya = max(E, E - oy0), yb = min(span - 1 - E, H - 1 - E - oy0);
        const int nx = xb - xa + 1;
        if (nx > 0)
            for (int i = tid; i < nx * (yb - ya + 1); i += kDenseThreads) {
                const int r = i / nx;
                const int y = ya + r, x = xa + i - r * nx;
                const long long e = (long long)(oy0 + y) * prs + (long long)(ox0 + x) * pps;
                const float m = __ldg(pmod + e);
                int b1 = -1;
                float w1 = 0.f;
                const int b0 = polar_bins<BIL>(__ldg(pang + e), a.pi_k, period, &b1, &w1);
                s_bin[y * span + x] = (int8_t)(m <= 0.f ? -1 : b0);
                if constexpr (BIL) {
                    s_bin1[y * span + x] = (int8_t)b1;
                    s_w1[y * span + x] = w1;
                }
                s_g[y * span + x] = m;
            }
    } else {
        dense_weights(tid, cs, span, ox0, oy0, s_bx, s_wx1, s_wx2, s_by, s_wy1, s_wy2);
        // ---- S2 (hog.c:631-682): per interior pixel, the gradient of every channel in ascending order, in float; a channel
        //      wins when its squared modulus (two rounded products, one rounded sum) is strictly larger, starting from 0, so a
        //      pixel whose channels all have a zero gradient does not vote.  8-bit gradients are integers: the nearest bin comes
        //      from the exact integer rule (hog_bin); float gradients, and both bins of the bilinear assignment, from the
        //      reference's float chain.
        const long long prs = fr.row_stride, pps = fr.pixel_stride, pcs = fr.channel_stride;
        const int xa = max(1, 1 - ox0), xb = min(span - 2, W - 2 - ox0);
        const int ya = max(1, 1 - oy0), yb = min(span - 2, H - 2 - oy0);
        const int nx = xb - xa + 1;
        if (nx > 0)
            for (int i = tid; i < nx * (yb - ya + 1); i += kDenseThreads) {
                const int r = i / nx;
                const int y = ya + r, x = xa + i - r * nx;
                const Pix* p = pimg + (long long)(oy0 + y) * prs + (long long)(ox0 + x) * pps;
                float gx = 0.f, gy = 0.f, g2 = 0.f;
                for (int c = 0; c < a.channels; ++c, p += pcs) {
                    const float gx_ = __fsub_rn((float)__ldg(p + pps), (float)__ldg(p - pps));
                    const float gy_ = __fsub_rn((float)__ldg(p + prs), (float)__ldg(p - prs));
                    const float g2_ = __fadd_rn(__fmul_rn(gx_, gx_), __fmul_rn(gy_, gy_));
                    if (g2_ > g2) { gx = gx_; gy = gy_; g2 = g2_; }
                }
                const float g = __fsqrt_rn(g2);
                int b0;
                if constexpr (BIL) {
                    int b1;
                    float w1;
                    hog_bins_bilinear(a.orient, a.pi_k, K, hog_unit(gx, g), hog_unit(gy, g), b0, b1, w1);
                    s_bin1[y * span + x] = (int8_t)b1;
                    s_w1[y * span + x] = w1;
                } else if constexpr (std::is_same<Pix, uint8_t>::value) {
                    b0 = hog_bin(a.orient, K, (int)gx, (int)gy, g);
                } else {
                    b0 = hog_bin_unit(a.orient, K, hog_unit(gx, g), hog_unit(gy, g));
                }
                s_bin[y * span + x] = (int8_t)b0;
                s_g[y * span + x] = g;
            }
    }
    __syncthreads();

    // ---- S3: bilinear spatial vote (hog.c:697-724), one thread per histogram cell, in the order of the patch kernel's two
    //      passes: per interior row y of the cell, T[b] = sum over the row's voting pixels x (ascending) of g * wx; then
    //      hist[b] += T[b] * wy, rows ascending.  Votes into cells outside the grid are never formed (hog.c:713-723).
    //      Bilinear orientations (hog.c:706-714 scale wx AND wy by the orientation weight w_o): T[b] += (g * (wx * w_o)) * w_o,
    //      which with w_o = 1 is the sum above.
    const int ncell = nhx * nhy;
    if (tid < ncell) {
        const int cyl = tid / nhx, cxl = tid - cyl * nhx;
        const int ci = hx0 + cxl, cj = hy0 + cyl;
        // the pixels of the frame that vote (interior, or every one for POLAR) into column ci / row cj: a contiguous run of
        // staged coordinates
        int xlo = span, xhi = -1, ylo = span, yhi = -1;
        for (int i = max(E, E - ox0); i <= min(span - 1 - E, W - 1 - E - ox0); ++i)
            if (s_bx[i] == ci || s_bx[i] == ci - 1) { xlo = min(xlo, i); xhi = i; }
        for (int i = max(E, E - oy0); i <= min(span - 1 - E, H - 1 - E - oy0); ++i)
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
                // axis, which the reference does not vote; or a polar pixel with a modulus <= 0 or a non-finite ho
                if (b < 0) continue;
                const float w = s_bx[x] == ci ? s_wx1[x] : s_wx2[x];
                float* q = T + b * hs;
                if constexpr (BIL) {
                    const float wo1 = s_w1[y * span + x], wo0 = __fsub_rn(1.f, wo1);
                    *q = __fadd_rn(*q, __fmul_rn(__fmul_rn(gp[x], __fmul_rn(w, wo0)), wo0));
                    const int b1 = s_bin1[y * span + x];
                    if (b1 >= 0) {
                        float* q1 = T + b1 * hs;
                        *q1 = __fadd_rn(*q1, __fmul_rn(__fmul_rn(gp[x], __fmul_rn(w, wo1)), wo1));
                    }
                } else {
                    *q = __fadd_rn(*q, __fmul_rn(gp[x], w));
                }
            }
            const float wy = s_by[y] == cj ? s_wy1[y] : s_wy2[y];
            for (int b = 0; b < 2 * K; ++b) {
                float* h = hist + b * hs;
                *h = __fadd_rn(*h, __fmul_rn(T[b * hs], wy));
            }
        }
        // ---- S4: undirected cell energy (hog.c:875-890)
        s_energy[tid] = hog_cell_energy(hist, hs, K);
    }
    __syncthreads();

    // ---- S5-S7: one thread per output cell: the four block factors in double (hog.c:930-982), normalise, clamp at 0.2 and
    //      project (hog.c:985-1044), texture dims summed in ascending k (hog.c:1046-1053).  Planar store: a warp writes runs of
    //      tw consecutive floats of each feature plane.
    if (tid < tw * th) {
        const int yl = tid / tw;
        const int x = tx0 + tid - yl * tw, y = ty0 + yl;
        const int c = (x - hx0) + (y - hy0) * nhx;
        const long long plane = (long long)hogW * hogH;
        float* __restrict__ out = a.out + (a.out_offset ? a.out_offset[f] : (long long)f * a.out_stride) + (long long)y * hogW + x;
        double fac[4];
        hog_cell_factors(s_energy, nhx, hx0, hy0, hogW, hogH, x, y, fac);
        hog_cell_features(fac, s_hist + c, hs, K, a.variant, [=](int d, float v) { out[d * plane] = v; });
    }
}

template <int KT>
__global__ void __launch_bounds__(kDenseThreads) hog_dense_kernel(const __grid_constant__ DenseArgs a, const __grid_constant__ CUtensorMap map)
{
    hog_dense_cta<KT, true, uint8_t, false>(a, &map);
}

template <int KT, class Pix, bool BIL>
__global__ void __launch_bounds__(kDenseThreads, 2) hog_images_kernel(const __grid_constant__ ImageArgs a)
{
    hog_dense_cta<KT, false, Pix, BIL>(a, nullptr);
}

template <int KT, bool BIL>
__global__ void __launch_bounds__(kDenseThreads, 2) hog_polar_kernel(const __grid_constant__ PolarArgs a)
{
    hog_dense_cta<KT, false, float, BIL>(a, nullptr);
}

typedef void (*ImagesKernel)(ImageArgs);
typedef void (*PolarKernel)(PolarArgs);

template <class Pix, bool BIL>
ImagesKernel images_kernel(int K)
{
    return K == 4 ? hog_images_kernel<4, Pix, BIL> : K == 9 ? hog_images_kernel<9, Pix, BIL> : hog_images_kernel<0, Pix, BIL>;
}

ImagesKernel images_kernel(int dtype, bool bil, int K)
{
    return dtype == SD_HOG_U8 ? (bil ? images_kernel<uint8_t, true>(K) : images_kernel<uint8_t, false>(K))
                              : (bil ? images_kernel<float, true>(K) : images_kernel<float, false>(K));
}

template <bool BIL>
PolarKernel polar_kernel(int K)
{
    return K == 4 ? hog_polar_kernel<4, BIL> : K == 9 ? hog_polar_kernel<9, BIL> : hog_polar_kernel<0, BIL>;
}

// Tile side of hog_images_kernel.  Nearest-bin: dense_tile's, as the 8-bit grey kernel.  Bilinear orientations hold 10 B per
// pixel, twice the nearest-bin figure, so at dense_tile's side a CTA of cs 8 takes 120 KB and only one fits on an SM, with
// (T + 2)^2 = 121 threads busy in S3.  There the tile with the most output cells in flight per SM, resident CTAs x T^2, wins
// (one thread per histogram cell walks all of its cell's pixels in S3, so a CTA takes about as long at any T): measured 25-35 %
// faster at cs 4 and 8 (DESIGN 4.9).  The same rule for nearest-bin frames chose T = 12 at two CTAs over T = 9 at three at
// cs 8, which measured 8-13 % slower.  hog_polar_kernel keeps the same per-pixel state and takes the same rule.
template <class Args>
int images_tile(void (*kern)(Args), int cs, int K, bool bil)
{
    if (!bil) return dense_tile(cs);
    int best = 1, most = 0;
    for (int t = 1; t <= kDenseMaxTile; ++t) {
        const int bytes = dense_smem_layout(cs * (t + 3) + 4, 0, K, dense_cells(t), bil).total;
        if (bytes > 227 * 1024) break;
        int ctas = 0;
        if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes) != cudaSuccess ||
            cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas, kern, kDenseThreads, bytes) != cudaSuccess)
            break;
        if (ctas * t * t > most) { most = ctas * t * t; best = t; }
    }
    return best;
}

// the rules of vl_hog_prepare_buffers (hog.c:542-548) and of this implementation's range, shared by both entry points
bool dense_shape(int width, int height, int cs, int K, int variant, int* hog_w, int* hog_h, int* dd)
{
    if (sd_hog_check_config(nullptr, __func__, variant, K, cs)) return false;
    if (width <= 3 || height <= 3) return false;
    const int w = (width + cs / 2) / cs, h = (height + cs / 2) / cs;
    if (w <= 0 || h <= 0) return false;
    *hog_w = w;
    *hog_h = h;
    *dd = sd_hog_dd(K, variant);
    return true;
}

// the configuration of hog_dense_kernel (sd_hog_dense, sd_hog_pyramid): tile, staged region and orientation table
DenseArgs dense_args(const uint8_t* images, const sd_frame* frames, int cs, int K, int variant, int dd, float* out,
                     const int64_t* out_offset)
{
    DenseArgs a;
    memset(&a, 0, sizeof(a));
    a.images = images;
    a.frames = frames;
    a.out = out;
    a.out_offset = out_offset;
    a.variant = variant; a.cs = cs; a.K = K; a.dd = dd;
    a.tile = dense_tile(cs);
    a.span = cs * (a.tile + 4) + 2;
    a.pitch = dense_align(a.span + 15, 16);
    hog_orientations(K, a.orient);   // hog.c:195-204
    return a;
}

typedef void (*DenseKernel)(DenseArgs, CUtensorMap);

DenseKernel dense_kernel(int K)
{
    return K == 4 ? hog_dense_kernel<4> : K == 9 ? hog_dense_kernel<9> : hog_dense_kernel<0>;
}

// a frame descriptor of sd_hog_dense_images: the size rule and non-negative offset and strides
bool image_ok(const sd_hog_image& d, int cs, int K, int variant, int* hog_w, int* hog_h, int* dd)
{
    return dense_shape(d.width, d.height, cs, K, variant, hog_w, hog_h, dd) && d.offset >= 0 && d.row_stride >= 0 &&
           d.pixel_stride >= 0 && d.channel_stride >= 0;
}

// The descriptor table of a batch, read back once: every frame passes the rules of its entry point (fn, for the messages),
// *max_w x *max_h cells cover the largest frame, and frames of different sizes need one output offset per frame (offsets).
template <class Frame>
int read_frames(sd_ctx* ctx, const char* fn, const Frame* d_frames, int count, int cs, int K, int variant, bool offsets,
                int* max_w, int* max_h, int* dd)
{
    std::vector<Frame> fr;
    if (const int rc = sd_fetch_table(ctx, d_frames, count, fr)) return rc;
    bool uniform = true;
    for (int i = 0; i < count; ++i) {
        const Frame& d = fr[i];
        int w, h;
        if constexpr (std::is_same<Frame, sd_frame>::value) {   // sd_hog_dense
            if (!dense_shape(d.width, d.height, cs, K, variant, &w, &h, dd))
                return sd_fail(ctx, SD_ERR_INVALID, "%s: frame %d is %d x %d: frames must be wider and taller than 3 px and at "
                               "least half a cell", fn, i, d.width, d.height);
            if (d.row_stride < d.width || d.offset < 0) return sd_fail(ctx, SD_ERR_INVALID, "%s: bad frame descriptor", fn);
        } else if (!image_ok(d, cs, K, variant, &w, &h, dd)) {   // sd_hog_dense_images
            return sd_fail(ctx, SD_ERR_INVALID, "%s: frame %d (%d x %d) breaks the size rule (wider and taller than 3 px, at least "
                           "half a cell) or has a negative offset or stride", fn, i, d.width, d.height);
        }
        *max_w = std::max(*max_w, w);
        *max_h = std::max(*max_h, h);
        uniform = uniform && d.width == fr[0].width && d.height == fr[0].height;
    }
    if (!offsets && !uniform) return sd_fail(ctx, SD_ERR_INVALID, "%s: frames of different sizes need one output offset per frame", fn);
    return SD_OK;
}

// Queues kern over the batch with smem bytes of shared memory: one launch per slice of at most 65,535 frames (the grid's z
// limit), a.frame0 the slice's first frame, and a grid of tiles of a.tile cells over the largest frame's max_w x max_h cells.
template <class Args, class... Maps>
int launch_dense(sd_ctx* ctx, const char* fn, const char* name, void (*kern)(Args, Maps...), Args a, int count, int max_w,
                 int max_h, int smem, const Maps&... maps)
{
    if (smem > 227 * 1024) return sd_fail(ctx, SD_ERR_INVALID, "%s: dense HOG configuration needs more than 227 KB of shared memory", fn);
    SD_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    const unsigned gx = (unsigned)sd_div_up(max_w, a.tile), gy = (unsigned)sd_div_up(max_h, a.tile);
    for (int f0 = 0; f0 < count; f0 += 65535) {
        a.frame0 = f0;
        const dim3 grid(gx, gy, (unsigned)std::min(count - f0, 65535));
        kern<<<grid, kDenseThreads, smem, ctx->stream>>>(a, maps...);
        SD_LAUNCH_CHECK(ctx, name);
    }
    return SD_OK;
}

// ---- the pyramid (sd_hog_pyramid, sd_hog_pyramid_images, sd_hog_pyramid_float): every level of every frame resized into
//      scratch, each channel on its own by the rule of the frames' type (hog_resize_tap, hog_resize_tap_f32) and written
//      interleaved ((H, W, C) elements of that type, rows at a pitch of C * w elements rounded up to 16 bytes), then all of them
//      through one dense pass.  The batch is cut into slices whose levels fit kPyramidSliceBytes (one frame at least), so the
//      scratch is bounded by the slice, not by the batch.
constexpr int kResizeW = 64, kResizeH = 16, kResizeThreads = 256;   // output pixels of a resize CTA
constexpr size_t kPyramidSliceBytes = size_t(64) << 20;
constexpr double kPyramidMaxSide = 1 << 28;                          // px per side of a level

// level size of a width x height frame at scale (both in double, as cv::Size(round(width * scale))): false for a scale that
// is not finite or lies outside (0, 4], or a frame or level outside [1, 2^28] px per side
bool pyramid_level(int width, int height, double scale, int* lw, int* lh)
{
    if (!(scale > 0.0 && scale <= 4.0) || width < 1 || height < 1) return false;   // NaN fails the first test
    const double w = floor((double)width * scale + 0.5), h = floor((double)height * scale + 0.5);
    if (w > kPyramidMaxSide || h > kPyramidMaxSide) return false;
    *lw = (int)w;
    *lh = (int)h;
    return true;
}

struct PyrImageLevel {
    long long src;               // element offset of the frame's pixel (0, 0, 0) from the batch's data
    long long rs, ps, chs;       // the frame's row, pixel and channel strides in elements
    long long dst;               // byte offset of the level from the scratch
    int W, H;                    // the frame
    int w, h, pitch;             // the level: size and row stride in bytes
    int tile0, tiles_x;          // the level's first CTA of the resize launch, and its CTAs per row of tiles
    int slot;                    // the level's index in the caller's output offsets
};

struct ResizeImagesArgs {
    const void* images;
    uint8_t* scratch;
    const PyrImageLevel* levels;
    int count, channels;
    const int64_t* out_offset;   // the caller's, per slot
    int64_t* level_offset;       // per level: the caller's offset of its slot (the dense kernel's out_offset)
    const int4* rect;            // kRect: per level, the origin (x, y) of its W x H source rectangle and the frame's size (z, w)
};

// One CTA per kResizeW x kResizeH pixel tile of one level: the taps of its columns and rows once, then cv::resize's two passes
// for every channel of every pixel with the channel fastest, so that a warp writes consecutive elements of the level, the
// source read through L1.  A level of the frame's own size is copied.  kC = 1: 8-bit frames of one channel, contiguous pixels
// (pixel stride 1), frames and levels of fewer than 2^31 bytes, the grey pyramid's: the pixel loop is spared two divisions by
// a run-time count and takes every offset in 32 bits.  kC = 0: any channel count, strides and sizes.  kRect (the box crops of
// sd_hog_box_scores and sd_hog_box_scores_images): the level's W x H source is the rectangle at rect[level].(x, y) of a rect.z x
// rect.w frame, its pixels outside the frame 0 (copyMakeBorder BORDER_CONSTANT); it writes no level offsets.  A float
// rectangle's pixel outside the frame is a tap holding +0.0f, read and multiplied like any other.
template <class T, int kC, bool kRect = false>
__global__ void __launch_bounds__(kResizeThreads) hog_pyramid_resize_images_kernel(const __grid_constant__ ResizeImagesArgs a)
{
    static_assert(kC != 1 || std::is_same<T, uint8_t>::value, "kC = 1 is 8-bit grey");
    constexpr bool f32 = std::is_same<T, float>::value;
    __shared__ int s_sx[kResizeW], s_xw[kResizeW], s_y0[kResizeH], s_y1[kResizeH], s_yw[kResizeH];
    const int b = blockIdx.x, tid = threadIdx.x, C = kC > 0 ? kC : a.channels;
    const int lo = sd_find_last_le(0, a.count - 1, b, [&](int i) { return a.levels[i].tile0; });
    const PyrImageLevel L = a.levels[lo];
    const int t = b - L.tile0, ty = t / L.tiles_x;
    const int x0 = (t - ty * L.tiles_x) * kResizeW, y0 = ty * kResizeH;
    if (!kRect && t == 0 && tid == 0) a.level_offset[lo] = a.out_offset[L.slot];
    const T* __restrict__ src = static_cast<const T*>(a.images) + L.src;
    uint8_t* __restrict__ dst = a.scratch + L.dst;
    const bool copy = L.w == L.W && L.h == L.H;
    if (!copy) {
        if (tid < kResizeW) {
            if (x0 + tid < L.w) {
                const HogResizeTap r = f32 ? hog_resize_tap_f32(x0 + tid, L.w, L.W) : hog_resize_tap(x0 + tid, L.w, L.W);
                s_sx[tid] = r.sx;
                s_xw[tid] = r.xw;
            }
        } else if (tid < kResizeW + kResizeH) {
            const int i = tid - kResizeW;
            if (y0 + i < L.h) {
                const HogResizeTap r = f32 ? hog_resize_tap_f32(y0 + i, L.h, L.H) : hog_resize_tap(y0 + i, L.h, L.H);
                s_y0[i] = r.y0;
                s_y1[i] = r.y1;
                s_yw[i] = r.yw;
            }
        }
        __syncthreads();
    }
    const int row = kResizeW * C;
    for (int i = tid; i < row * kResizeH; i += kResizeThreads) {
        const int r = i / row, j = i - r * row;
        const int c = j / C, ch = j - c * C;
        const int x = x0 + c, y = y0 + r;
        if (x >= L.w || y >= L.h) continue;
        const T* s = src + ch * L.chs;
        if constexpr (kRect) {
            using V = typename std::conditional<f32, float, int>::type;
            const int4 R = a.rect[lo];
            const auto px = [&](int u, int v) -> V {   // pixel (u, v) of the rectangle
                const long long fx = (long long)R.x + u, fy = (long long)R.y + v;
                if (!(fx >= 0 && fx < R.z && fy >= 0 && fy < R.w)) return V(0);
                return (V)__ldg(s + fy * L.rs + (kC == 1 ? fx : fx * L.ps));
            };
            V v;
            if (copy) {
                v = px(x, y);
            } else if constexpr (f32) {
                const int sx = s_sx[c];
                const float fx = __int_as_float(s_xw[c]);
                const auto row_at = [&](int yy) {   // hog_resize_row_f32 of rectangle row yy
                    const float t = __fmul_rn(px(sx, yy), __fsub_rn(1.f, fx));
                    return sx == L.W - 1 ? t : __fadd_rn(t, __fmul_rn(px(sx + 1, yy), fx));
                };
                v = hog_resize_out_f32(__int_as_float(s_yw[r]), row_at(s_y0[r]), row_at(s_y1[r]));
            } else {
                const int sx = s_sx[c], sx1 = min(sx + 1, L.W - 1);
                const int ax = (short)s_xw[c], bx = s_xw[c] >> 16;
                v = hog_resize_out(s_yw[r], px(sx, s_y0[r]) * ax + px(sx1, s_y0[r]) * bx, px(sx, s_y1[r]) * ax + px(sx1, s_y1[r]) * bx);
            }
            reinterpret_cast<T*>(dst + (long long)y * L.pitch)[(long long)x * C + ch] = (T)v;
        } else if constexpr (f32) {
            float v;
            if (copy) {
                v = __ldg(s + y * L.rs + x * L.ps);   // a bit copy: no arithmetic touches the value
            } else {
                const int sx = s_sx[c];
                const float fx = __int_as_float(s_xw[c]);
                v = hog_resize_out_f32(__int_as_float(s_yw[r]), hog_resize_row_f32(s + s_y0[r] * L.rs, L.ps, sx, fx, L.W - 1),
                                       hog_resize_row_f32(s + s_y1[r] * L.rs, L.ps, sx, fx, L.W - 1));
            }
            reinterpret_cast<float*>(dst + (long long)y * L.pitch)[x * C + ch] = v;
        } else {
            using Off = typename std::conditional<kC == 1, int, long long>::type;   // offsets within the frame and the level
            const Off rs = (Off)L.rs, ps = kC == 1 ? 1 : (Off)L.ps;
            int v;
            if (copy) {
                v = __ldg(s + (Off)y * rs + x * ps);
            } else {
                const int sx = s_sx[c], sx1 = min(sx + 1, L.W - 1);   // a clamped tap has zero weight
                const int ax = (short)s_xw[c], bx = s_xw[c] >> 16;
                const uint8_t* r0 = s + (Off)s_y0[r] * rs;
                const uint8_t* r1 = s + (Off)s_y1[r] * rs;
                v = hog_resize_out(s_yw[r], (int)__ldg(r0 + sx * ps) * ax + (int)__ldg(r0 + sx1 * ps) * bx,
                                   (int)__ldg(r1 + sx * ps) * ax + (int)__ldg(r1 + sx1 * ps) * bx);
            }
            dst[(Off)y * L.pitch + x * C + ch] = (uint8_t)v;
        }
    }
}

// Where hog_box_levels_kernel finds frame f: a grey batch's sd_frame table, an sd_hog_images table, or equally sized frames
// (frame, offset advanced by image_stride elements per frame).
struct BoxFrameTable {
    const sd_frame* grey_frames;
    const sd_hog_image* frames;
    sd_hog_image frame;
    long long image_stride;
};

// The level of box i of sd_hog_box_crops: its context rectangle of its frame, resized to the crop size; a box whose d_ok byte is
// 0 takes the 1 x 1 rectangle at (0, 0).  One thread per box.
__global__ void hog_box_levels_kernel(const BoxFrameTable t, const int32_t* __restrict__ box_frame, const int32_t* __restrict__ boxes,
                                      const uint8_t* __restrict__ ok, int n, int fw, int fh, int cw, int ch, int pitch, int tiles_x,
                                      int tiles_per_box, PyrImageLevel* __restrict__ levels, int4* __restrict__ rect)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int f = box_frame[i];
    sd_hog_image d;
    if (t.grey_frames) {
        const sd_frame g = t.grey_frames[f];
        d = sd_hog_image{g.width, g.height, g.offset, g.row_stride, 1, 0};
    } else if (t.frames) {
        d = t.frames[f];
    } else {
        d = t.frame;
        d.offset += (long long)f * t.image_stride;
    }
    int rx = 0, ry = 0, rw = 1, rh = 1;
    if (!ok || ok[i]) sd_box_context(boxes[4 * i], boxes[4 * i + 1], boxes[4 * i + 2], boxes[4 * i + 3], fw, fh, &rx, &ry, &rw, &rh);
    PyrImageLevel L{};
    L.src = d.offset;
    L.rs = d.row_stride; L.ps = d.pixel_stride; L.chs = d.channel_stride;
    L.dst = (long long)i * pitch * ch;
    L.W = rw; L.H = rh;
    L.w = cw; L.h = ch; L.pitch = pitch;
    L.tile0 = i * tiles_per_box; L.tiles_x = tiles_x;
    L.slot = i;
    levels[i] = L;
    rect[i] = make_int4(rx, ry, d.width, d.height);
}

// The scratch of one slice: [levels (bytes, 16-byte aligned) | level table | the dense kernel's descriptors | per-level
// output offsets], the two tables uploaded.  Returns the scratch, or nullptr (the context holds the error).
template <class Desc>
uint8_t* pyramid_scratch(sd_ctx* ctx, long long bytes, const PyrImageLevel* levels, const std::vector<Desc>& desc,
                         PyrImageLevel** d_lv, Desc** d_desc, int64_t** d_off)
{
    const size_t n = desc.size();
    const size_t pix = sd_round16((size_t)bytes), lv_bytes = sizeof(PyrImageLevel) * n, desc_bytes = sizeof(Desc) * n;
    uint8_t* ws = static_cast<uint8_t*>(sd_workspace(ctx, SD_WS_PYRAMID, pix + lv_bytes + desc_bytes + sizeof(int64_t) * n));
    if (!ws) return nullptr;
    *d_lv = reinterpret_cast<PyrImageLevel*>(ws + pix);
    *d_desc = reinterpret_cast<Desc*>(ws + pix + lv_bytes);
    *d_off = reinterpret_cast<int64_t*>(ws + pix + lv_bytes + desc_bytes);
    if (sd_check_cuda(ctx, cudaMemcpyAsync(*d_lv, levels, lv_bytes, cudaMemcpyHostToDevice, ctx->stream), "pyramid levels") ||
        sd_check_cuda(ctx, cudaMemcpyAsync(*d_desc, desc.data(), desc_bytes, cudaMemcpyHostToDevice, ctx->stream), "pyramid levels"))
        return nullptr;
    return ws;
}

// Queues the levels of a pyramid one slice of whole frames at a time, the frames' levels fitting kPyramidSliceBytes (one
// frame at least).  lv: every non-empty level, frame f's at lv[first[f] .. first[f + 1]).  Per slice it places the levels in
// scratch (dst, tile0), uploads them with the dense kernel's descriptor desc_of(level) of each, resizes them in one launch and
// calls dense(n, scratch, d_desc, d_off, max_w, max_h): its level count, the descriptors and per-level output offsets in
// scratch, and its largest cell grid.
template <class DescOf, class Dense>
int pyramid_slices(sd_ctx* ctx, const char* fn, const HogPyramidFrames& src, std::vector<PyrImageLevel>& lv,
                   const std::vector<int>& first, int count, int cell_size, const int64_t* d_out_offset, DescOf desc_of, Dense dense)
{
    using Desc = decltype(desc_of(lv[0]));
    for (int f0 = 0; f0 < count;) {
        size_t bytes = 0;
        int f1 = f0;
        for (; f1 < count; ++f1) {
            size_t fb = 0;
            for (int l = first[f1]; l < first[f1 + 1]; ++l) fb += (size_t)lv[l].pitch * lv[l].h;
            if (f1 > f0 && bytes + fb > kPyramidSliceBytes) break;
            bytes += fb;
        }
        const int l0 = first[f0], n = first[f1] - l0;
        f0 = f1;
        if (n == 0) continue;
        long long pos = 0;
        int tiles = 0, max_w = 0, max_h = 0;
        bool grey = src.dtype == SD_HOG_U8 && src.channels == 1;   // hog_pyramid_resize_images_kernel's kC = 1
        std::vector<Desc> desc(n);
        for (int i = 0; i < n; ++i) {
            PyrImageLevel& L = lv[l0 + i];
            L.dst = pos;
            L.tile0 = tiles;
            if ((long long)tiles + (long long)L.tiles_x * sd_div_up(L.h, kResizeH) > INT_MAX)
                return sd_fail(ctx, SD_ERR_INVALID, "%s: level too large", fn);
            tiles += L.tiles_x * sd_div_up(L.h, kResizeH);
            pos += (long long)L.pitch * L.h;
            max_w = std::max(max_w, (L.w + cell_size / 2) / cell_size);
            max_h = std::max(max_h, (L.h + cell_size / 2) / cell_size);
            desc[i] = desc_of(L);
            grey = grey && L.ps == 1 && (long long)(L.H - 1) * L.rs + L.W <= INT_MAX && (long long)L.pitch * L.h <= INT_MAX;
        }
        PyrImageLevel* d_lv;
        Desc* d_desc;
        int64_t* d_off;
        uint8_t* ws = pyramid_scratch(ctx, pos, lv.data() + l0, desc, &d_lv, &d_desc, &d_off);
        if (!ws) return SD_ERR_CUDA;

        ResizeImagesArgs r;
        r.images = src.data;
        r.scratch = ws;
        r.levels = d_lv;
        r.count = n;
        r.channels = src.channels;
        r.out_offset = d_out_offset;
        r.level_offset = d_off;
        const auto resize = grey ? hog_pyramid_resize_images_kernel<uint8_t, 1>
                            : src.dtype == SD_HOG_F32 ? hog_pyramid_resize_images_kernel<float, 0> : hog_pyramid_resize_images_kernel<uint8_t, 0>;
        resize<<<(unsigned)tiles, kResizeThreads, 0, ctx->stream>>>(r);
        SD_LAUNCH_CHECK(ctx, "hog_pyramid_resize_images_kernel");
        if (const int rc = dense(n, ws, d_desc, d_off, max_w, max_h)) return rc;
    }
    return SD_OK;
}

// The argument checks the pyramid entry points share, in their order (fn names the entry point in messages): channels,
// orientation assignment, configuration, scales, frame count, data, alignment of float frames and the number of levels.
// A call without frames passes once its count is checked.
#define PYR_REQUIRE(cond, msg)                                                         \
    do {                                                                               \
        if (!(cond)) return sd_fail(ctx, SD_ERR_INVALID, "%s: %s", fn, msg);           \
    } while (0)
int pyramid_check(sd_ctx* ctx, const char* fn, int channels, int bilinear_orientations, int cell_size, int num_bins, int variant,
                  const double* h_scales, int num_scales, int count, const void* d_data, bool f32)
{
    PYR_REQUIRE(channels >= 1 && channels <= kDenseMaxChannels, "channels must be in [1,16]");
    PYR_REQUIRE(bilinear_orientations == 0 || bilinear_orientations == 1, "bilinear_orientations must be 0 or 1");
    if (const int rc = sd_hog_check_config(ctx, fn, variant, num_bins, cell_size)) return rc;
    PYR_REQUIRE(num_scales >= 1, "num_scales must be at least 1");
    for (int s = 0; s < num_scales; ++s)
        PYR_REQUIRE(h_scales[s] > 0.0 && h_scales[s] <= 4.0, "every scale must be finite and in (0, 4]");
    PYR_REQUIRE(count >= 0, "negative frame count");
    if (count == 0) return SD_OK;
    PYR_REQUIRE(d_data, "null argument");
    PYR_REQUIRE(!f32 || sd_aligned(d_data, 4), "float frames must be 4-byte aligned");
    PYR_REQUIRE((long long)count * num_scales <= INT_MAX, "too many levels");
    return SD_OK;
}

// contiguous 8-bit grey frames of one size, nearest bins: hog_dense_kernel's frames, whose features it computes bit for bit
// as hog_images_kernel does (sd_hog_dense_images and sd_hog_pyramid_images run it there)
bool grey_batch(const sd_hog_images* images, int bilinear_orientations)
{
    const sd_hog_image& f = images->frame;
    return images->dtype == SD_HOG_U8 && images->channels == 1 && !bilinear_orientations && !images->d_frames &&
           f.pixel_stride == 1 && f.row_stride >= f.width && f.row_stride <= INT_MAX && (images->count == 1 || images->image_stride > 0);
}

// sd_hog_pyramid_images and sd_hog_pyramid_float past their null and dtype checks
int pyramid_images(sd_ctx* ctx, const char* fn, const sd_hog_images* images, const double* h_scales, int num_scales, int cell_size,
                   int num_bins, int variant, int bilinear_orientations, float* d_out, const int64_t* d_out_offset)
{
    if (const int rc = pyramid_check(ctx, fn, images->channels, bilinear_orientations, cell_size, num_bins, variant, h_scales,
                                     num_scales, images->count, images->d_data, images->dtype == SD_HOG_F32))
        return rc;
    if (images->count == 0) return SD_OK;
    HogPyramidFrames fr;
    if (const int rc = sd_hog_read_image_frames(ctx, fn, images, bilinear_orientations, &fr)) return rc;
    return sd_hog_pyramid_frames(ctx, fn, fr, 0, images->count, h_scales, num_scales, cell_size, num_bins, variant, d_out, d_out_offset);
}
#undef PYR_REQUIRE

}  // namespace

size_t sd_hog_box_table_bytes(int n) { return sd_round16(sizeof(PyrImageLevel) * (size_t)n) + sizeof(int4) * (size_t)n; }

int sd_hog_box_crops(sd_ctx* ctx, const BoxFrames& src, const int32_t* d_box_frame, const int32_t* d_boxes, const uint8_t* d_ok,
                     int n, int fw, int fh, int cell_size, uint8_t* d_crops, int pitch, void* d_tables)
{
    if (n == 0) return SD_OK;
    const int cw = (fw + 2) * cell_size, ch = (fh + 2) * cell_size;
    const int tiles_x = sd_div_up(cw, kResizeW), tiles_per_box = tiles_x * sd_div_up(ch, kResizeH);
    if ((long long)n * tiles_per_box > INT_MAX) return sd_fail(ctx, SD_ERR_INVALID, "sd_hog_box_scores: too many boxes for one launch");
    PyrImageLevel* levels = static_cast<PyrImageLevel*>(d_tables);
    int4* rect = reinterpret_cast<int4*>(static_cast<uint8_t*>(d_tables) + sd_round16(sizeof(PyrImageLevel) * (size_t)n));
    BoxFrameTable t{};
    if (src.grey) {
        t.grey_frames = src.grey->d_frames;
        t.frame = sd_hog_image{src.grey->width, src.grey->height, 0, src.grey->row_stride, 1, 0};
        t.image_stride = src.grey->image_stride;
    } else {
        t.frames = src.images->d_frames;
        t.frame = src.images->frame;
        t.image_stride = src.images->image_stride;
    }
    hog_box_levels_kernel<<<sd_div_up(n, 128), 128, 0, ctx->stream>>>(t, d_box_frame, d_boxes, d_ok, n, fw, fh, cw, ch, pitch, tiles_x,
                                                                      tiles_per_box, levels, rect);
    SD_LAUNCH_CHECK(ctx, "hog_box_levels_kernel");
    ResizeImagesArgs r;
    memset(&r, 0, sizeof(r));
    r.images = src.data();
    r.scratch = d_crops;
    r.levels = levels;
    r.count = n;
    r.channels = src.channels();
    r.rect = rect;
    // kC = 1 for frames whose pixels are known to be contiguous bytes of one channel: a grey batch, or such an sd_hog_images batch
    // of equally sized frames
    const bool grey = src.grey || (src.dtype() == SD_HOG_U8 && src.channels() == 1 && !t.frames && t.frame.pixel_stride == 1);
    const auto resize = grey ? hog_pyramid_resize_images_kernel<uint8_t, 1, true>
                        : src.dtype() == SD_HOG_F32 ? hog_pyramid_resize_images_kernel<float, 0, true>
                                                    : hog_pyramid_resize_images_kernel<uint8_t, 0, true>;
    resize<<<(unsigned)(n * tiles_per_box), kResizeThreads, 0, ctx->stream>>>(r);
    SD_LAUNCH_CHECK(ctx, "hog_pyramid_resize_images_kernel");
    return SD_OK;
}

int sd_hog_read_grey_frames(sd_ctx* ctx, const char* fn, const sd_image_batch* images, HogPyramidFrames* out)
{
    const int count = images->count;
    std::vector<sd_frame> fr;
    if (images->d_frames) {
        if (const int rc = sd_fetch_table(ctx, images->d_frames, count, fr)) return rc;
    } else {
        if (!(count == 1 || images->image_stride > 0)) return sd_fail(ctx, SD_ERR_INVALID, "%s: bad strides", fn);
        fr.assign(count, sd_frame{images->width, images->height, images->row_stride, 0, 0});
        for (int i = 0; i < count; ++i) fr[i].offset = (int64_t)i * images->image_stride;
    }
    out->data = images->d_data;
    out->dtype = SD_HOG_U8;
    out->channels = 1;
    out->bilinear = 0;
    out->grey_kernel = 1;
    out->frames.resize(count);
    for (int f = 0; f < count; ++f) {
        const sd_frame& d = fr[f];
        if (d.width < 1 || d.height < 1 || d.row_stride < d.width || d.offset < 0)
            return sd_fail(ctx, SD_ERR_INVALID, "%s: frame %d (%d x %d, row stride %d, offset %lld) is not a frame", fn, f, d.width,
                           d.height, d.row_stride, (long long)d.offset);
        out->frames[f] = sd_hog_image{d.width, d.height, d.offset, d.row_stride, 1, 0};
    }
    return SD_OK;
}

int sd_hog_read_image_frames(sd_ctx* ctx, const char* fn, const sd_hog_images* images, int bilinear_orientations, HogPyramidFrames* out)
{
    const int count = images->count;
    std::vector<sd_hog_image>& fr = out->frames;
    if (images->d_frames) {
        if (const int rc = sd_fetch_table(ctx, images->d_frames, count, fr)) return rc;
    } else {
        if (images->image_stride < 0) return sd_fail(ctx, SD_ERR_INVALID, "%s: negative image stride", fn);
        fr.assign(count, images->frame);
        for (int i = 0; i < count; ++i) fr[i].offset += (int64_t)i * images->image_stride;
    }
    for (int f = 0; f < count; ++f) {
        const sd_hog_image& d = fr[f];
        if (d.width < 1 || d.height < 1 || d.offset < 0 || d.row_stride < 0 || d.pixel_stride < 0 || d.channel_stride < 0)
            return sd_fail(ctx, SD_ERR_INVALID, "%s: frame %d (%d x %d) is smaller than 1 x 1 or has a negative offset or stride",
                           fn, f, d.width, d.height);
    }
    out->data = images->d_data;
    out->dtype = images->dtype;
    out->channels = images->channels;
    out->bilinear = bilinear_orientations;
    out->grey_kernel = grey_batch(images, bilinear_orientations);
    return SD_OK;
}

int sd_hog_pyramid_frames(sd_ctx* ctx, const char* fn, const HogPyramidFrames& src, int f0, int f1, const double* h_scales,
                          int num_scales, int cell_size, int num_bins, int variant, float* d_out, const int64_t* d_out_offset)
{
    const int C = src.channels, es = src.dtype == SD_HOG_F32 ? 4 : 1, count = f1 - f0;
    // every non-empty level of every frame, in the order of the caller's slots
    std::vector<PyrImageLevel> lv;
    std::vector<int> first(count + 1, 0);
    for (int i = 0; i < count; ++i) {
        const int f = f0 + i;
        const sd_hog_image& d = src.frames[f];
        first[i] = (int)lv.size();
        for (int s = 0; s < num_scales; ++s) {
            PyrImageLevel L{};
            int hw, hh, dd;
            if (!pyramid_level(d.width, d.height, h_scales[s], &L.w, &L.h))
                return sd_fail(ctx, SD_ERR_INVALID, "%s: frame %d at scale %g is larger than 2^28 px per side", fn, f, h_scales[s]);
            if (!dense_shape(L.w, L.h, cell_size, num_bins, variant, &hw, &hh, &dd)) continue;
            if ((long long)L.w * C * es > INT_MAX - 15) return sd_fail(ctx, SD_ERR_INVALID, "%s: frame %d: level too large", fn, f);
            L.src = d.offset;
            L.rs = d.row_stride; L.ps = d.pixel_stride; L.chs = d.channel_stride;
            L.W = d.width; L.H = d.height;
            L.pitch = dense_align(L.w * C * es, 16);
            L.tiles_x = sd_div_up(L.w, kResizeW);
            L.slot = i * num_scales + s;
            lv.push_back(L);
        }
    }
    first[count] = (int)lv.size();
    if (lv.empty()) return SD_OK;

    const int dd = sd_hog_dd(num_bins, variant);
    if (src.grey_kernel) {   // sd_frame descriptors, staged by the load loop: the levels differ in size
        DenseArgs a = dense_args(nullptr, nullptr, cell_size, num_bins, variant, dd, d_out, nullptr);
        const DenseSmem lay = dense_smem_layout(a.span, a.pitch, num_bins, dense_cells(a.tile));
        CUtensorMap map;                             // not read
        memset(&map, 0, sizeof(map));
        return pyramid_slices(
            ctx, fn, src, lv, first, count, cell_size, d_out_offset,
            [](const PyrImageLevel& L) { return sd_frame{L.w, L.h, L.pitch, 0, L.dst}; },
            [&](int n, uint8_t* ws, const sd_frame* d_desc, const int64_t* d_off, int max_w, int max_h) {
                a.images = ws;
                a.frames = d_desc;
                a.out_offset = d_off;
                return launch_dense(ctx, fn, "hog_dense_kernel", dense_kernel(num_bins), a, n, max_w, max_h, lay.total, map);
            });
    }
    const bool bil = src.bilinear != 0;
    const ImagesKernel kern = images_kernel(src.dtype, bil, num_bins);
    ImageArgs a;
    memset(&a, 0, sizeof(a));
    a.channels = C;
    a.out = d_out;
    a.variant = variant; a.cs = cell_size; a.K = num_bins; a.dd = dd;
    a.tile = images_tile(kern, cell_size, num_bins, bil);
    a.span = cell_size * (a.tile + 3) + 4;
    a.pi_k = 3.141592653589793 / (double)num_bins;    // VL_PI / numOrientations (hog.c:677)
    hog_orientations(num_bins, a.orient);
    const DenseSmem lay = dense_smem_layout(a.span, 0, num_bins, dense_cells(a.tile), bil);
    return pyramid_slices(
        ctx, fn, src, lv, first, count, cell_size, d_out_offset,
        [&](const PyrImageLevel& L) { return sd_hog_image{L.w, L.h, L.dst / es, L.pitch / es, C, 1}; },   // elements of the type
        [&](int n, uint8_t* ws, const sd_hog_image* d_desc, const int64_t* d_off, int max_w, int max_h) {
            a.data = ws;
            a.frames = d_desc;
            a.out_offset = d_off;
            return launch_dense(ctx, fn, "hog_images_kernel", kern, a, n, max_w, max_h, lay.total);
        });
}

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
    if (const int rc = sd_hog_check_config(ctx, __func__, variant, num_bins, cell_size)) return rc;
    SD_REQUIRE(ctx, images->count >= 0, "negative frame count");
    const int count = images->count;
    if (count == 0) return SD_OK;
    SD_REQUIRE(ctx, images->d_data, "null argument");

    // frame sizes: the batch's, or the descriptor table read back once (the grid covers the largest frame)
    int max_w = 0, max_h = 0, dd = 0;
    if (images->d_frames) {
        const int rc = read_frames(ctx, __func__, images->d_frames, count, cell_size, num_bins, variant, d_out_offset, &max_w,
                                   &max_h, &dd);
        if (rc) return rc;
    } else {
        SD_REQUIRE(ctx, dense_shape(images->width, images->height, cell_size, num_bins, variant, &max_w, &max_h, &dd),
                   "frames must be wider and taller than 3 px and at least half a cell");
        SD_REQUIRE(ctx, images->row_stride >= images->width && (count == 1 || images->image_stride > 0), "bad strides");
    }

    DenseArgs a = dense_args(images->d_data, images->d_frames, cell_size, num_bins, variant, dd, d_out, d_out_offset);
    a.width = images->width; a.height = images->height; a.row_stride = images->row_stride;
    a.image_stride = images->image_stride;
    a.out_stride = (long long)dd * max_w * max_h;

    // TMA staging: equally sized frames with 16-byte aligned base and pitches (a box of pitch x span bytes per CTA; bytes past
    // the frame's edge are zero-filled and never read)
    CUtensorMap map;
    memset(&map, 0, sizeof(map));
    a.tma = hog_frame_map(images, a.pitch, a.span, &map);

    const DenseSmem lay = dense_smem_layout(a.span, a.pitch, num_bins, dense_cells(a.tile));
    return launch_dense(ctx, __func__, "hog_dense_kernel", dense_kernel(num_bins), a, count, max_w, max_h, lay.total, map);
}

int sd_hog_pyramid_shape(int width, int height, double scale, int cell_size, int num_bins, int variant, int* level_w, int* level_h,
                         int* hog_w, int* hog_h, int* dd)
{
    if (!level_w || !level_h || !hog_w || !hog_h || !dd) return SD_ERR_INVALID;
    if (sd_hog_check_config(nullptr, __func__, variant, num_bins, cell_size)) return SD_ERR_INVALID;
    int lw, lh;
    if (!pyramid_level(width, height, scale, &lw, &lh)) return SD_ERR_INVALID;
    int w = 0, h = 0, d = sd_hog_dd(num_bins, variant);
    if (!dense_shape(lw, lh, cell_size, num_bins, variant, &w, &h, &d)) w = h = 0;   // an empty level
    *level_w = lw;
    *level_h = lh;
    *hog_w = w;
    *hog_h = h;
    *dd = d;
    return SD_OK;
}

int sd_hog_pyramid(sd_ctx* ctx, const sd_image_batch* images, const double* h_scales, int num_scales, int cell_size, int num_bins,
                   int variant, float* d_out, const int64_t* d_out_offset)
{
    if (!ctx) return SD_ERR_INVALID;
    SD_REQUIRE(ctx, images && h_scales && d_out && d_out_offset, "null argument");
    SD_REQUIRE(ctx, !images->d_roi, "a batch with regions of interest has no whole frames");
    if (const int rc = pyramid_check(ctx, __func__, 1, 0, cell_size, num_bins, variant, h_scales, num_scales, images->count,
                                     images->d_data, false))
        return rc;
    if (images->count == 0) return SD_OK;
    HogPyramidFrames fr;
    if (const int rc = sd_hog_read_grey_frames(ctx, __func__, images, &fr)) return rc;
    return sd_hog_pyramid_frames(ctx, __func__, fr, 0, images->count, h_scales, num_scales, cell_size, num_bins, variant, d_out,
                                 d_out_offset);
}

int sd_hog_pyramid_images(sd_ctx* ctx, const sd_hog_images* images, const double* h_scales, int num_scales, int cell_size,
                          int num_bins, int variant, int bilinear_orientations, float* d_out, const int64_t* d_out_offset)
{
    if (!ctx) return SD_ERR_INVALID;
    SD_REQUIRE(ctx, images && h_scales && d_out && d_out_offset, "null argument");
    SD_REQUIRE(ctx, images->dtype == SD_HOG_U8, "dtype must be SD_HOG_U8: the levels are resized by the 8-bit rule");
    return pyramid_images(ctx, __func__, images, h_scales, num_scales, cell_size, num_bins, variant, bilinear_orientations, d_out,
                          d_out_offset);
}

int sd_hog_pyramid_float(sd_ctx* ctx, const sd_hog_images* images, const double* h_scales, int num_scales, int cell_size,
                         int num_bins, int variant, int bilinear_orientations, float* d_out, const int64_t* d_out_offset)
{
    if (!ctx) return SD_ERR_INVALID;
    SD_REQUIRE(ctx, images && h_scales && d_out && d_out_offset, "null argument");
    SD_REQUIRE(ctx, images->dtype == SD_HOG_F32, "dtype must be SD_HOG_F32: the levels are resized by the float rule");
    return pyramid_images(ctx, __func__, images, h_scales, num_scales, cell_size, num_bins, variant, bilinear_orientations, d_out,
                          d_out_offset);
}

int sd_hog_dense_images(sd_ctx* ctx, const sd_hog_images* images, int cell_size, int num_bins, int variant,
                        int bilinear_orientations, float* d_out, const int64_t* d_out_offset)
{
    if (!ctx) return SD_ERR_INVALID;
    SD_REQUIRE(ctx, images && d_out, "null argument");
    SD_REQUIRE(ctx, images->dtype == SD_HOG_U8 || images->dtype == SD_HOG_F32, "dtype must be SD_HOG_U8 or SD_HOG_F32");
    SD_REQUIRE(ctx, images->channels >= 1 && images->channels <= kDenseMaxChannels, "channels must be in [1,16]");
    SD_REQUIRE(ctx, bilinear_orientations == 0 || bilinear_orientations == 1, "bilinear_orientations must be 0 or 1");
    if (const int rc = sd_hog_check_config(ctx, __func__, variant, num_bins, cell_size)) return rc;
    SD_REQUIRE(ctx, images->count >= 0, "negative frame count");
    const int count = images->count;
    if (count == 0) return SD_OK;
    SD_REQUIRE(ctx, images->d_data, "null argument");
    SD_REQUIRE(ctx, images->dtype == SD_HOG_U8 || (reinterpret_cast<uintptr_t>(images->d_data) & 3) == 0,
               "float frames must be 4-byte aligned");

    int max_w = 0, max_h = 0, dd = 0;
    if (images->d_frames) {
        const int rc = read_frames(ctx, __func__, images->d_frames, count, cell_size, num_bins, variant, d_out_offset, &max_w,
                                   &max_h, &dd);
        if (rc) return rc;
    } else {
        SD_REQUIRE(ctx, image_ok(images->frame, cell_size, num_bins, variant, &max_w, &max_h, &dd) && images->image_stride >= 0,
                   "frames must be wider and taller than 3 px and at least half a cell, with non-negative offset and strides");
    }

    // 8-bit grey frames with contiguous rows: the staged (TMA) kernel of sd_hog_dense computes the same features
    if (grey_batch(images, bilinear_orientations)) {
        const sd_hog_image& fr = images->frame;
        sd_image_batch ib{};
        ib.d_data = static_cast<const uint8_t*>(images->d_data) + fr.offset;
        ib.width = fr.width; ib.height = fr.height; ib.row_stride = (int32_t)fr.row_stride;
        ib.image_stride = images->image_stride;
        ib.count = count;
        return sd_hog_dense(ctx, &ib, cell_size, num_bins, variant, d_out, d_out_offset);
    }

    ImageArgs a;
    memset(&a, 0, sizeof(a));
    a.data = images->d_data;
    a.frame = images->frame;
    a.image_stride = images->image_stride;
    a.frames = images->d_frames;
    a.channels = images->channels;
    a.out = d_out;
    a.out_offset = d_out_offset;
    a.out_stride = (long long)dd * max_w * max_h;
    a.variant = variant; a.cs = cell_size; a.K = num_bins; a.dd = dd;
    const bool bil = bilinear_orientations != 0;
    const ImagesKernel kern = images_kernel(images->dtype, bil, num_bins);
    a.tile = images_tile(kern, cell_size, num_bins, bil);
    a.span = cell_size * (a.tile + 3) + 4;
    a.pi_k = 3.141592653589793 / (double)num_bins;    // VL_PI / numOrientations (hog.c:677)
    hog_orientations(num_bins, a.orient);

    const DenseSmem lay = dense_smem_layout(a.span, 0, num_bins, dense_cells(a.tile), bil);
    return launch_dense(ctx, __func__, "hog_images_kernel", kern, a, count, max_w, max_h, lay.total);
}

int sd_hog_dense_polar(sd_ctx* ctx, const sd_hog_polar_fields* fields, int cell_size, int num_bins, int variant, int directed,
                       int bilinear_orientations, float* d_out, const int64_t* d_out_offset)
{
    if (!ctx) return SD_ERR_INVALID;
    SD_REQUIRE(ctx, fields && d_out, "null argument");
    SD_REQUIRE(ctx, directed == 0 || directed == 1, "directed must be 0 or 1");
    SD_REQUIRE(ctx, bilinear_orientations == 0 || bilinear_orientations == 1, "bilinear_orientations must be 0 or 1");
    if (const int rc = sd_hog_check_config(ctx, __func__, variant, num_bins, cell_size)) return rc;
    SD_REQUIRE(ctx, fields->count >= 0, "negative field count");
    const int count = fields->count;
    if (count == 0) return SD_OK;
    SD_REQUIRE(ctx, fields->d_modulus && fields->d_angle, "null argument");
    SD_REQUIRE(ctx, ((reinterpret_cast<uintptr_t>(fields->d_modulus) | reinterpret_cast<uintptr_t>(fields->d_angle)) & 3) == 0,
               "fields must be 4-byte aligned");

    int max_w = 0, max_h = 0, dd = 0;
    if (fields->d_frames) {
        const int rc = read_frames(ctx, __func__, fields->d_frames, count, cell_size, num_bins, variant, d_out_offset, &max_w,
                                   &max_h, &dd);
        if (rc) return rc;
    } else {
        SD_REQUIRE(ctx, image_ok(fields->frame, cell_size, num_bins, variant, &max_w, &max_h, &dd) && fields->image_stride >= 0,
                   "fields must be wider and taller than 3 px and at least half a cell, with non-negative offset and strides");
    }

    PolarArgs a;
    memset(&a, 0, sizeof(a));
    a.modulus = fields->d_modulus;
    a.angle = fields->d_angle;
    a.frame = fields->frame;
    a.image_stride = fields->image_stride;
    a.frames = fields->d_frames;
    a.directed = directed;
    a.out = d_out;
    a.out_offset = d_out_offset;
    a.out_stride = (long long)dd * max_w * max_h;
    a.variant = variant; a.cs = cell_size; a.K = num_bins; a.dd = dd;
    const bool bil = bilinear_orientations != 0;
    const PolarKernel kern = bil ? polar_kernel<true>(num_bins) : polar_kernel<false>(num_bins);
    a.tile = images_tile(kern, cell_size, num_bins, bil);
    a.span = cell_size * (a.tile + 3) + 4;
    a.pi_k = 3.141592653589793 / (double)num_bins;    // angleStep = VL_PI / numOrientations (hog.c:756)

    const DenseSmem lay = dense_smem_layout(a.span, 0, num_bins, dense_cells(a.tile), bil);
    return launch_dense(ctx, __func__, "hog_polar_kernel", kern, a, count, max_w, max_h, lay.total);
}

}  // extern "C"
