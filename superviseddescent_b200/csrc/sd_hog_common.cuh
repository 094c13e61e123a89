// VLFeat's HOG arithmetic, the TMA staging and the frame tensor map, shared by the landmark-patch kernel (sd_hog.cu) and the
// dense whole-frame kernel (sd_hog_dense.cu): one copy, so an fs x fs frame gives bit for bit the features of an fs x fs patch.
#pragma once

#include <cmath>

#include "sd_internal.cuh"

namespace {

// Margin of hog_bin's sector test against the reference's first-maximum rule: a lead of the winning |<g, o_k>| over every other
// one of more than eps |g| cannot change the reference's arg-max or its sign (derivation at hog_bin).
constexpr double kBinLead = 4e-6;

// Orientation directions (hog.c:195-204: host libm cos/sin, as the reference) and the reference bin of a gradient (0, gy):
// vbin[0] for gy > 0, vbin[1] for gy < 0.  ox / oy hold SD_MAX_BINS entries; those past K are zero.  For hog_bin's sector
// search: the directions (bx_j, by_j) = (cos, sin)((2j + 1) pi / 2K) of the sector boundaries inside the open first quadrant
// (j < K / 2), and the margin eps / (2 sin(pi / 2K)) on |cross(b, g)| / |g| that gives a lead of eps.  Every kernel argument
// block carries one (hog_orientations fills it).
struct HogOrient {
    float ox[SD_MAX_BINS], oy[SD_MAX_BINS];   // orientation k: (cos, sin)(k pi / K) in float
    int vbin[2];                              // reference bin of a gradient (0, gy): [0] gy > 0, [1] gy < 0
    float bx[SD_MAX_BINS / 2], by[SD_MAX_BINS / 2], bin_margin;   // hog_bin's sector boundaries and margin
};

inline void hog_orientations(int K, HogOrient& o)
{
    for (int k = 0; k < SD_MAX_BINS; ++k) { o.ox[k] = 0.f; o.oy[k] = 0.f; }
    for (int k = 0; k < K; ++k) {
        const double angle = k * 3.141592653589793 / K;
        o.ox[k] = (float)cos(angle);
        o.oy[k] = (float)sin(angle);
    }
    for (int j = 0; j < SD_MAX_BINS / 2; ++j) {
        const double angle = (2 * j + 1) * 3.141592653589793 / (2 * K);
        o.bx[j] = j < K / 2 ? (float)cos(angle) : 0.f;
        o.by[j] = j < K / 2 ? (float)sin(angle) : 0.f;
    }
    o.bin_margin = (float)(kBinLead / (2.0 * sin(3.141592653589793 / (2 * K))));
    // hog.c:645-672 at gx = 0: ux = +0 and uy = +-1 exactly (the root of gy^2 is exact), so s_k = +-oy_k exactly; the first
    // strict maximum of oy_k > 0 wins, in the lower half-plane when gy < 0 (K = 1: no k has oy_k > 0, bin -1)
    {
        float best = 0.f;
        int bin = -1;
        for (int k = 0; k < K; ++k) if (o.oy[k] > best) { best = o.oy[k]; bin = k; }
        o.vbin[0] = bin;
        o.vbin[1] = bin < 0 ? -1 : bin + K;
    }
}

// ---- one component of the reference's unit gradient (hog.c:645-647): (float)((double)v / max((double)g, 1e-10)).  For
//      g > 1e-10 that is v / g in float: double rounding is innocuous for division when the wide format has >= 2p+2 bits
//      (53 >= 50).  Below, the floor divides in double (tiny float images; g itself may come from a subnormal square).
__device__ __forceinline__ float hog_unit(float v, float g)
{
    return (double)g > 1e-10 ? __fdiv_rn(v, g) : (float)__ddiv_rn((double)v, 1e-10);
}

// ---- the first maximum of |<u, o_k>| in ascending k for a unit gradient u (hog.c:656-672, nearest-bin assignment) ----
__device__ __forceinline__ int hog_bin_unit(const HogOrient& o, int K, float ux, float uy)
{
    float best = 0.f;
    int bin = -1;
#pragma unroll
    for (int k = 0; k < K; ++k) {
        float s = __fadd_rn(__fmul_rn(ux, o.ox[k]), __fmul_rn(uy, o.oy[k]));
        int b = k;
        if (s < 0.f) { s = -s; b += K; }
        if (s > best) { best = s; bin = b; }   // strict >, ascending k
    }
    return bin;
}

// ---- orientation bin of a pixel with a non-zero integer-valued gradient (gx, gy), the reference's float expression
//      verbatim (hog.c:645-672): modulus, normalised gradient (g >= 1, so hog_unit is a float division), then the bin ------
__device__ __forceinline__ int hog_bin_reference(const HogOrient& o, int K, float gx, float gy, float g)
{
    return hog_bin_unit(o, K, __fdiv_rn(gx, g), __fdiv_rn(gy, g));
}

// ---- bilinear orientation assignment (hog.c:656-678): the reference's top-two tracking of |<u, o_k>| verbatim (a score
//      replaces the first only when strictly larger, else the second when strictly larger), then
//        w1 = (float)((double)acosf(min(s0, 1)) / (pi / K)),  w0 = 1 - w1.
//      b1 = -1 when no second score is positive (K = 1 among others); b0 = -1 for a zero gradient.  pi_k is pi / K in double.
//      acos in double rounded to float stays within an ulp of the reference's acosf. ------------------------------------
__device__ __forceinline__ void hog_bins_bilinear(const HogOrient& o, double pi_k, int K, float ux, float uy, int& b0, int& b1,
                                                  float& w1)
{
    float s0 = 0.f, s1 = 0.f;
    b0 = -1;
    b1 = -1;
#pragma unroll
    for (int k = 0; k < K; ++k) {
        float s = __fadd_rn(__fmul_rn(ux, o.ox[k]), __fmul_rn(uy, o.oy[k]));
        int b = k;
        if (s < 0.f) { s = -s; b += K; }
        if (s > s0) { b1 = b0; s1 = s0; b0 = b; s0 = s; }
        else if (s > s1) { b1 = b; s1 = s; }
    }
    const float angle0 = (float)acos((double)fminf(s0, 1.f));
    w1 = (float)__ddiv_rn((double)angle0, pi_k);
}

// ---- orientation bin of an interior pixel without a division, by sector search.  Exactly, the reference's bin (the first
//      strict maximum of |<u, o_k>|, k or k + K by its sign) is the index of the one of 2K angular sectors centred on k pi / K
//      that holds theta = arg g; the sector boundaries are the bisectors (2j + 1) pi / 2K.  Two exact folds on the integers
//      bring g into the quadrant gx >= 0, gy >= 0: the point reflection g -> -g maps bin k to k + K (mod 2K), and the mirror
//      gx -> -gx maps the half-plane sector s (centre s pi / K, s = 0..K) to K - s.  There only the K / 2 boundaries
//      b_j = (cos, sin)((2j + 1) pi / 2K) are left (and pi / 2 for odd K, the gx = 0 axis), so the sector is the count of
//      positive cross products c_j = cross(b_j, g) = r sin(theta - beta_j), r = |g|: at most 8 of them, no indexed loads.
//      Accepting it is exact when the nearest boundary, at angle delta, has |c| > C r, C = eps / (2 sin(pi / 2K)):
//        - the winner's exact |cos(theta - k pi / K)| leads every other one by 2 sin(pi / 2K) sin delta, and is >= sin delta;
//        - u = 2^-24.  s_k (the reference's float dot product of gx/g, gy/g) is within 4u of the exact dot product with the
//          float o_k, which is within u of cos(theta - k pi / K).  c_j (one product, one FMA, float b_j) is within 3u r of
//          r sin(theta - beta_j).  The test m > fl(C g) carries another ~3u relative;
//        - so sin delta > C - 4u, the exact lead exceeds eps - 8u and the reference's lead exceeds eps - 18u > 0
//          (eps = 4e-6 is ~67u).  The winner's |s_k| > sin delta - 5u > 0 fixes the sign, and every c_j, whose |c_j| is at
//          least r sin delta > 3u r, has the right sign: the count is the exact sector.
//      The folds need no symmetry of the float tables, since the exact sectors have it.  m is the least |c_j|: the other
//      boundaries (outside the quadrant) are mirror images at the same or a larger angle.  Pixels that miss the margin, nearly
//      all exactly on a boundary, take the reference expression.  gx = 0 stays in the quadrant: at even K it is the centre of
//      sector K / 2 and the count decides it; at odd K it is a boundary (m = |gx| = 0), common in real patches, and the
//      reference's unit vector there is exactly (0, +-1), so its bin is a function of K and the sign of gy alone
//      (hog_orientations).  g = 0 makes every c_j zero and also misses the margin (bin -1).  tests/test_gpu_hog_orientation.py and tests/test_gpu_hog_sector.py check every (gx, gy) in
//      [-255, 255]^2 at every K in 1..16. -------------------------------------------------------------------------------
__device__ __forceinline__ int hog_bin(const HogOrient& o, int K, int gx, int gy, float g)
{
    const float fx = (float)abs(gx), fy = (float)abs(gy);
    float m = (K & 1) ? fx : INFINITY;   // odd K: |cross((0, 1), g)| against the boundary pi / 2
    int s = 0;
#pragma unroll
    for (int j = 0; j < K / 2; ++j) {
        const float c = fmaf(o.bx[j], fy, -(o.by[j] * fx));
        s += c > 0.f;
        m = fminf(m, fabsf(c));
    }
    if (m > o.bin_margin * g) {
        const bool neg = gy < 0;
        if ((gx < 0) != neg) s = K - s;
        if (neg) s += K;
        return s < 2 * K ? s : 0;
    }
    if (gx == 0) return gy == 0 ? -1 : o.vbin[gy < 0];
    return hog_bin_reference(o, K, (float)gx, (float)gy, g);
}

// ---- spatial binning of pixel coordinate t (hog.c:697-709, rounded as there): h = (t + 0.5) / cs - 0.5, b = floor(h),
//      w2 = h - b, w1 = (float)(1.0 - w2); the pixel adds w1 to cell b and w2 to cell b + 1 ------------------------------
__device__ __forceinline__ void hog_spatial_weight(int t, int cs, int* b, float* w1, float* w2)
{
    const float h = (float)__dadd_rn(__ddiv_rn((double)t + 0.5, (double)cs), -0.5);
    int bb = (int)h;                                  // vl_floor_f, hog.h:52-58
    if (!(h >= 0.f || (float)bb == h)) bb -= 1;
    *b = bb;
    *w2 = __fsub_rn(h, (float)bb);
    *w1 = (float)__dadd_rn(1.0, -(double)*w2);
}

// ---- undirected cell energy (hog.c:875-890) in float: sum over k of (h_k + h_{k+K})^2, h_b = hist[b * stride] -----------
__device__ __forceinline__ float hog_cell_energy(const float* hist, int stride, int K)
{
    float e = 0.f;
    for (int k = 0; k < K; ++k) {
        const float h = __fadd_rn(hist[k * stride], hist[(k + K) * stride]);
        e = __fadd_rn(e, __fmul_rn(h, h));
    }
    return e;
}

// ---- block factor in double (hog.c:930-982) of the 2 x 2 cells at columns xa, xb and rows ya, yb of the energies E (row
//      stride ld; float, or the same values already widened to double).  factor1: n1+n2+n4+n5, factor2: n2+n3+n5+n6,
//      factor3: n4+n5+n7+n8, factor4: n5+n6+n8+n9 ------------------------------------------------------------------------
template <class T>
__device__ __forceinline__ double hog_block_factor(const T* E, int ld, int xa, int xb, int ya, int yb)
{
    double s = (double)E[xa + ya * ld];
    s = __dadd_rn(s, (double)E[xb + ya * ld]);
    s = __dadd_rn(s, (double)E[xa + yb * ld]);
    s = __dadd_rn(s, (double)E[xb + yb * ld]);
    s = __dadd_rn(s, 1e-4);
    return __ddiv_rn(1.0, sqrt(s));
}

// ---- normalise bins k and k + K of a cell (ha, hb) by its four block factors, clamp at 0.2 and project (hog.c:985-1044).
//      keep(f, hc) takes block f's clamped sum, which the texture dims add up over k (hog.c:1046-1053); store(d, v) writes
//      feature dimension d of the cell.
template <class Keep, class Store>
__device__ __forceinline__ void hog_project(const double* fac, double ha, double hb, int k, int K, int variant, Keep keep, Store store)
{
    double sa = 0.0, sb = 0.0, sc = 0.0;
    double hcv[4];
#pragma unroll
    for (int f = 0; f < 4; ++f) {
        double haf = __dmul_rn(fac[f], ha);
        double hbf = __dmul_rn(fac[f], hb);
        double hcf = __dadd_rn(haf, hbf);
        haf = (0.2 < haf) ? 0.2 : haf;
        hbf = (0.2 < hbf) ? 0.2 : hbf;
        hcf = (0.2 < hcf) ? 0.2 : hcf;
        hcv[f] = hcf;
        sa = (f == 0) ? haf : __dadd_rn(sa, haf);
        sb = (f == 0) ? hbf : __dadd_rn(sb, hbf);
        sc = (f == 0) ? hcf : __dadd_rn(sc, hcf);
        keep(f, hcf);
    }
    if (variant == 1) {                                 // UoCTTI
        store(k, (float)__dmul_rn(0.5, sa));
        store(k + K, (float)__dmul_rn(0.5, sb));
        store(k + 2 * K, (float)__dmul_rn(0.5, sc));
    } else {                                            // Dalal-Triggs
#pragma unroll
        for (int f = 0; f < 4; ++f) store(k + f * K, (float)hcv[f]);
    }
}

// ---- the four block factors of the cell at column x, row y of a gw x gh cell grid (hog.c:930-982), from the energies E
//      (E[(x - ex0) + (y - ey0) * lde]: a window of the grid that holds the cell's neighbours).  Factor q covers the block
//      whose columns are (x - 1, x) for even q, (x, x + 1) for odd q, and rows (y - 1, y) for q < 2, (y, y + 1) above,
//      clamped to the grid.
__device__ __forceinline__ void hog_cell_factors(const float* E, int lde, int ex0, int ey0, int gw, int gh, int x, int y,
                                                 double fac[4])
{
    const int xm = max(x - 1, 0), xp = min(x + 1, gw - 1);
    const int ym = max(y - 1, 0), yp = min(y + 1, gh - 1);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const int xa = ((q & 1) ? x : xm) - ex0, xb = ((q & 1) ? xp : x) - ex0;
        const int ya = ((q & 2) ? y : ym) - ey0, yb = ((q & 2) ? yp : y) - ey0;
        fac[q] = hog_block_factor(E, lde, xa, xb, ya, yb);
    }
}

// ---- the features of a cell from its four block factors (hog.c:985-1053): hog_project for k = 0..K-1 on its bins
//      h[b * hs], and the texture dims 1/sqrt(18) * sum_k hc_f summed in ascending k (UoCTTI).  store(d, v) writes feature
//      dimension d of the cell.
template <class Store>
__device__ __forceinline__ void hog_cell_features(const double* fac, const float* h, int hs, int K, int variant, Store store)
{
    double t[4] = {0.0, 0.0, 0.0, 0.0};
    for (int k = 0; k < K; ++k)
        hog_project(fac, (double)h[k * hs], (double)h[(k + K) * hs], k, K, variant,
                    [&](int q, double hc) { t[q] = __dadd_rn(t[q], hc); }, store);
    if (variant == 1) {
        const float c18 = __fdiv_rn(1.0f, __fsqrt_rn(18.0f));
#pragma unroll
        for (int q = 0; q < 4; ++q) store(3 * K + q, (float)__dmul_rn((double)c18, t[q]));
    }
}

// ---- cv::resize INTER_LINEAR of 8-bit pixels (11-bit fixed point), the landmark patches' resize (sd_hog.cu) and the pyramid
//      levels' (sd_hog_dense.cu).  The taps of output coordinate t of a src -> dst px axis, in OpenCV's arithmetic: scale =
//      1 / (dst / src) in double, f = (t + 0.5) scale - 0.5 rounded to float, s = floor(f).  Column taps: source index sx (s
//      clamped to [0, src - 1], where its fraction becomes 0) and the weights xw = (1 - fx) | fx << 16, each 2048 x rounded
//      to int16; row taps: source rows y0, y1 (s and s + 1 clamped) and the weights yw of the unclamped fraction. ------------
struct HogResizeTap {
    int sx, xw, y0, y1, yw;
};

__device__ __forceinline__ int clip_index(int x, int a, int b) { return x >= a ? (x < b ? x : b - 1) : a; }
__device__ __forceinline__ short sat_short(int v) { return (short)(v > 32767 ? 32767 : (v < -32768 ? -32768 : v)); }

// The source coordinate of output coordinate t, split into s = floor(f) (returned) and the fraction *f, both rules' first step
__device__ __forceinline__ int hog_resize_coord(int t, int dst, int src, float* frac)
{
    const double inv_scale = __ddiv_rn((double)dst, (double)src);
    const double scale = __ddiv_rn(1.0, inv_scale);
    const float f = (float)__dadd_rn(__dmul_rn((double)t + 0.5, scale), -0.5);
    const int s = (int)floorf(f);
    *frac = __fsub_rn(f, (float)s);
    return s;
}

__device__ __forceinline__ HogResizeTap hog_resize_tap(int t, int dst, int src)
{
    float f;
    const int s = hog_resize_coord(t, dst, src, &f);
    int sx = s;
    float fx = f;
    if (sx < 0) { fx = 0.f; sx = 0; }
    if (sx >= src - 1) { fx = 0.f; sx = src - 1; }
    const short2 xa = make_short2(sat_short(__float2int_rn(__fmul_rn(__fsub_rn(1.f, fx), 2048.f))),
                                  sat_short(__float2int_rn(__fmul_rn(fx, 2048.f))));
    const short2 yb = make_short2(sat_short(__float2int_rn(__fmul_rn(__fsub_rn(1.f, f), 2048.f))),
                                  sat_short(__float2int_rn(__fmul_rn(f, 2048.f))));
    HogResizeTap r;
    r.sx = sx;
    r.xw = *reinterpret_cast<const int*>(&xa);
    r.y0 = clip_index(s, 0, src);
    r.y1 = clip_index(s + 1, 0, src);
    r.yw = *reinterpret_cast<const int*>(&yb);
    return r;
}

// cv::resize's vertical step of one output pixel from its horizontal sums t0, t1 of source rows 0 and 1 and the y weights
// yb = weight 0 | weight 1 << 16 (int16 each): (b * (t >> 4)) >> 16 per row, then + 2 >> 2
__device__ __forceinline__ int hog_resize_out(int yb, int t0, int t1)
{
    return (((((int)(short)yb) * (t0 >> 4)) >> 16) + (((yb >> 16) * (t1 >> 4)) >> 16) + 2) >> 2;
}

// ---- cv::resize INTER_LINEAR of float pixels, the float pyramid's levels (sd_hog_pyramid_float): the coordinate of
//      hog_resize_coord; column taps sx (clamped as above, its fraction then 0) and xw = the fraction's float bits; row taps y0,
//      y1 as above and yw = the unclamped fraction's float bits.  Every product and sum rounded on its own (no FMA). -----------
__device__ __forceinline__ HogResizeTap hog_resize_tap_f32(int t, int dst, int src)
{
    float f;
    const int s = hog_resize_coord(t, dst, src, &f);
    int sx = s;
    float fx = f;
    if (sx < 0) { fx = 0.f; sx = 0; }
    if (sx >= src - 1) { fx = 0.f; sx = src - 1; }
    HogResizeTap r;
    r.sx = sx;
    r.xw = __float_as_int(fx);
    r.y0 = clip_index(s, 0, src);
    r.y1 = clip_index(s + 1, 0, src);
    r.yw = __float_as_int(f);
    return r;
}

// One source row's value at column taps (sx, fx): S[sx] (1 - fx) + S[sx + 1] fx, or S[sx] (1 - fx) alone at the last column.
// A tap of weight 0 is still read and multiplied, so inf * 0 gives NaN as in cv::resize.
__device__ __forceinline__ float hog_resize_row_f32(const float* row, long long ps, int sx, float fx, int last)
{
    const float a = __fmul_rn(__ldg(row + sx * ps), __fsub_rn(1.f, fx));
    return sx == last ? a : __fadd_rn(a, __fmul_rn(__ldg(row + (sx + 1) * ps), fx));
}

// The vertical step: t0 (1 - fy) + t1 fy
__device__ __forceinline__ float hog_resize_out_f32(float fy, float t0, float t1)
{
    return __fadd_rn(__fmul_rn(t0, __fsub_rn(1.f, fy)), __fmul_rn(t1, fy));
}

// ---- TMA staging: one thread copies the box at (x, y, z) of a 3-D tensor map (`bytes` bytes; x a multiple of 16, bytes
//      outside the tensor zero-filled) to dst on the mbarrier at mbar, and every thread waits in hog_tma_wait ----------------
__device__ __forceinline__ void hog_tma_load(uint64_t* mbar, void* dst, const CUtensorMap* map, int x, int y, int z, int bytes)
{
    const uint32_t bar = (uint32_t)__cvta_generic_to_shared(mbar);
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
                 ::"r"((uint32_t)__cvta_generic_to_shared(dst)), "l"(map), "r"(bar), "r"(x), "r"(y), "r"(z) : "memory");
}

__device__ __forceinline__ void hog_tma_wait(uint64_t* mbar)
{
    const uint32_t bar = (uint32_t)__cvta_generic_to_shared(mbar);
    uint32_t ok = 0;
    const long long t0 = clock64();
    while (!ok) {                                      // bounded: a protocol bug must trap, never hang the GPU
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(ok) : "r"(bar) : "memory");
        if (!ok && clock64() - t0 > 4000000000LL) __trap();
    }
}

// ---- the 3-D u8 tensor map {width, height, count} of equally sized frames with a box_w x box_h x 1 box; false for per-frame
//      descriptors, a base or pitch that is not 16-byte aligned, or a box the driver refuses
inline bool hog_frame_map(const sd_image_batch* images, int box_w, int box_h, CUtensorMap* map)
{
    if (images->d_frames || (reinterpret_cast<uintptr_t>(images->d_data) & 15) || images->row_stride % 16 ||
        (images->count > 1 && images->image_stride % 16))
        return false;
    const sd_encode_tiled_fn enc = sd_encode_tiled();
    if (!enc) return false;
    cuuint64_t gdim[3] = {(cuuint64_t)images->width, (cuuint64_t)images->height, (cuuint64_t)images->count};
    cuuint64_t gstride[2] = {(cuuint64_t)images->row_stride,
                             (cuuint64_t)(images->count > 1 ? images->image_stride : (int64_t)images->row_stride * images->height)};
    if (gstride[1] % 16) gstride[1] = (gstride[1] + 15) / 16 * 16;
    cuuint32_t box[3] = {(cuuint32_t)box_w, (cuuint32_t)box_h, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    return enc(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, const_cast<uint8_t*>(images->d_data), gdim, gstride, box, estr,
               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

}  // namespace
