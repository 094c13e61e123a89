// Pieces of VLFeat's HOG shared by the landmark-patch kernel (sd_hog.cu) and the dense whole-frame kernel (sd_hog_dense.cu):
// the orientation bin of an 8-bit gradient, the orientation table it reads, and the driver entry point of the TMA tensor maps.
// Both kernels call the same functions, so tests/test_gpu_hog_orientation.py covers the bin rule of both.
#pragma once

#include <cuda.h>
#include <cuda_runtime.h>

#include <cmath>

#include "sd_internal.cuh"

namespace {

// Margin of hog_bin's sector test against the reference's first-maximum rule: a lead of the winning |<g, o_k>| over every other
// one of more than eps |g| cannot change the reference's arg-max or its sign (derivation at hog_bin).
constexpr double kBinLead = 4e-6;

// Orientation directions (hog.c:195-204: host libm cos/sin, as the reference) and the reference bin of a gradient (0, gy):
// vbin[0] for gy > 0, vbin[1] for gy < 0.  ox / oy hold SD_MAX_BINS entries; those past K are zero.  For hog_bin's sector
// search: the directions (bx_j, by_j) = (cos, sin)((2j + 1) pi / 2K) of the sector boundaries inside the open first quadrant
// (j < K / 2), and the margin eps / (2 sin(pi / 2K)) on |cross(b, g)| / |g| that gives a lead of eps.
//   Args: any kernel argument block with the members ox, oy, vbin, bx, by and bin_margin.
template <class Args>
inline void hog_orientations(int K, Args& a)
{
    float* ox = a.ox;
    float* oy = a.oy;
    int* vbin = a.vbin;
    for (int k = 0; k < SD_MAX_BINS; ++k) { ox[k] = 0.f; oy[k] = 0.f; }
    for (int k = 0; k < K; ++k) {
        const double angle = k * 3.141592653589793 / K;
        ox[k] = (float)cos(angle);
        oy[k] = (float)sin(angle);
    }
    for (int j = 0; j < SD_MAX_BINS / 2; ++j) {
        const double angle = (2 * j + 1) * 3.141592653589793 / (2 * K);
        a.bx[j] = j < K / 2 ? (float)cos(angle) : 0.f;
        a.by[j] = j < K / 2 ? (float)sin(angle) : 0.f;
    }
    a.bin_margin = (float)(kBinLead / (2.0 * sin(3.141592653589793 / (2 * K))));
    // hog.c:645-672 at gx = 0: ux = +0 and uy = +-1 exactly (the root of gy^2 is exact), so s_k = +-oy_k exactly; the first
    // strict maximum of oy_k > 0 wins, in the lower half-plane when gy < 0 (K = 1: no k has oy_k > 0, bin -1)
    {
        float best = 0.f;
        int bin = -1;
        for (int k = 0; k < K; ++k) if (oy[k] > best) { best = oy[k]; bin = k; }
        vbin[0] = bin;
        vbin[1] = bin < 0 ? -1 : bin + K;
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
//      Args: any kernel argument block with the members ox, oy and vbin that hog_orientations fills.
template <class Args>
__device__ __forceinline__ int hog_bin_unit(const Args& a, int K, float ux, float uy)
{
    float best = 0.f;
    int bin = -1;
#pragma unroll
    for (int k = 0; k < K; ++k) {
        float s = __fadd_rn(__fmul_rn(ux, a.ox[k]), __fmul_rn(uy, a.oy[k]));
        int b = k;
        if (s < 0.f) { s = -s; b += K; }
        if (s > best) { best = s; bin = b; }   // strict >, ascending k
    }
    return bin;
}

// ---- orientation bin of a pixel with a non-zero integer-valued gradient (gx, gy), the reference's float expression
//      verbatim (hog.c:645-672): modulus, normalised gradient (g >= 1, so hog_unit is a float division), then the bin ------
template <class Args>
__device__ __forceinline__ int hog_bin_reference(const Args& a, int K, float gx, float gy, float g)
{
    return hog_bin_unit(a, K, __fdiv_rn(gx, g), __fdiv_rn(gy, g));
}

// ---- bilinear orientation assignment (hog.c:656-678): the reference's top-two tracking of |<u, o_k>| verbatim (a score
//      replaces the first only when strictly larger, else the second when strictly larger), then
//        w1 = (float)((double)acosf(min(s0, 1)) / (pi / K)),  w0 = 1 - w1.
//      b1 = -1 when no second score is positive (K = 1 among others); b0 = -1 for a zero gradient.  pi_k is pi / K in double.
//      acos in double rounded to float stays within an ulp of the reference's acosf. ------------------------------------
template <class Args>
__device__ __forceinline__ void hog_bins_bilinear(const Args& a, int K, float ux, float uy, int& b0, int& b1, float& w1)
{
    float s0 = 0.f, s1 = 0.f;
    b0 = -1;
    b1 = -1;
#pragma unroll
    for (int k = 0; k < K; ++k) {
        float s = __fadd_rn(__fmul_rn(ux, a.ox[k]), __fmul_rn(uy, a.oy[k]));
        int b = k;
        if (s < 0.f) { s = -s; b += K; }
        if (s > s0) { b1 = b0; s1 = s0; b0 = b; s0 = s; }
        else if (s > s1) { b1 = b; s1 = s; }
    }
    const float angle0 = (float)acos((double)fminf(s0, 1.f));
    w1 = (float)__ddiv_rn((double)angle0, a.pi_k);
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
template <class Args>
__device__ __forceinline__ int hog_bin(const Args& a, int K, int gx, int gy, float g)
{
    const float fx = (float)abs(gx), fy = (float)abs(gy);
    float m = (K & 1) ? fx : INFINITY;   // odd K: |cross((0, 1), g)| against the boundary pi / 2
    int s = 0;
#pragma unroll
    for (int j = 0; j < K / 2; ++j) {
        const float c = fmaf(a.bx[j], fy, -(a.by[j] * fx));
        s += c > 0.f;
        m = fminf(m, fabsf(c));
    }
    if (m > a.bin_margin * g) {
        const bool neg = gy < 0;
        if ((gx < 0) != neg) s = K - s;
        if (neg) s += K;
        return s < 2 * K ? s : 0;
    }
    if (gx == 0) return gy == 0 ? -1 : a.vbin[gy < 0];
    return hog_bin_reference(a, K, (float)gx, (float)gy, g);
}

typedef CUresult (*PFN_hogEncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                       const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                       CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

PFN_hogEncodeTiled hog_encode_fn()
{
    static PFN_hogEncodeTiled fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<PFN_hogEncodeTiled>(p);
    }
    return fn;
}

}  // namespace
