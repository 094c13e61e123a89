// Pieces of VLFeat's HOG shared by the landmark-patch kernel (sd_hog.cu) and the dense whole-frame kernel (sd_hog_dense.cu):
// the orientation bin of an 8-bit gradient, the orientation table it reads, and the driver entry point of the TMA tensor maps.
// Both kernels call the same functions, so tests/test_gpu_hog_orientation.py covers the bin rule of both.
#pragma once

#include <cuda.h>
#include <cuda_runtime.h>

#include <cmath>

#include "sd_internal.cuh"

namespace {

// Orientation directions (hog.c:195-204: host libm cos/sin, as the reference) and the reference bin of a gradient (0, gy):
// vbin[0] for gy > 0, vbin[1] for gy < 0.  ox / oy hold SD_MAX_BINS entries; those past K are zero.
inline void hog_orientations(int K, float* ox, float* oy, int* vbin)
{
    for (int k = 0; k < SD_MAX_BINS; ++k) { ox[k] = 0.f; oy[k] = 0.f; }
    for (int k = 0; k < K; ++k) {
        const double angle = k * 3.141592653589793 / K;
        ox[k] = (float)cos(angle);
        oy[k] = (float)sin(angle);
    }
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

// ---- orientation bin of a pixel with a non-zero gradient (gx, gy), the reference's float expression verbatim
//      (hog.c:645-672): modulus, normalised gradient, then the first maximum of |<u, o_k>| in ascending k -------------
//      Args: any kernel argument block with the members ox, oy and vbin that hog_orientations fills.
template <class Args>
__device__ __forceinline__ int hog_bin_reference(const Args& a, int K, float gx, float gy, float g)
{
    // (float)((double)gx / max((double)g, 1e-10)) == gx / g in float: double rounding is innocuous for
    // division when the wide format has >= 2p+2 bits (53 >= 50).
    const float ux = __fdiv_rn(gx, g);
    const float uy = __fdiv_rn(gy, g);
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

// ---- orientation bin of an interior pixel without a division.  t_k = gx ox_k + gy oy_k on the integer gradient decides the
//      arg-max whenever its winner leads the runner-up by more than eps |g|; only the other lanes need the exact answer below.
//      Why that is exact (u = 2^-24, r = |g| exact, e_k = gx ox_k + gy oy_k exact, ox_k^2 + oy_k^2 = 1 + O(u)):
//        |t_k - e_k|     <= 2u r                           (one product, one FMA)
//        |s_k - e_k / r| <= 4u                              (s_k: the reference's float dot product of gx/g, gy/g)
//      so t_b leading every other |t_j| by eps r makes |s_b| lead every |s_j| by (eps - 12u) > 0, and |t_b| > eps r fixes
//      the sign of s_b: the reference's first strict maximum is the same k and the same half-plane.  eps = 4e-6 is ~33u;
//      the slack also covers the rounding of the test itself (squared, against eps^2 g2, to avoid the root).
//      tests/test_gpu_hog_orientation.py checks every (gx, gy) in [-255, 255]^2 at every K in 1..16. ------------------------
constexpr float kBinMargin2 = 4e-6f * 4e-6f;

template <class Args>
__device__ __forceinline__ int hog_bin(const Args& a, int K, int gx, int gy, int g2, float g)
{
    if (g2 == 0) return -1;
    const float fx = (float)gx, fy = (float)gy;
    float m1 = 0.f, m2 = 0.f;            // largest and second largest |t_k| (a tie leaves m1 == m2: no margin)
    int best = 0;
    bool neg = false;
#pragma unroll
    for (int k = 0; k < K; ++k) {
        const float t = fmaf(fx, a.ox[k], fy * a.oy[k]);
        const float m = fabsf(t);
        if (m > m1) { m2 = m1; m1 = m; best = k; neg = t < 0.f; }
        else if (m > m2) m2 = m;
    }
    const float d = m1 - m2;
    if (d * d > kBinMargin2 * (float)g2) return neg ? best + K : best;
    // the gx = 0 axis is a bin boundary for odd K and common in real patches; the reference's unit vector there is exactly
    // (0, +-1), so its bin is a function of K and the sign of gy alone (hog_orientations)
    if (gx == 0) return a.vbin[gy < 0];
    return hog_bin_reference(a, K, fx, fy, g);
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
