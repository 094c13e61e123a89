// Batched per-landmark HOG projection: the CUDA restatement of rcr::HogTransform::operator()
// (reference include/rcr/adaptive_vlhog.hpp:109-185) fused with VLFeat's vl_hog_put_image /
// vl_hog_extract (reference include/rcr/hog.c:595-728, :857-1062).
//
// hog_patch_kernel: one CTA per (sample, landmark) patch, from the 8-bit source image in HBM to the patch's cell histograms,
// which it leaves in its slice of the feature row; hog_normalise_kernel, several patches per CTA, turns them into the
// features in place (the last four steps below):
//   geometry (IED -> half patch size, cvRound centre)            adaptive_vlhog.hpp:123,132-133
//   zero-padded crop: ONE TMA tile load per patch (3-D tensor map over the frame batch; out-of-frame
//     bytes are zero-filled by the TMA = copyMakeBorder(BORDER_CONSTANT 0))   adaptive_vlhog.hpp:135-151
//   cv::resize INTER_LINEAR (fixed point), tables precomputed once per face   adaptive_vlhog.hpp:154-155
//   gradient, orientation arg-max and modulus in registers (bit exact: margin-checked arg-max, exact fallback)  hog.c:631-672
//   bilinear spatial vote as two separable passes (rows x cell columns, then cell rows; no atomics)      hog.c:697-724
//   cell energy, 2x2-block normalisation in double, clamp 0.2    hog.c:875-1053
//   per-dimension transpose + landmark concatenation + bias      adaptive_vlhog.hpp:166-183
//
// Arithmetic that decides an INTEGER result (crop centre, half size, resize taps, orientation bin)
// is written with explicit round-to-nearest intrinsics so that no FMA contraction can change it;
// the reference is built for baseline x86-64 (mul then add).  The orientation bin's margin test (hog_bin) is the exception:
// its error bound allows FMA, and the pixels it cannot decide take the reference expression.  The only deviation from the
// reference's value stream is the summation ORDER of the float votes inside a cell histogram
// (fixed, deterministic tree here; raster order there): ~1e-7 relative.
#include "sd_internal.cuh"
#include "sd_hog_common.cuh"
#include "sd_warp.cuh"

#include <cmath>
#include <type_traits>
#include <cuda_pipeline.h>

namespace {

// CTA size of hog_normalise_kernel and of the run-time hog_patch_kernel schedules; the compiled-in schedules pick their
// own (launch_hog)
constexpr int kHogThreads = 256;

struct HogArgs {
    const uint8_t* images;
    int width, height, row_stride;
    long long image_stride;
    int image_count;
    const int* image_index;
    const sd_roi* roi;          // optional: only a region of every frame is resident
    const sd_frame* frames;     // optional: frames of different sizes
    uint8_t* roi_miss;
    const float* x;
    long long ldx;
    int N, L;
    int variant, nc, cs, K, fs, dd;
    const int* half;            // per sample: half patch size (hog_geometry_kernel)
    HogOrient orient;           // orientation table, host libm (hog.c:195-204), and hog_bin's sector search
    const int* rtab;            // per sample: resize tables [5][fs] (hog_geometry_kernel)
    const float* btab;          // per launch: spatial binning weights [nc][fs], then lo[nc], hi[nc] (hog_bintab_kernel)
    int tma_count;              // number of usable tensor-map size classes (0: the window is staged by load loops)
    float* A;
    long long ld;
    int* geometry;
    uint8_t* patches;
    int8_t* bins;
    int* status;
};

// ---- per-sample geometry: IED -> half patch size (adaptive_vlhog.hpp:123) and the interpolation tables of cv::resize
//      (INTER_LINEAR, 8U, 11-bit fixed point) for a P x P -> fs x fs resize, once per sample instead of once per thread of
//      every one of its L patches.  One CTA per sample.  rtab[sample][0..4][fs]: x source index, x weights (2 x int16),
//      y source index 0 / 1 (clamped), y weights (hog_resize_tap).  face_flag (optional): a degenerate sample also sets its
//      own byte, so that a caller can drop that face alone (sd_track_faces).  Warped launches (warp.in) also check each
//      sample's warp here and copy it to warp.out, an invalid one (or one whose frame index is out of range) as a 0 x 0 V that
//      the HOG kernel reads no pixel of. -----------------------------------------------------------------------------------------
struct HogWarpCheck {
    const sd_sample_warp* in;   // the caller's table, or NULL: no warp
    sd_sample_warp* out;        // what hog_patch_kernel reads
    const int* image_index;
    int image_count, width, height;
    const sd_frame* frames;
};

__global__ void hog_geometry_kernel(const float* __restrict__ x, long long ldx, int N, int L, const sd_eyes_dev eyes, float rel,
                                    int fixed_half, int fs, int* __restrict__ half_out, int* __restrict__ rtab, int* __restrict__ status,
                                    uint8_t* __restrict__ face_flag, const HogWarpCheck warp)
{
    const int i = blockIdx.x;
    if (i >= N) return;
    __shared__ int s_half;
    if (threadIdx.x == 0) {
        bool degenerate;
        const int half = sd_patch_half(x + (long long)i * ldx, L, eyes, rel, fixed_half, &degenerate);
        if (degenerate) {                      // cv::resize would throw on the empty ROI; flag it and keep going
            atomicOr(status, 1);
            if (face_flag) face_flag[i] = 1;
        }
        half_out[i] = half;
        s_half = half;
        if (warp.in) {
            sd_sample_warp w = warp.in[i];
            const int f = warp.image_index ? warp.image_index[i] : i;   // a mirrored bit is out of range: no decoding
            bool ok = f >= 0 && f < warp.image_count;                   // out of range: hog_patch_kernel flags it
            if (ok) {
                const int fw = warp.frames ? warp.frames[f].width : warp.width, fh = warp.frames ? warp.frames[f].height : warp.height;
                ok = sd_warp_valid(w, fw, fh);
                if (!ok) atomicOr(status, 4);
            }
            if (!ok) w.width = w.height = 0;
            warp.out[i] = w;
        }
    }
    __syncthreads();
    const int P = 2 * s_half;
    int* rt = rtab + (long long)i * 5 * fs;
    for (int t = threadIdx.x; t < fs; t += blockDim.x) {
        const HogResizeTap r = hog_resize_tap(t, fs, P);
        rt[t] = r.sx;
        rt[fs + t] = r.xw;
        rt[2 * fs + t] = r.y0;
        rt[3 * fs + t] = r.y1;
        rt[4 * fs + t] = r.yw;
    }
}

// ---- spatial binning tables of vl_hog_put_image (hog.c:697-709), once per launch: btab[c * pw + t - 1] = weight with which
//      interior pixel coordinate t (1 .. fs - 2) votes into cell index c (w1 for its own bin, w2 for the next one, 0 otherwise;
//      pw = fs - 2 rounded up to even, the padding entry 0); then, as ints, the first and last interior coordinate that votes
//      into cell c (same tables for rows and columns: square patch, square cells) ------------------------------------------
__global__ void hog_bintab_kernel(int fs, int nc, int cs, int pw, float* __restrict__ btab)
{
    __shared__ int s_sbin[256];
    for (int t = threadIdx.x; t < fs; t += blockDim.x) {
        int b;
        float w1, w2;
        hog_spatial_weight(t, cs, &b, &w1, &w2);
        s_sbin[t] = b;
        if (t >= 1 && t <= fs - 2)
            for (int c = 0; c < nc; ++c) btab[c * pw + t - 1] = (b == c) ? w1 : ((b == c - 1) ? w2 : 0.f);
        else if (t == fs - 1 && pw > fs - 2)
            for (int c = 0; c < nc; ++c) btab[c * pw + pw - 1] = 0.f;
    }
    __syncthreads();
    int* lohi = reinterpret_cast<int*>(btab + nc * pw);
    for (int c = threadIdx.x; c < nc; c += blockDim.x) {
        int lo = fs, hi = -1;
        for (int t = 1; t <= fs - 2; ++t) {
            const int b = s_sbin[t];
            if (b == c || b == c - 1) { if (t < lo) lo = t; hi = t; }
        }
        lohi[c] = lo;
        lohi[nc + c] = hi;
    }
}

// byte n (0..7) of the 8 bytes lo, hi (little endian)
__device__ __forceinline__ int byte_of(unsigned lo, unsigned hi, int n) { return (int)(((n < 4 ? lo : hi) >> (8 * (n & 3))) & 0xffu); }

// shared-memory carve-up (same function on host and device)
struct HogSmem {
    int patch, bin, r1, tab, xa, wcell, lo, hi, vote, mbar, stage_end, total;
    int pp;        // row pitch of the resized patch: fs rounded up to a multiple of 4
    int pb, pm;    // row pitches of the interior bins (bytes, a multiple of 4) and moduli (floats, odd)
    int pw;        // row pitch of the binning weights (floats, even)
    int tpad;      // tasks of the horizontal vote pass, padded to a multiple of 32
};

__host__ __device__ inline int align_up(int v, int a) { return (v + a - 1) / a * a; }

// [bin | r1 | vote] is dead during S1, so that whole span is the staging area of the source window.  The cell histograms
// go from the vote's second pass straight to global memory (hog_normalise_kernel takes them from there).  The patch rows
// are word aligned (pitch pp) so that S1 stores and S2 loads whole words.  Bins and moduli hold the interior pixels only,
// pixel (y, x) at (y - 1) * pitch + x - 1, so that S2's runs of four start on a word of bins.  Pass 1 of the vote reads
// one row per lane: an odd pitch (moduli) keeps those reads free of bank conflicts, and so does an odd number of words
// between rows of bins where that fits in fs * fs bytes.  Both regions hold fs * fs pixels, as before: the staging area
// and the largest configuration are the same.  The binning weights hold the interior coordinates only, t at c * pw + t - 1
// with an even pitch, so that a pair (t, t + 1) with t odd is one aligned 8-byte word of weights and one 16-bit word of bins.
__host__ __device__ inline HogSmem hog_smem_layout(int fs, int nc, int K)
{
    HogSmem s;
    s.pp = align_up(fs, 4);
    s.pm = align_up(fs - 2, 4) + 1;                         // a row's runs of four, odd: (fs - 2) * pm < fs * fs
    s.pb = s.pm - 1;
    if ((s.pb & 7) == 0 && (fs - 2) * (s.pb + 4) <= fs * fs) s.pb += 4;
    int o = 0;
    s.patch = o;
    o = align_up(s.pp * fs, 16);
    s.tab = o;    o += fs * 16;                             // int4 {x source index, y source index 0 / 1, y weights (2 x int16)}
    s.xa = o;     o += fs * 4;                              // x weights, 2 x int16
    s.pw = align_up(fs - 2, 2);
    s.wcell = align_up(o, 8); o = s.wcell + nc * s.pw * 4; // weight of pixel t for cell index c (0 if it does not vote)
    s.lo = o;     o += nc * 4;
    s.hi = o;     o += nc * 4;
    s.mbar = align_up(o, 8); o = s.mbar + 8;
    o = align_up(o, 128);
    s.bin = o;    o = align_up(o + fs * fs, 16);            // staging area from here to stage_end (128-byte aligned: TMA destination)
    s.r1 = o;     o = align_up(o + fs * fs * 4, 16);        // r1 = gradient modulus
    s.tpad = align_up((fs - 2) * nc, 32);
    s.vote = o;                                             // horizontal pass of the vote: T[bin][(cell column, row)]
    o += 2 * K * s.tpad * 4;
    s.stage_end = o;
    s.total = align_up(o + 8, 16);                          // S1's word loads read up to 7 bytes past the staged window
    return s;
}

// KT / NCT / CST > 0 bake the bin count, cells per side and cell size into the kernel (the schedules the
// reference ships: 5x5 cells of 11/10/8/6 px, K = 4 or 9), which lets the compiler strength-reduce every
// index computation; 0 = taken from the arguments at run time (any other configuration).
// tensor maps of the frame batch (u8, dims {W, H, count}), one per square box size: a patch uses the smallest box that covers
// its P x P source window
constexpr int kTmaClasses = 8;
__host__ __device__ constexpr int hog_tma_box(int c) { return c == 0 ? 32 : c == 1 ? 48 : c == 2 ? 64 : c == 3 ? 80 : c == 4 ? 96 : c == 5 ? 112 : c == 6 ? 128 : 160; }
struct HogMaps { CUtensorMap m[kTmaClasses]; };
// The second parameter of hog_patch_kernel: the tensor maps, or in a warped launch (which loads no window) the checked warps.
// A type rather than a third parameter, so that the unwarped instantiations keep their code.
template <bool WARP> using HogSource = typename std::conditional<WARP, const sd_sample_warp*, HogMaps>::type;

// Pixel (u, v) of the V of warp sw, computed from the four taps it reads in the frame (resident region rx, ry, rw, rh; a tap
// outside the frame reads 0, one inside the frame but outside the region sets *miss): the unstaged route's window pixel.
__device__ __noinline__ int hog_warp_pixel(const sd_sample_warp* __restrict__ sw, int u, int v, const uint8_t* __restrict__ img, int W,
                                           int H, int rs, int rx, int ry, int rw, int rh, bool* miss)
{
    if ((unsigned)u >= (unsigned)sw->width || (unsigned)v >= (unsigned)sw->height) return 0;
    const int2 d = sd_warp_col(sw->m, (double)u), r = sd_warp_row(sw->m, (double)v);
    return sd_warp_sample<uint8_t>((r.x + d.x) >> 5, (r.y + d.y) >> 5, [&](int ix, int iy) -> uint8_t {
        if ((unsigned)ix >= (unsigned)W || (unsigned)iy >= (unsigned)H) return 0;
        if (ix < rx || ix >= rx + rw || iy < ry || iy >= ry + rh) {
            *miss = true;
            return 0;
        }
        return __ldg(img + (long long)(iy - ry) * rs + (ix - rx));
    });
}

// Whether sample i is a sample of its frame's mirror (CTA-uniform).  Only the MIR instantiations, launched for an index that
// may carry SD_SAMPLE_MIRRORED, ask; the others compile to the unmirrored kernel.  hog_patch_kernel asks again where it needs
// the answer instead of keeping a flag live through S1, which would push the compiled-in schedules past 32 registers.
template <bool MIR>
__device__ __forceinline__ bool hog_sample_mirrored(const HogArgs& a, int sample)
{
    return MIR && sd_sample_is_mirrored(a.image_index[sample]);
}

// NT threads per CTA.  The compiled-in schedules fit 32 registers without spills, so an SM holds 2048 / NT CTAs where shared
// memory allows; the run-time ones (NT = 256) spill at that bound and keep the compiler's choice (a minimum of 0 CTAs per SM
// sets no bound).  The WARP instantiations of the compiled-in schedules spill at 32 registers (the double-precision warp terms
// and the tap arithmetic of S1) and are bounded at 1024 / NT CTAs per SM, 64 registers, instead (DESIGN §4.12).
//
// WARP: sample i is a sample of the V of warps[i] (sd_sample_warp; hog_geometry_kernel's checked copy, an invalid warp as a 0 x 0
// V).  Only launches with a warp table take the WARP instantiations (MIR = false: a mirrored bit is an index out of range); in
// the others `warps` is unused and the code is the unwarped kernel's.
template <int KT, int NCT, int CST, int NT, bool MIR, bool WARP>
__global__ void __launch_bounds__(NT, NCT > 0 ? (WARP ? 1024 : 2048) / NT : 0) hog_patch_kernel(const __grid_constant__ HogArgs a,
                                                                                                 const __grid_constant__ HogSource<WARP> maps)
{
    // whole warps, and at least one row group of the fs <= 64 resize (NT / fs >= 1)
    static_assert(NT % 32 == 0 && NT >= 64, "hog_patch_kernel needs whole warps and at least 64 threads");
    constexpr int kWarps = NT / 32;
    extern __shared__ __align__(128) unsigned char smem[];
    const int K = KT > 0 ? KT : a.K;
    const int nc = NCT > 0 ? NCT : a.nc;
    const int fs = (NCT > 0 && CST > 0) ? NCT * CST : a.fs;
    const int cells = nc * nc;
    const HogSmem lay = hog_smem_layout(fs, nc, K);
    const int pp = lay.pp, pb = lay.pb, pm = lay.pm, pw = lay.pw;
    uint8_t* s_patch = smem + lay.patch;
    int8_t* s_bin = reinterpret_cast<int8_t*>(smem + lay.bin);
    float* s_gmag = reinterpret_cast<float*>(smem + lay.r1);
    int4* s_tab = reinterpret_cast<int4*>(smem + lay.tab);
    short2* s_xa = reinterpret_cast<short2*>(smem + lay.xa);
    float* s_wcell = reinterpret_cast<float*>(smem + lay.wcell);
    int* s_lo = reinterpret_cast<int*>(smem + lay.lo);
    int* s_hi = reinterpret_cast<int*>(smem + lay.hi);
    float* s_T = reinterpret_cast<float*>(smem + lay.vote);
    uint64_t* s_mbar = reinterpret_cast<uint64_t*>(smem + lay.mbar);

    const int tid = threadIdx.x;
    const int lane = tid & 31, warp = tid >> 5;
    const long long patch_id = blockIdx.x;
    const int sample = (int)(patch_id / a.L);
    const int lm = (int)(patch_id - (long long)sample * a.L);

    // ---- S0: geometry: half size from the per-sample pre-pass, centre = cvRound (adaptive_vlhog.hpp:132-133)
    const float* __restrict__ row = a.x + (long long)sample * a.ldx;
    const int half = __ldg(a.half + sample);
    const int P = 2 * half;
    const int cx = __float2int_rn(row[lm]);
    const int cy = __float2int_rn(row[lm + a.L]);
    int img_idx = a.image_index ? a.image_index[sample] : sample;
    if (MIR) img_idx = sd_sample_frame_of(img_idx);
    if (img_idx < 0 || img_idx >= a.image_count) {
        img_idx = 0;
        if (tid == 0 && a.status) atomicOr(a.status, 2);
    }
    // resident region of this frame: the whole frame, or the ROI that sd_detect_faces_host gathered
    int W = a.width, H = a.height, rs = a.row_stride;
    const uint8_t* __restrict__ img = a.images + (long long)img_idx * a.image_stride;
    if (a.frames) {
        const sd_frame f = a.frames[img_idx];
        W = f.width; H = f.height; rs = f.row_stride;
        img = a.images + f.offset;
    }
    int rx = 0, ry = 0, rw = W, rh = H;
    if (a.roi) {
        const sd_roi r = a.roi[img_idx];
        rx = r.x; ry = r.y; rw = r.w; rh = r.h; rs = r.row_stride;
        img = a.images + r.offset;
    }
    if (tid == 0 && a.geometry) {
        a.geometry[patch_id * 3 + 0] = cx;
        a.geometry[patch_id * 3 + 1] = cy;
        a.geometry[patch_id * 3 + 2] = half;
    }

    // ---- S1: zero-padded crop + fixed-point bilinear resize.  The P x P source window is staged in shared memory with its
    //      zero padding materialised, then resampled from there: one output row per warp pass, lanes along x.  A mirrored
    //      sample's centre cx is a column of the mirror M; its window is the frame's window starting at x0 (sd_window_x0), which
    //      is staged by the same route as any other and then reversed row by row in shared memory, so that from then on column
    //      c of the staged window is M's column c and the resize, and everything after it, runs on M's window unchanged.
    const int x0 = sd_window_x0(cx, half, W, hog_sample_mirrored<MIR>(a, sample)), y0 = cy - half;
    uint8_t* s_stage = smem + lay.bin;                             // [bin | r1 | vote] are dead until S2
    const int stage_cap = lay.stage_end - lay.bin;
    // TMA route: whole frames resident and describable by a tensor map; the smallest box class that covers the window and
    // fits the staging area
    int tma_box = 0;
    // The TMA wants the box to start on a 16-byte boundary of the innermost dimension (an unaligned start faults with "illegal
    // instruction"): the box starts at x0 rounded down to a multiple of 16 and the window sits tma_shift bytes into its rows.
    const int tma_shift = x0 & 15;
#pragma unroll
    for (int c = kTmaClasses - 1; c >= 0; --c)
        if (c < a.tma_count && hog_tma_box(c) >= P + tma_shift && hog_tma_box(c) * hog_tma_box(c) <= stage_cap) tma_box = hog_tma_box(c);
    if constexpr (!WARP) if (tma_box > 0 && tid == 0) {
        // one elected thread: the box lands densely (pitch = box width); bytes outside the frame are zero-filled by the TMA,
        // which is exactly copyMakeBorder(..., BORDER_CONSTANT, 0) (adaptive_vlhog.hpp:136-147)
        int cls = 0;
#pragma unroll
        for (int c = 0; c < kTmaClasses; ++c) if (hog_tma_box(c) == tma_box) cls = c;
        hog_tma_load(s_mbar, s_stage, &maps.m[cls], x0 - tma_shift, y0, img_idx, tma_box * tma_box);
    }

    // tables: cv::resize taps of this sample (hog_geometry_kernel), spatial binning weights of this launch (hog_bintab_kernel)
    {
        const int* __restrict__ rt = a.rtab + (long long)sample * 5 * fs;
        for (int t = tid; t < fs; t += NT) {
            const int xa = __ldg(rt + fs + t);
            s_xa[t] = *reinterpret_cast<const short2*>(&xa);
            s_tab[t] = make_int4(__ldg(rt + t), __ldg(rt + 2 * fs + t), __ldg(rt + 3 * fs + t), __ldg(rt + 4 * fs + t));
        }
        for (int i = tid; i < nc * pw; i += NT) s_wcell[i] = __ldg(a.btab + i);
        const int* __restrict__ lohi = reinterpret_cast<const int*>(a.btab + nc * pw);
        if (tid < nc) { s_lo[tid] = __ldg(lohi + tid); s_hi[tid] = __ldg(lohi + nc + tid); }
    }
    {
        const bool resident = x0 >= rx && y0 >= ry && x0 + P <= rx + rw && y0 + P <= ry + rh && x0 >= 0 && y0 >= 0 && x0 + P <= W && y0 + P <= H;
        const uintptr_t align_bits = reinterpret_cast<uintptr_t>(img) | (uintptr_t)rs;
        const bool vec16 = !tma_box && resident && (align_bits & 15) == 0;      // rows can be fetched as aligned 16-byte vectors
        const bool words = !tma_box && resident && (align_bits & 3) == 0;
        // column c of the staged window sits at byte shiftb + c of its row
        const int shiftb = tma_box ? tma_shift : (vec16 ? ((x0 - rx) & 15) : (words ? ((x0 - rx) & 3) : 0));
        const int pitch = tma_box ? tma_box : ((P + 15 + 15) & ~15);
        // A warped window is computed pixel by pixel, never loaded (the launch has no tensor maps: tma_box = 0), at byte shiftb of
        // its staged rows as any window; its per-column and per-row terms (4 x P ints) follow the rows.  `if constexpr` keeps the
        // unwarped instantiations' code as it was.
        const bool staged = (pitch + (WARP ? 16 : 0)) * P <= stage_cap;
        bool miss = false;
        if (staged) {
            if constexpr (WARP) {
                // cv::warpAffine's terms once per patch, as face_chip_warp_kernel does per tile: adelta / bdelta of each window
                // column, X0 / Y0 of each window row (only inside V), then each window pixel from its four taps in the frame
                const sd_sample_warp* __restrict__ warps = maps;                // a warped launch's second parameter
                const sd_sample_warp* __restrict__ sw = warps + sample;
                const int Wv = sw->width, Hv = sw->height;
                int* s_wt = reinterpret_cast<int*>(s_stage + pitch * P);   // [adelta | bdelta | X0 | Y0], P each
                for (int t = tid; t < P; t += NT) {
                    if ((unsigned)(x0 + t) < (unsigned)Wv) {
                        const int2 d = sd_warp_col(sw->m, (double)(x0 + t));
                        s_wt[t] = d.x;
                        s_wt[P + t] = d.y;
                    }
                    if ((unsigned)(y0 + t) < (unsigned)Hv) {
                        const int2 r = sd_warp_row(sw->m, (double)(y0 + t));
                        s_wt[2 * P + t] = r.x;
                        s_wt[3 * P + t] = r.y;
                    }
                }
                __syncthreads();
                for (int r = warp; r < P; r += kWarps) {
                    const bool rowin = (unsigned)(y0 + r) < (unsigned)Hv;
                    const int X0 = s_wt[2 * P + r], Y0 = s_wt[3 * P + r];
#pragma unroll 1
                    for (int c = lane; c < P; c += 32) {
                        uint8_t v = 0;
                        if (rowin && (unsigned)(x0 + c) < (unsigned)Wv)
                            v = sd_warp_sample<uint8_t>((X0 + s_wt[c]) >> 5, (Y0 + s_wt[P + c]) >> 5, [&](int ix, int iy) -> uint8_t {
                                if ((unsigned)ix >= (unsigned)W || (unsigned)iy >= (unsigned)H) return 0;
                                if (ix < rx || ix >= rx + rw || iy < ry || iy >= ry + rh) {
                                    miss = true;                   // a frame pixel that was not uploaded
                                    return 0;
                                }
                                return __ldg(img + (long long)(iy - ry) * rs + (ix - rx));
                            });
                        s_stage[r * pitch + shiftb + c] = v;
                    }
                }
            } else if (tma_box) {
                // nothing to do: the tile is in flight
            } else if (vec16) {
                // 8 / 16 / 32 lanes per source row, one aligned uint4 each: ~P * nvec / 32 warp loads in total
                const int nvec = (shiftb + P + 15) >> 4;
                const int gs = nvec <= 8 ? 3 : (nvec <= 16 ? 4 : 5);
                const int lv = lane & ((1 << gs) - 1), lr = lane >> gs, rows_per_pass = 32 >> gs;
                const uint8_t* wrow = img + (long long)(y0 - ry) * rs + (x0 - rx - shiftb);
                // not unrolled (here and in the word loop): unrolled, they spill at 32 registers at fs = 30, K = 4
                for (int r = warp * rows_per_pass + lr; r < P; r += kWarps * rows_per_pass)
#pragma unroll 1
                    for (int v = lv; v < nvec; v += (1 << gs))
                        reinterpret_cast<uint4*>(s_stage + r * pitch)[v] = __ldg(reinterpret_cast<const uint4*>(wrow + (long long)r * rs) + v);
            } else if (words) {
                const int nwords = (shiftb + P + 3) >> 2;
                const uint8_t* wrow = img + (long long)(y0 - ry) * rs + (x0 - rx - shiftb);
                for (int r = warp; r < P; r += kWarps) {
                    const uint32_t* src = reinterpret_cast<const uint32_t*>(wrow + (long long)r * rs);
                    uint32_t* dst = reinterpret_cast<uint32_t*>(s_stage + r * pitch);
#pragma unroll 1
                    for (int w = lane; w < nwords; w += 32) dst[w] = __ldg(src + w);
                }
            } else {
                for (int r = warp; r < P; r += kWarps) {
                    const int iy = y0 + r;
                    const bool rowin = (unsigned)iy < (unsigned)H;
                    const bool rowres = iy >= ry && iy < ry + rh;
                    for (int c = lane; c < P; c += 32) {
                        const int ix = x0 + c;
                        int v = 0;
                        if (rowin && (unsigned)ix < (unsigned)W) {
                            if (rowres && ix >= rx && ix < rx + rw) v = __ldg(img + (long long)(iy - ry) * rs + (ix - rx));
                            else miss = true;                      // a frame pixel that was not uploaded
                        }
                        s_stage[r * pitch + c] = (uint8_t)v;
                    }
                }
            }
            __syncthreads();                                       // tables (and the load loops' stores) visible
            if (tma_box) hog_tma_wait(s_mbar);
            if (hog_sample_mirrored<MIR>(a, sample)) {
                // swap columns c and P - 1 - c of every staged row (P is even), a row per warp, lanes along the row; the resize's
                // clamped tap P - 1 + 1 (weight 0) may still read the unreversed byte past the window
#pragma unroll 1
                for (int r = warp; r < P; r += kWarps) {
                    uint8_t* q = s_stage + r * pitch + shiftb;
#pragma unroll 1
                    for (int c = lane; c < half; c += 32) {
                        const uint8_t u = q[c], v = q[P - 1 - c];
                        q[c] = v;
                        q[P - 1 - c] = u;
                    }
                }
                __syncthreads();
            }
            if (fs <= 64) {
                // a thread keeps TWO adjacent output columns (their taps and weights stay in registers) and walks down the
                // rows: NT / ceil(fs / 2) row groups, the rest of the threads idle.  When the four taps of the pair lie in the
                // 8 bytes from the word at q (any window up to about 3x the patch), a row costs one table load, two word loads
                // per source row and one 16-bit store for both outputs; a byte permute puts a tap pair in the low half of a
                // word and dp2a forms its weighted sum, the same integer as the scalar products.  Odd fs: the last thread's
                // second output repeats its first into the padding column.
                const int np = (fs + 1) >> 1, groups = NT / np;
                const int j = tid % np, g = tid / np;
                if (g < groups) {
                    const int dxa = 2 * j, dxb = min(dxa + 1, fs - 1);
                    const int sxa = s_tab[dxa].x, sxb = s_tab[dxb].x;
                    const unsigned xa = *reinterpret_cast<const unsigned*>(s_xa + dxa), xb = *reinterpret_cast<const unsigned*>(s_xa + dxb);
                    const int q = (shiftb + sxa) & ~3;
                    const int oa = shiftb + sxa - q, ob = shiftb + sxb - q;
                    uint8_t* out = s_patch + dxa;                  // s_patch precedes the staging area: no overlap
                    if (ob <= 6) {
                        // tap sx + 1 of a clamped column (sx = P - 1) may lie past the window: its weight is 0
                        const unsigned sa = oa | (oa + 1) << 4, sb = ob | (ob + 1) << 4;
                        const uint8_t* base = s_stage + q;
#pragma unroll 2
                        for (int dy = g; dy < fs; dy += groups) {
                            const int4 yt = s_tab[dy];
                            const unsigned* r0 = reinterpret_cast<const unsigned*>(base + yt.y * pitch);
                            const unsigned* r1 = reinterpret_cast<const unsigned*>(base + yt.z * pitch);
                            const unsigned a0 = r0[0], a1 = r0[1], b0 = r1[0], b1 = r1[1];
                            const int va = hog_resize_out(yt.w, __dp2a_lo(xa, __byte_perm(a0, a1, sa), 0u), __dp2a_lo(xa, __byte_perm(b0, b1, sa), 0u));
                            const int vb = hog_resize_out(yt.w, __dp2a_lo(xb, __byte_perm(a0, a1, sb), 0u), __dp2a_lo(xb, __byte_perm(b0, b1, sb), 0u));
                            *reinterpret_cast<uint16_t*>(out + dy * pp) = (uint16_t)(va | vb << 8);
                        }
                    } else {
                        const int ax = s_xa[dxa].x, bx = s_xa[dxa].y, cx = s_xa[dxb].x, dx = s_xa[dxb].y;
                        const int sxa1 = min(sxa + 1, P - 1), sxb1 = min(sxb + 1, P - 1);   // clamped tap has zero weight
                        const uint8_t* base = s_stage + shiftb;
                        for (int dy = g; dy < fs; dy += groups) {
                            const int4 yt = s_tab[dy];
                            const uint8_t* r0 = base + yt.y * pitch;
                            const uint8_t* r1 = base + yt.z * pitch;
                            const int va = hog_resize_out(yt.w, (int)r0[sxa] * ax + (int)r0[sxa1] * bx, (int)r1[sxa] * ax + (int)r1[sxa1] * bx);
                            const int vb = hog_resize_out(yt.w, (int)r0[sxb] * cx + (int)r0[sxb1] * dx, (int)r1[sxb] * cx + (int)r1[sxb1] * dx);
                            *reinterpret_cast<uint16_t*>(out + dy * pp) = (uint16_t)(va | vb << 8);
                        }
                    }
                }
            } else {
                for (int dy = warp; dy < fs; dy += kWarps) {
                    const int4 yt = s_tab[dy];
                    const uint8_t* r0 = s_stage + yt.y * pitch + shiftb;
                    const uint8_t* r1 = s_stage + yt.z * pitch + shiftb;
                    for (int dx = lane; dx < fs; dx += 32) {
                        const int sx = s_tab[dx].x;
                        const int sx1 = min(sx + 1, P - 1);
                        const short2 xa = s_xa[dx];
                        const int t0 = (int)r0[sx] * xa.x + (int)r0[sx1] * xa.y;
                        const int t1 = (int)r1[sx] * xa.x + (int)r1[sx1] * xa.y;
                        s_patch[dy * pp + dx] = (uint8_t)hog_resize_out(yt.w, t0, t1);
                    }
                }
            }
        } else {
            // window too large for the staging area: sample straight from global memory with full checks; a mirrored sample's
            // column u of M's window is column P - 1 - u of the frame's
            const bool mirrored = hog_sample_mirrored<MIR>(a, sample);
            __syncthreads();                                       // tables visible
            for (int dy = warp; dy < fs; dy += kWarps) {
                const int4 yt = s_tab[dy];
                const int iy0 = y0 + yt.y, iy1 = y0 + yt.z;
                for (int dx = lane; dx < fs; dx += 32) {
                    const int sx = s_tab[dx].x;
                    const short2 xa = s_xa[dx];
                    int p[4];
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        const int u = sx + (q & 1);
                        const int ix = mirrored ? x0 + P - 1 - u : x0 + u, iy = (q & 2) ? iy1 : iy0;
                        int v = 0;
                        if ((q & 1) && xa.y == 0) { p[q] = 0; continue; }
                        if constexpr (WARP) {
                            // (ix, iy) is a pixel of V: its value from its four taps in the frame, 0 outside V
                            const sd_sample_warp* __restrict__ warps = maps;        // a warped launch's second parameter
                            p[q] = hog_warp_pixel(warps + sample, ix, iy, img, W, H, rs, rx, ry, rw, rh, &miss);
                            continue;
                        }
                        if ((unsigned)ix < (unsigned)W && (unsigned)iy < (unsigned)H) {
                            if (ix >= rx && ix < rx + rw && iy >= ry && iy < ry + rh) v = __ldg(img + (long long)(iy - ry) * rs + (ix - rx));
                            else miss = true;
                        }
                        p[q] = v;
                    }
                    const int t0 = p[0] * xa.x + p[1] * xa.y;
                    const int t1 = p[2] * xa.x + p[3] * xa.y;
                    s_patch[dy * pp + dx] = (uint8_t)hog_resize_out(yt.w, t0, t1);
                }
            }
        }
        if (miss && a.roi_miss) a.roi_miss[img_idx] = 1;
        if (a.patches) {
            __syncthreads();
            for (int i = tid; i < fs * fs; i += NT) {
                const int y = i / fs;
                a.patches[patch_id * fs * fs + i] = s_patch[y * pp + (i - y * fs)];
            }
        }
    }
    __syncthreads();

    // ---- S2: gradient + orientation arg-max per interior pixel (hog.c:631-672), in registers: the gradient of an 8-bit
    //      patch is a pair of integers in [-255, 255], its squared modulus an exact float integer whose correctly rounded
    //      root is the reference's sqrtf, and hog_bin decides the reference's arg-max -----------------------------------
    {
        // linear index over (interior row, run of 4 pixels): the run's three source rows come in as two words each and its
        // bins go out in one 32-bit store.  A row's last run may reach up to 3 pixels past the interior: they land in the
        // padding columns (x - 1 < pb), which nothing reads.
        const int iw = fs - 2, runs = (iw + 3) >> 2, nitem = iw * runs;
        const int pw = pp >> 2;                                    // row pitch in words
        for (int i = tid; i < nitem; i += NT) {
            const int y = i / runs, r = i - y * runs;              // pixels (y + 1, 4r + 1 .. 4r + 4)
            const unsigned* c = reinterpret_cast<const unsigned*>(s_patch) + (y + 1) * pw + r;
            const unsigned c0 = c[0], c1 = c[1], u0 = c[-pw], u1 = c[1 - pw], d0 = c[pw], d1 = c[pw + 1];
            unsigned bins = 0;
            float* gm = s_gmag + y * pm + 4 * r;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                // bytes k .. k + 2 of the centre row's 8, byte k + 1 of the rows above and below
                const int gx = byte_of(c0, c1, k + 2) - byte_of(c0, c1, k);
                const int gy = byte_of(d0, d1, k + 1) - byte_of(u0, u1, k + 1);
                const int g2 = gx * gx + gy * gy;
                const float g = __fsqrt_rn((float)g2);
                const int b = hog_bin(a.orient, K, gx, gy, g);
                bins |= (unsigned)(b & 0xff) << (8 * k);
                gm[k] = b < 0 ? 0.f : g;                           // no bin, no vote (hog.c:694): g = 0, or gx = 0 at K = 1
            }
            *reinterpret_cast<unsigned*>(s_bin + y * pb + 4 * r) = bins;
        }
    }
    if (a.bins) {
        __syncthreads();
        for (int idx = tid; idx < fs * fs; idx += NT) {
            const int y = idx / fs, x = idx - y * fs;
            const bool interior = x >= 1 && x <= fs - 2 && y >= 1 && y <= fs - 2;
            a.bins[patch_id * fs * fs + idx] = interior ? s_bin[(y - 1) * pb + x - 1] : (int8_t)-1;
        }
    }
    if (!a.A) return;                                             // sd_hog_debug: geometry, patches and bins only
    __syncthreads();

    // ---- S3: bilinear spatial vote (hog.c:697-724), separable:  hist[b][cj][ci] = sum_y wy[cj][y] * ( sum_x wx[ci][x] * g[y][x] * [bin[y][x] == b] ).
    //      Pass 1: one thread per (cell column ci, interior row y) walks the <= 2*cs pixels of that row that vote into ci and adds
    //      g * wx into ITS OWN column of T[bin][task] (bank == task mod 32: conflict free, no atomics, fixed order).  It takes
    //      the pixels in aligned pairs (x, x + 1), x odd: one 16-bit load of their bins and one 8-byte load of their weights.
    //      Pass 2: one thread per (bin b < K, cell) folds the rows with wy for bins b and b + K, one weight load for both.  The
    //      reference adds (g * wx) * wy per pixel in raster order; this is the same sum associated differently (~1e-7
    //      relative), deterministic, and every product and add is the dense kernel's (sd_hog_dense.cu) in its order.
    {
        const int nrow = fs - 2, ntask = nrow * nc, tpad = lay.tpad;
        for (int task = tid; task < ntask; task += NT) {
            const int ci = task / nrow, y = 1 + task - ci * nrow;
            const int xlo = s_lo[ci], xhi = s_hi[ci];
            // pixel x of this row and cell column: bin bp[x], modulus gp[x], weight wp[x]
            const int8_t* bp = s_bin + (y - 1) * pb - 1;
            const float* gp = s_gmag + (y - 1) * pm - 1;
            const float* wp = s_wcell + ci * pw - 1;
            float* T = s_T + task;
            for (int b = 0; b < 2 * K; ++b) T[b * tpad] = 0.f;        // T shares the staging area of S1: clear this column first
            // no bin: bin -1, modulus stored as 0 -> adds +0 to bin 0
            const auto vote = [&](int b, float p) { float* q = T + max(b, 0) * tpad; *q = __fadd_rn(*q, p); };
            int x = xlo;
            if (!(x & 1) && x <= xhi) { vote(bp[x], __fmul_rn(gp[x], wp[x])); ++x; }
            // both vote loops rolled: unrolled, they push S1's cold load loops of some schedules past 32 registers
#pragma unroll 1
            for (; x < xhi; x += 2) {
                const unsigned bb = *reinterpret_cast<const unsigned short*>(bp + x);
                const float2 w = *reinterpret_cast<const float2*>(wp + x);
                vote((int)(int8_t)bb, __fmul_rn(gp[x], w.x));
                vote((int)(int8_t)(bb >> 8), __fmul_rn(gp[x + 1], w.y));
            }
            if (x == xhi) vote(bp[x], __fmul_rn(gp[x], wp[x]));
        }
        __syncthreads();
        // Only the ntask columns that pass 1 cleared and filled are read here: hog_bintab_kernel keeps lo and hi inside the
        // interior [1, fs - 2], so rows ylo..yhi stay in column block ci.  The padding columns [ntask, tpad) still hold bytes
        // of the staged window (they were not cleared) and must never be read.
        // The histogram hist[b * cells + c] goes to the first 2K cells floats of this landmark's slice of the feature row
        // (which holds cells * dd >= 3K cells floats), where hog_normalise_kernel turns it into the features.
        float* __restrict__ out = a.A + (long long)sample * a.ld + (long long)lm * cells * a.dd;
        for (int i = tid; i < K * cells; i += NT) {
            const int b = i / cells, c = i - b * cells;
            const int cj = c / nc, ci = c - cj * nc;                  // cell row (y), cell column (x)
            const int ylo = s_lo[cj], yhi = s_hi[cj];
            const float* Tp = s_T + b * tpad + ci * nrow + (ylo - 1);
            const float* wy = s_wcell + cj * pw + (ylo - 1);
            float acc = 0.f, acc2 = 0.f;                              // bins b and b + K
#pragma unroll 1
            for (int y = ylo; y <= yhi; ++y) {
                const float w = *wy++;
                acc = __fadd_rn(acc, __fmul_rn(Tp[0], w));
                acc2 = __fadd_rn(acc2, __fmul_rn(Tp[K * tpad], w));
                ++Tp;
            }
            out[i] = acc;
            out[i + K * cells] = acc2;
        }
    }
}

// ---- S4-S8 of a batch of patches whose cell histograms hog_patch_kernel left in their feature slices: undirected cell
//      energy (hog.c:875-890), the block factors in double (hog.c:930-982), then per cell normalise, clamp at 0.2, project
//      and texture sums (hog_cell_features, hog.c:985-1053), stored per dimension transposed (adaptive_vlhog.hpp:168-174)
//      over the same slice, and the bias (:182-183).  `per_cta` patches per CTA, one thread per (patch, cell).  The factor
//      of a block (a square root and a division in double) is computed once per block, (nc + 1)^2 of them per patch, not
//      once for each of the up to four cells that use it, and the energies are widened to double once per cell.  Each CTA reads its
//      patches' whole histograms into shared memory before a barrier and writes features only after it, so the in-place
//      update is safe; slices start at any float offset (ld is any value >= D), so the loads and stores are scalar.
struct NormArgs {
    float* A;
    long long ld;
    int N, L, nc, K, dd, variant, per_cta;
};

// per patch: slice offset, histograms, energies (double), block factors (double)
__host__ __device__ inline int hog_norm_smem(int nc, int K, int per_cta)
{
    const int cells = nc * nc;
    return per_cta * (8 + 2 * K * cells * 4 + cells * 8 + (nc + 1) * (nc + 1) * 8);
}

template <int KT>
__global__ void __launch_bounds__(kHogThreads) hog_normalise_kernel(const NormArgs a)
{
    extern __shared__ __align__(16) unsigned char s_norm[];
    const int K = KT > 0 ? KT : a.K;
    const int nc = a.nc, nb = nc + 1, cells = nc * nc, blocks = nb * nb, hsz = 2 * K * cells, per_lm = cells * a.dd;
    const long long first = (long long)blockIdx.x * a.per_cta;
    const int np = (int)min((long long)a.per_cta, (long long)a.N * a.L - first);
    long long* s_slice = reinterpret_cast<long long*>(s_norm);   // [patch] offset of its slice in A
    double* s_energy = reinterpret_cast<double*>(s_slice + a.per_cta);   // [patch][cells]
    double* s_fac = s_energy + a.per_cta * cells;                 // [patch][block row jy][block column jx]
    float* s_hist = reinterpret_cast<float*>(s_fac + a.per_cta * blocks);   // [patch][2K][cells]
    for (int p = threadIdx.x; p < np; p += kHogThreads) {
        const long long id = first + p;
        const int sample = (int)(id / a.L), lm = (int)(id - (long long)sample * a.L);
        s_slice[p] = (long long)sample * a.ld + (long long)lm * per_lm;
        if (lm == 0) a.A[(long long)sample * a.ld + (long long)a.L * per_lm] = 1.0f;   // bias, outside every slice
    }
    __syncthreads();
    // asynchronous copies: every load of a thread is in flight at once (a load-then-store loop waits out the latency of
    // each one in turn, which took most of this kernel's time)
    for (int i = threadIdx.x; i < np * hsz; i += kHogThreads) {
        const int p = i / hsz;
        __pipeline_memcpy_async(s_hist + i, a.A + s_slice[p] + (i - p * hsz), sizeof(float));
    }
    __pipeline_commit();
    __pipeline_wait_prior(0);
    __syncthreads();
    for (int i = threadIdx.x; i < np * cells; i += kHogThreads) {
        const int p = i / cells, c = i - p * cells;
        s_energy[i] = (double)hog_cell_energy(s_hist + p * hsz + c, cells, K);
    }
    __syncthreads();
    // block (jx, jy): cell columns max(jx - 1, 0) and min(jx, nc - 1), rows likewise.  Factor q of cell (x, y) is block
    // (x + (q & 1), y + (q >> 1)), the block hog_cell_factors forms for it.
    for (int i = threadIdx.x; i < np * blocks; i += kHogThreads) {
        const int p = i / blocks, j = i - p * blocks;
        const int jy = j / nb, jx = j - jy * nb;
        s_fac[i] = hog_block_factor(s_energy + p * cells, nc, max(jx - 1, 0), min(jx, nc - 1), max(jy - 1, 0), min(jy, nc - 1));
    }
    __syncthreads();
    for (int i = threadIdx.x; i < np * cells; i += kHogThreads) {
        const int p = i / cells, c = i - p * cells;
        const int cj = c / nc, ci = c - cj * nc;                 // cell row (y), cell column (x)
        const double* F = s_fac + p * blocks + cj * nb + ci;
        const double fac[4] = {F[0], F[1], F[nb], F[nb + 1]};
        float* __restrict__ out = a.A + s_slice[p] + ci * nc + cj;   // per-dimension transpose
        hog_cell_features(fac, s_hist + p * hsz + c, cells, K, a.variant, [=](int d, float v) { out[d * cells] = v; });
    }
}

// the hog_patch_kernel instantiation of a configuration and its threads per CTA: a compiled-in schedule (DESIGN §4.1) or a run-time one
template <bool MIR, bool WARP>
decltype(&hog_patch_kernel<0, 0, 0, kHogThreads, MIR, WARP>) pick_hog_kernel(int K, int nc, int cs, int* threads)
{
    *threads = kHogThreads;
    if (nc == 5 && (K == 4 || K == 9)) {
#define SD_HOG_PICK(KK, CC, TT) if (K == KK && cs == CC) { *threads = TT; return hog_patch_kernel<KK, 5, CC, TT, MIR, WARP>; }
        SD_HOG_PICK(4, 11, 224) SD_HOG_PICK(4, 10, 160) SD_HOG_PICK(4, 8, 160) SD_HOG_PICK(4, 6, 128)
        SD_HOG_PICK(9, 11, 256) SD_HOG_PICK(9, 10, 160) SD_HOG_PICK(9, 8, 160) SD_HOG_PICK(9, 6, 128)
#undef SD_HOG_PICK
    }
    return K == 4 ? hog_patch_kernel<4, 0, 0, kHogThreads, MIR, WARP> : K == 9 ? hog_patch_kernel<9, 0, 0, kHogThreads, MIR, WARP>
                                                                             : hog_patch_kernel<0, 0, 0, kHogThreads, MIR, WARP>;
}

// d_warp (optional): the samples' warps (sd_hog_batch_warped); the launch then reads no mirrored bit
int launch_hog(sd_ctx* ctx, const sd_image_batch* images, const int32_t* d_image_index, bool mirrors, const sd_sample_warp* d_warp,
               const float* d_x, int64_t ldx, int N, int L, const sd_normalisation* eyes, const sd_hog_param* p, float* d_A,
               int64_t ld, int32_t* d_geometry, uint8_t* d_patches, int8_t* d_bins, uint8_t* d_face_degenerate = nullptr)
{
    SD_REQUIRE(ctx, images && images->d_data && d_x && p, "null argument");
    SD_REQUIRE(ctx, N >= 0 && L >= 1, "bad sample / landmark count");
    if (const int rc = sd_hog_check_config(ctx, __func__, p->variant, p->num_bins)) return rc;
    SD_REQUIRE(ctx, p->num_cells >= 1 && p->cell_size >= 1, "bad cell configuration");
    const int fs = p->num_cells * p->cell_size;
    SD_REQUIRE(ctx, fs > 3 && fs <= 256, "resized patch must be 4..256 px (hog.c:545-546 asserts > 3)");
    SD_REQUIRE(ctx, (fs + p->cell_size / 2) / p->cell_size == p->num_cells, "hogWidth != num_cells");
    SD_REQUIRE(ctx, ldx >= 2 * L, "ldx < 2L");
    if (N == 0) return SD_OK;
    // eyes == NULL (or kind 0): the fixed-patch HogTransform of the hello-world example (examples/landmark_detection.cpp:
    // 195-261): half = num_cells * (cell_size / 2), no resize.  The kernel's resize stage is the identity when the patch is
    // already num_cells * cell_size wide, which holds for even cell sizes; an odd cell size would change the HOG grid of
    // the un-resized patch and is rejected.
    const bool fixed = !eyes || eyes->kind == 0;
    int fixed_half = 0;
    if (fixed) {
        fixed_half = p->num_cells * (p->cell_size / 2);
        SD_REQUIRE(ctx, 2 * fixed_half == fs, "the fixed-patch HogTransform needs an even cell_size (patch == num_cells * cell_size)");
    } else if (eyes->kind != 1) {
        return sd_fail(ctx, SD_ERR_INVALID, "unknown normalisation kind");
    }

    HogArgs a;
    sd_eyes_dev eyes_dev;
    memset(&eyes_dev, 0, sizeof(eyes_dev));
    int rc = fixed ? SD_OK : sd_eyes_to_dev(ctx, eyes, L, &eyes_dev);
    if (rc) return rc;
    a.images = images->d_data;
    a.width = images->width; a.height = images->height; a.row_stride = images->row_stride;
    a.image_stride = images->image_stride; a.image_count = images->count;
    a.image_index = d_image_index;
    a.roi = images->d_roi;
    a.roi_miss = images->d_roi_miss;
    a.frames = images->d_frames;
    if (!d_image_index) SD_REQUIRE(ctx, images->count >= N, "fewer images than samples and no image index");
    a.x = d_x; a.ldx = ldx; a.N = N; a.L = L;
    a.variant = p->variant; a.nc = p->num_cells; a.cs = p->cell_size; a.K = p->num_bins; a.fs = fs;
    a.dd = sd_hog_dd(p->num_bins, p->variant);
    a.A = d_A; a.ld = ld;
    if (d_A) SD_REQUIRE(ctx, ld >= (int64_t)L * a.nc * a.nc * a.dd + 1, "ld < feature length");
    // every argument check before the first launch: a rejected configuration queues no work
    const HogSmem lay = hog_smem_layout(fs, a.nc, a.K);
    const int cells = a.nc * a.nc;
    NormArgs na;
    na.A = d_A; na.ld = ld; na.N = N; na.L = L; na.nc = a.nc; na.K = a.K; na.dd = a.dd; na.variant = a.variant;
    na.per_cta = cells < kHogThreads ? kHogThreads / cells : 1;  // one thread per cell of the CTA's patches
    const int norm_smem = hog_norm_smem(a.nc, a.K, na.per_cta);
    SD_REQUIRE(ctx, lay.total <= 227 * 1024 && norm_smem <= 227 * 1024, "HOG configuration needs more than 227 KB of shared memory");
    const long long blocks = (long long)N * L;
    SD_REQUIRE(ctx, blocks < 2147483647LL, "too many patches for one launch");
    a.geometry = d_geometry; a.patches = d_patches; a.bins = d_bins;
    a.status = reinterpret_cast<int*>(ctx->d_scratch) + 1;   // the projection's own status word: bit 0 empty patch, bit 1 bad image index

    hog_orientations(a.K, a.orient);   // hog.c:195-204

    // per-sample tables (half size, cv::resize taps), the per-launch spatial binning table and, warped, the checked warps
    const size_t tab_bytes = (size_t)N * sizeof(int) + (size_t)N * 5 * fs * sizeof(int) + (size_t)(a.nc * fs + 2 * a.nc) * sizeof(float);
    const size_t geom_bytes = d_warp ? sd_round16(tab_bytes) + (size_t)N * sizeof(sd_sample_warp) : tab_bytes;
    int* d_half = (int*)sd_workspace(ctx, SD_WS_GEOM, geom_bytes);
    if (!d_half) return SD_ERR_CUDA;
    int* d_rtab = d_half + N;
    float* d_btab = reinterpret_cast<float*>(d_rtab + (size_t)N * 5 * fs);
    HogWarpCheck wc{};
    if (d_warp) {
        wc = HogWarpCheck{d_warp, reinterpret_cast<sd_sample_warp*>(reinterpret_cast<uint8_t*>(d_half) + sd_round16(tab_bytes)), d_image_index,
                          images->count, images->width, images->height, images->d_frames};
    }
    hog_geometry_kernel<<<N, 64, 0, ctx->stream>>>(d_x, ldx, N, L, eyes_dev, p->relative_patch_size, fixed_half, fs, d_half, d_rtab, a.status,
                                                    d_face_degenerate, wc);
    SD_LAUNCH_CHECK(ctx, "hog_geometry_kernel");
    hog_bintab_kernel<<<1, 256, 0, ctx->stream>>>(fs, a.nc, a.cs, lay.pw, d_btab);
    SD_LAUNCH_CHECK(ctx, "hog_bintab_kernel");
    a.half = d_half;
    a.rtab = d_rtab;
    a.btab = d_btab;

    // tensor maps of the frame batch for the TMA staging route: whole frames resident, 16-byte aligned base and pitches
    HogMaps maps;
    memset(&maps, 0, sizeof(maps));
    a.tma_count = 0;
    if (!d_warp && !images->d_roi && (images->image_stride % 16) == 0 && (images->count == 1 || images->image_stride > 0)) {
        // classes are usable up to the first one that cannot be encoded
        for (int c = 0; c < kTmaClasses && hog_tma_box(c) <= 256; ++c) {
            if (!hog_frame_map(images, hog_tma_box(c), hog_tma_box(c), &maps.m[c])) break;
            a.tma_count = c + 1;
        }
    }

    // a warp table takes the WARP instantiations; otherwise an index that may carry SD_SAMPLE_MIRRORED takes the MIR ones, and
    // without one (or for detect's face_frame) the launch is the unmirrored kernel
    int threads = kHogThreads;
    const auto launch = [&](auto kern, const auto& src) -> int {
        SD_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, lay.total));
        kern<<<(unsigned)blocks, threads, lay.total, ctx->stream>>>(a, src);
        SD_LAUNCH_CHECK(ctx, "hog_patch_kernel");
        return SD_OK;
    };
    // Default shared-memory carve-out: the maximum one ran the four detect levels no faster (5.84 ms both, 4096 faces, one
    // H100 80GB HBM3 at a 400 W power limit; measured at 256 threads, when registers, not shared memory, bounded the CTAs per
    // SM at fs = 55 / 50 / 40).  With the default, every compiled schedule reaches the CTAs per SM that the thread and
    // shared-memory limits allow (DESIGN §4.1; counted per SM on an H100 and equal to cudaOccupancyMaxActiveBlocksPerMultiprocessor).
    rc = d_warp ? launch(pick_hog_kernel<false, true>(a.K, a.nc, a.cs, &threads), wc.out)
                : launch(mirrors && d_image_index ? pick_hog_kernel<true, false>(a.K, a.nc, a.cs, &threads)
                                                  : pick_hog_kernel<false, false>(a.K, a.nc, a.cs, &threads), maps);
    if (rc) return rc;
    if (!d_A) return SD_OK;
    auto norm = a.K == 4 ? hog_normalise_kernel<4> : a.K == 9 ? hog_normalise_kernel<9> : hog_normalise_kernel<0>;
    SD_CUDA(ctx, cudaFuncSetAttribute(norm, cudaFuncAttributeMaxDynamicSharedMemorySize, norm_smem));
    norm<<<(unsigned)sd_div_up(blocks, na.per_cta), kHogThreads, norm_smem, ctx->stream>>>(na);
    SD_LAUNCH_CHECK(ctx, "hog_normalise_kernel");
    return SD_OK;
}

}  // namespace

int sd_hog_batch_unmirrored(sd_ctx* ctx, const sd_image_batch* images, const int32_t* d_image_index, const float* d_x, int64_t ldx,
                            int num_samples, int num_landmarks, const sd_normalisation* eyes, const sd_hog_param* p, float* d_A,
                            int64_t ld, uint8_t* d_face_degenerate, const sd_sample_warp* d_warp)
{
    if (num_samples == 0) return SD_OK;
    SD_REQUIRE(ctx, d_A, "null output");
    return launch_hog(ctx, images, d_image_index, false, d_warp, d_x, ldx, num_samples, num_landmarks, eyes, p, d_A, ld, nullptr, nullptr,
                      nullptr, d_face_degenerate);
}

namespace {
// cv::cvtColor(BGR2GRAY), 8-bit, OpenCV >= 3 fixed point (15-bit coefficients): HBM-bound, 3 bytes read + 1 written per
// pixel.  A thread converts four pixels: three aligned 32-bit loads, one 32-bit store (scalar path for the row tail or
// unaligned rows).
__global__ void bgr2gray_kernel(const uint8_t* __restrict__ bgr, int width, int height, long long srow, long long simg, int count,
                                uint8_t* __restrict__ gray, long long drow, long long dimg, int vec_ok)
{
    const int groups = (width + 3) >> 2;
    const long long total = (long long)count * height * groups;
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const int g = (int)(t % groups);
        const long long ry = t / groups;
        const int y = (int)(ry % height);
        const long long im = ry / height;
        const uint8_t* s = bgr + im * simg + (long long)y * srow + 12 * g;
        uint8_t* d = gray + im * dimg + (long long)y * drow + 4 * g;
        const int x0 = 4 * g;
        if (vec_ok && x0 + 4 <= width) {
            const uint32_t w0 = *reinterpret_cast<const uint32_t*>(s), w1 = *reinterpret_cast<const uint32_t*>(s + 4),
                           w2 = *reinterpret_cast<const uint32_t*>(s + 8);
            // bytes: w0 = B0 G0 R0 B1 | w1 = G1 R1 B2 G2 | w2 = R2 B3 G3 R3   (little endian)
            const uint32_t b0 = w0 & 255, g0 = (w0 >> 8) & 255, r0 = (w0 >> 16) & 255, b1 = w0 >> 24;
            const uint32_t g1 = w1 & 255, r1 = (w1 >> 8) & 255, b2 = (w1 >> 16) & 255, g2 = w1 >> 24;
            const uint32_t r2 = w2 & 255, b3 = (w2 >> 8) & 255, g3 = (w2 >> 16) & 255, r3 = w2 >> 24;
            const uint32_t y0 = sd_bgr_to_gray(b0, g0, r0), y1 = sd_bgr_to_gray(b1, g1, r1);
            const uint32_t y2 = sd_bgr_to_gray(b2, g2, r2), y3 = sd_bgr_to_gray(b3, g3, r3);
            *reinterpret_cast<uint32_t*>(d) = y0 | (y1 << 8) | (y2 << 16) | (y3 << 24);
        } else {
            for (int k = 0; k < 4 && x0 + k < width; ++k) d[k] = (uint8_t)sd_bgr_to_gray(s[3 * k], s[3 * k + 1], s[3 * k + 2]);
        }
    }
}

// sd_bgr2gray_images: frame f0 + blockIdx.y of an sd_hog_images batch of B, G, R bytes (per-frame table src_frames, or equally sized
// frames src_frame image_stride elements apart) into its grey frame (per-frame table dst_frames, or dst_image_stride bytes apart
// at a pitch of dst_pitch).  The CTAs of a frame walk its rows, the threads a row's pixels.
__global__ void bgr2gray_images_kernel(const uint8_t* __restrict__ src, const sd_hog_image* __restrict__ src_frames, sd_hog_image src_frame,
                                       long long image_stride, int f0, uint8_t* __restrict__ dst, const sd_frame* __restrict__ dst_frames,
                                       long long dst_image_stride, int dst_pitch)
{
    const int f = f0 + blockIdx.y;
    sd_hog_image d;
    if (src_frames) {
        d = src_frames[f];
    } else {
        d = src_frame;
        d.offset += (long long)f * image_stride;
    }
    const long long o = dst_frames ? dst_frames[f].offset : (long long)f * dst_image_stride;
    const long long pitch = dst_frames ? dst_frames[f].row_stride : dst_pitch;
    const long long cs = d.channel_stride;
    for (int y = blockIdx.x; y < d.height; y += gridDim.x) {
        const uint8_t* s = src + d.offset + (long long)y * d.row_stride;
        uint8_t* g = dst + o + y * pitch;
        for (int x = threadIdx.x; x < d.width; x += blockDim.x) {
            const uint8_t* p = s + (long long)x * d.pixel_stride;
            g[x] = (uint8_t)sd_bgr_to_gray(__ldg(p), __ldg(p + cs), __ldg(p + 2 * cs));
        }
    }
}
}  // namespace

extern "C" {

int sd_hog_feature_length(int num_landmarks, const sd_hog_param* p)
{
    if (!p) return -1;
    const int dd = sd_hog_dd(p->num_bins, p->variant);
    return num_landmarks * p->num_cells * p->num_cells * dd + 1;
}

int sd_hog_batch(sd_ctx* ctx, const sd_image_batch* images, const int32_t* d_image_index, const float* d_x,
                 int64_t ldx, int num_samples, int num_landmarks, const sd_normalisation* eyes,
                 const sd_hog_param* p, float* d_A, int64_t ld)
{
    if (!ctx) return SD_ERR_INVALID;
    if (num_samples == 0) return SD_OK;
    SD_REQUIRE(ctx, d_A, "null output");
    return launch_hog(ctx, images, d_image_index, true, nullptr, d_x, ldx, num_samples, num_landmarks, eyes, p, d_A, ld,
                      nullptr, nullptr, nullptr);
}

int sd_hog_batch_warped(sd_ctx* ctx, const sd_image_batch* images, const int32_t* d_image_index, const float* d_x, int64_t ldx,
                        int num_samples, int num_landmarks, const sd_normalisation* eyes, const sd_hog_param* p,
                        const sd_sample_warp* d_warp, float* d_A, int64_t ld)
{
    if (!ctx) return SD_ERR_INVALID;
    SD_REQUIRE(ctx, images && !images->d_roi, "a warped batch must hold whole frames (no d_roi)");
    SD_REQUIRE(ctx, d_warp, "null warp table");
    return sd_hog_batch_unmirrored(ctx, images, d_image_index, d_x, ldx, num_samples, num_landmarks, eyes, p, d_A, ld, nullptr, d_warp);
}

int sd_hog_debug(sd_ctx* ctx, const sd_image_batch* images, const int32_t* d_image_index, const float* d_x,
                 int64_t ldx, int num_samples, int num_landmarks, const sd_normalisation* eyes,
                 const sd_hog_param* p, int32_t* d_geometry, uint8_t* d_patches, int8_t* d_bins)
{
    if (!ctx) return SD_ERR_INVALID;
    return launch_hog(ctx, images, d_image_index, true, nullptr, d_x, ldx, num_samples, num_landmarks, eyes, p, nullptr, 0,
                      d_geometry, d_patches, d_bins);
}

int sd_hog_debug_warped(sd_ctx* ctx, const sd_image_batch* images, const int32_t* d_image_index, const float* d_x, int64_t ldx,
                        int num_samples, int num_landmarks, const sd_normalisation* eyes, const sd_hog_param* p,
                        const sd_sample_warp* d_warp, int32_t* d_geometry, uint8_t* d_patches, int8_t* d_bins)
{
    if (!ctx) return SD_ERR_INVALID;
    SD_REQUIRE(ctx, images && !images->d_roi, "a warped batch must hold whole frames (no d_roi)");
    SD_REQUIRE(ctx, d_warp, "null warp table");
    return launch_hog(ctx, images, d_image_index, false, d_warp, d_x, ldx, num_samples, num_landmarks, eyes, p, nullptr, 0,
                      d_geometry, d_patches, d_bins);
}

int sd_bgr2gray(sd_ctx* ctx, const uint8_t* d_bgr, int width, int height, int64_t bgr_row_stride, int64_t bgr_image_stride,
                int count, uint8_t* d_gray, int64_t gray_row_stride, int64_t gray_image_stride)
{
    if (!ctx) return SD_ERR_INVALID;
    SD_REQUIRE(ctx, count >= 0 && width > 0 && height > 0, "bad argument");
    if (count == 0) return SD_OK;
    SD_REQUIRE(ctx, d_bgr && d_gray && bgr_row_stride >= 3LL * width && gray_row_stride >= width, "bad argument");
    const int vec_ok = ((reinterpret_cast<uintptr_t>(d_bgr) | reinterpret_cast<uintptr_t>(d_gray) | (uintptr_t)bgr_row_stride |
                         (uintptr_t)bgr_image_stride | (uintptr_t)gray_row_stride | (uintptr_t)gray_image_stride) & 3) == 0;
    const long long total = (long long)count * height * ((width + 3) >> 2);
    const int blocks = (int)(sd_div_up(total, 256) < 16LL * ctx->sm_count ? sd_div_up(total, 256) : 16LL * ctx->sm_count);
    bgr2gray_kernel<<<blocks, 256, 0, ctx->stream>>>(d_bgr, width, height, bgr_row_stride, bgr_image_stride, count, d_gray,
                                                     gray_row_stride, gray_image_stride, vec_ok);
    SD_LAUNCH_CHECK(ctx, "bgr2gray_kernel");
    return SD_OK;
}

int sd_bgr2gray_images(sd_ctx* ctx, const sd_hog_images* bgr, void* d_buf, size_t* bytes, sd_image_batch* out)
{
    if (!ctx) return SD_ERR_INVALID;
    SD_REQUIRE(ctx, bgr && bytes && bgr->count >= 1 && bgr->d_data, "bad argument");
    SD_REQUIRE(ctx, bgr->dtype == SD_HOG_U8 && bgr->channels == 3, "frames must be SD_HOG_U8 with 3 channels (B, G, R)");
    const int count = bgr->count;
    HogPyramidFrames fr;
    if (const int rc = sd_hog_read_image_frames(ctx, __func__, bgr, 0, &fr)) return rc;
    std::vector<sd_frame> desc(count);
    bool uniform = true;
    const size_t gray = sd_gray_layout(fr.frames.data(), count, desc.data(), &uniform);
    const size_t need = gray + (uniform ? 0 : (size_t)count * sizeof(sd_frame));   // the descriptors follow the grey frames
    if (!d_buf) {
        *bytes = need;
        return SD_OK;
    }
    SD_REQUIRE(ctx, out && sd_aligned(d_buf, 16) && *bytes >= need,
               "d_buf must be 16-byte aligned and hold the size the query gives; out must not be NULL");
    uint8_t* base = static_cast<uint8_t*>(d_buf);
    const sd_image_batch ib = sd_gray_batch(base, desc.data(), count, uniform, reinterpret_cast<const sd_frame*>(base + gray));
    if (!uniform)
        SD_CUDA(ctx, cudaMemcpyAsync(base + gray, desc.data(), (size_t)count * sizeof(sd_frame), cudaMemcpyHostToDevice, ctx->stream));
    int max_h = 0;
    for (const sd_frame& d : desc) max_h = std::max(max_h, d.height);
    const unsigned rows = (unsigned)std::min(max_h, 1024);
    for (int f0 = 0; f0 < count; f0 += 65535) {
        const dim3 grid(rows, (unsigned)std::min(count - f0, 65535));
        bgr2gray_images_kernel<<<grid, 128, 0, ctx->stream>>>(static_cast<const uint8_t*>(bgr->d_data), bgr->d_frames, bgr->frame,
                                                             bgr->image_stride, f0, base, ib.d_frames, (long long)desc[0].row_stride * desc[0].height,
                                                             desc[0].row_stride);
        SD_LAUNCH_CHECK(ctx, "bgr2gray_images_kernel");
    }
    *out = ib;
    return SD_OK;
}

}  // extern "C"
