// Deformable part models over HOG pyramids (sd_hog_distance_transform, sd_hog_distance_transform_exact, sd_hog_part_scores,
// sd_hog_part_placements, sd_hog_part_placements_mapped): the bounded and the exact generalised distance transforms of part score
// maps, the star model's score maps, and the part boxes of each detection.
//
//   dt_tile_kernel        one CTA per 32 x 32 output tile of one plane: the tile's rows with R rows of halo above and below and
//                         R columns either side are staged in shared memory, pass X runs over every staged row (32 columns),
//                         pass Y over the tile.  Both passes take candidates in ascending displacement through dt_take.
//   part_scores_kernel    one thread per root score: the root score plus each part's transformed score at its anchor.
//   part_place_kernel     one warp per (detection, part): the rule of dt_tile_kernel at the one anchor, through dt_take again,
//                         so that the placement is bit for bit the transform's.
//
//   dt_exact_kernel<X>    (sd_hog_distance_transform_exact) one warp per block of 32 rows of one plane, a row per lane: the
//                         block is staged through shared memory 32 columns at a time, so every global access is a whole row
//                         segment; each lane builds its row's lower envelope and then writes the row's values.
//   dt_exact_kernel<Y>    one warp per block of 32 adjacent columns, a column per lane: every step reads and writes 32
//                         consecutive floats, in place on pass X's output.
//   part_mapped_kernel    (sd_hog_part_placements_mapped) one thread per (detection, part): the transform's value and
//                         placement at the anchor.
//
// Every kernel walks a flat list of work items with a grid-stride loop over blockIdx.x; no count is bound by gridDim.y / z.
// There are no atomics: each output element is written by one thread.
//
// Scratch (SD_WS_PARTS): the cost tables or deformations, the per-map first tiles or line blocks of a table route, the
// placements' per-detection map index, and the envelopes of lines too long for shared memory.
#include "sd_internal.cuh"

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>
#include <map>
#include <vector>

namespace {

constexpr int kT = 32;                 // output tile side of the transform
constexpr int kThreads = 256;
constexpr int kNone = INT_MIN;         // "no candidate chosen"
constexpr int kScoreTile = kThreads * 4;
constexpr int kPlaceWarps = 4;

// The rule's update, shared by every kernel: a non-NaN candidate replaces the current best when there is none yet or when it
// is strictly greater.  Called in ascending displacement order, the choice is the smallest displacement that reaches the max.
__device__ __forceinline__ void dt_take(float cand, int k, float& best, int& arg)
{
    if (!isnan(cand) && (arg == kNone || cand > best)) {
        best = cand;
        arg = k;
    }
}

// ---- the transform ----------------------------------------------------------------------------------------------------------

struct DtArgs {
    const float* in;
    float* out;
    int2* place;                  // may be null
    const sd_hog_grid* grids;     // null: equally sized maps
    int width, height;            // equally sized maps
    int num_maps, P, R;
    const float* costs;           // [P][2][2R + 1]: cx then cy
    const long long* tile0;       // table route: each map's first tile
    long long total_tiles;
};

__global__ void __launch_bounds__(kThreads) dt_tile_kernel(const __grid_constant__ DtArgs a)
{
    extern __shared__ __align__(16) unsigned char smem[];
    const int R = a.R, span = kT + 2 * R, taps = 2 * R + 1;
    float* s_in = reinterpret_cast<float*>(smem);                 // [span][span]
    float* s_t = s_in + span * span;                              // [span][kT]
    float* s_c = s_t + span * kT;                                 // [2][taps]
    signed char* s_dx = reinterpret_cast<signed char*>(s_c + 2 * taps);   // [span][kT]; -128: none
    const int tid = threadIdx.x;

    for (long long t = blockIdx.x; t < a.total_tiles; t += gridDim.x) {
        int m, w, h;
        long long base, obase, local;
        if (a.grids) {
            m = sd_find_last_le(0, a.num_maps - 1, t, [&](int i) { return __ldg(a.tile0 + i); });
            const sd_hog_grid g = a.grids[m];
            w = g.width; h = g.height; base = g.offset; obase = g.out_offset;
            local = t - __ldg(a.tile0 + m);
        } else {
            w = a.width; h = a.height;
            const long long per = (long long)a.P * ((w + kT - 1) / kT) * ((h + kT - 1) / kT);
            m = (int)(t / per);
            local = t - (long long)m * per;
            base = obase = (long long)m * a.P * w * h;
        }
        const int tx = (w + kT - 1) / kT, ty = (h + kT - 1) / kT;
        const int k = (int)(local / ((long long)tx * ty));
        const int r = (int)(local - (long long)k * tx * ty);
        const int x0 = (r % tx) * kT, y0 = (r / tx) * kT;
        const long long plane = (long long)k * w * h;
        const float* in = a.in + base + plane;

        __syncthreads();                                          // the previous tile is done with shared memory
        for (int i = tid; i < 2 * taps; i += kThreads) s_c[i] = __ldg(a.costs + (size_t)k * 2 * taps + i);
        const int ylo = max(0, y0 - R), yhi = min(h, y0 + kT + R);
        const int xlo = max(0, x0 - R), xhi = min(w, x0 + kT + R);
        const int cols = xhi - xlo;
        for (int i = tid; i < (yhi - ylo) * cols; i += kThreads) {
            const int y = ylo + i / cols, x = xlo + i % cols;
            s_in[(y - y0 + R) * span + (x - x0 + R)] = __ldg(in + (long long)y * w + x);
        }
        __syncthreads();

        // pass X over every staged row, the tile's columns
        const int xe = min(kT, w - x0);
        for (int i = tid; i < (yhi - ylo) * kT; i += kThreads) {
            const int c = i & (kT - 1), y = ylo + i / kT;
            if (c >= xe) continue;
            const int u = x0 + c;
            const float* row = s_in + (y - y0 + R) * span + (c + R);
            float best = -INFINITY;
            int arg = kNone;
            for (int d = -R; d <= R; ++d)
                if (u + d >= 0 && u + d < w) dt_take(__fsub_rn(row[d], s_c[d + R]), d, best, arg);
            s_t[(y - y0 + R) * kT + c] = best;
            s_dx[(y - y0 + R) * kT + c] = arg == kNone ? (signed char)-128 : (signed char)arg;
        }
        __syncthreads();

        // pass Y over the tile
        const int ye = min(kT, h - y0);
        for (int i = tid; i < ye * kT; i += kThreads) {
            const int c = i & (kT - 1), rr = i / kT;
            if (c >= xe) continue;
            const int u = x0 + c, v = y0 + rr;
            float best = -INFINITY;
            int arg = kNone;
            for (int e = -R; e <= R; ++e)
                if (v + e >= 0 && v + e < h) dt_take(__fsub_rn(s_t[(rr + e + R) * kT + c], s_c[taps + e + R]), e, best, arg);
            const long long o = obase + plane + (long long)v * w + u;
            a.out[o] = best;
            if (a.place) {
                int2 p = make_int2(-1, -1);
                if (arg != kNone) {
                    const int dx = s_dx[(rr + arg + R) * kT + c];
                    if (dx != -128) p = make_int2(u + dx, v + arg);
                }
                a.place[o] = p;
            }
        }
    }
}

// ---- the exact transform --------------------------------------------------------------------------------------------------------
// The header's rule, in its operation order: every double operation is an explicit _rn intrinsic, so nvcc contracts nothing
// into an FMA and tests/hog_dt_exact_ref.py reproduces each rounding.

constexpr int kExactWarps = 4;        // warps per CTA of the exact passes
constexpr int kEnvShared = 32;        // lines of at most this many positions keep their envelopes in shared memory
constexpr int kTileStride = 33;       // pass X's staging tiles: 32 x 32 with a padded row, conflict-free either way
constexpr int kEnvBytes = 20;         // per envelope entry: z (double), index, score, pass X's placement (int32 each)

// cost of displacement d: (float)((double) w0 d d + (double) w1 d), the bounded call's cost-table formula
__device__ __forceinline__ float dt_exact_cost(double a, double b, int d)
{
    const double x = (double)d;
    return __double2float_rn(__dadd_rn(__dmul_rn(__dmul_rn(a, x), x), __dmul_rn(b, x)));
}

// the first position r (> q) owns against q: p* = (((f(q) - f(r)) + a (r - q)(r + q)) + b (r - q)) / ((a + a)(r - q))
__device__ __forceinline__ double dt_exact_meet(int q, float fq, int r, float fr, double a, double b)
{
    const double dq = (double)(r - q), sq = (double)((long long)(r - q) * (long long)(r + q));
    const double num = __dadd_rn(__dadd_rn(__dsub_rn((double)fq, (double)fr), __dmul_rn(a, sq)), __dmul_rn(b, dq));
    return __ddiv_rn(num, __dmul_rn(__dadd_rn(a, a), dq));
}

struct ExactArgs {
    const float* in;              // pass X: the maps at each grid's offset; pass Y: d_values at out_offset
    float* out;                   // d_values
    int* place;                   // d_place as int32 (u, v) pairs, or null; pass X leaves each row's owner in u
    const sd_hog_grid* grids;     // null: equally sized maps
    int width, height;            // equally sized maps
    int num_maps, P;
    const float* deformation;     // [P][4]
    const long long* item0;       // table route: each map's first line block
    long long total_items;
    unsigned char* env;           // scratch route: nmax entries per lane of every warp of the grid; null: shared memory
    int nmax;                     // the longest line of the pass
};

// One pass over every line of every plane: kY = false, rows (pass X); kY = true, columns (pass Y).  A lane's envelope is
// entries [0, cnt): owner index v, its score f, and z, the point past which it owns (z[0] = -inf); the entries of a warp are
// interleaved, entry i of lane l at i * 32 + l.
template <bool kY>
__global__ void __launch_bounds__(kExactWarps * 32) dt_exact_kernel(const __grid_constant__ ExactArgs a)
{
    extern __shared__ __align__(16) unsigned char smem[];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const size_t tile_bytes = kY ? 0 : 2 * 32 * kTileStride * sizeof(float);
    unsigned char* wsm = smem + (size_t)wid * (tile_bytes + (a.env ? 0 : (size_t)kEnvBytes * a.nmax * 32));
    float* tile = reinterpret_cast<float*>(wsm);                 // pass X: 32 x 32 scores, then 32 x 32 owners
    int* otile = reinterpret_cast<int*>(tile + 32 * kTileStride);
    const long long gw = (long long)blockIdx.x * kExactWarps + wid;
    unsigned char* env = a.env ? a.env + (size_t)gw * kEnvBytes * a.nmax * 32 : wsm + tile_bytes;
    double* ez = reinterpret_cast<double*>(env) + lane;
    int* ev = reinterpret_cast<int*>(env + (size_t)8 * a.nmax * 32) + lane;
    float* ef = reinterpret_cast<float*>(ev + a.nmax * 32);
    int* ex = ev + 2 * a.nmax * 32;

    for (long long it = gw; it < a.total_items; it += (long long)gridDim.x * kExactWarps) {
        int m, w, h;
        long long ibase, obase, local;
        if (a.grids) {
            m = sd_find_last_le(0, a.num_maps - 1, it, [&](int i) { return __ldg(a.item0 + i); });
            const sd_hog_grid g = a.grids[m];
            w = g.width; h = g.height; obase = g.out_offset; ibase = kY ? g.out_offset : g.offset;
            local = it - __ldg(a.item0 + m);
        } else {
            w = a.width; h = a.height;
            const long long per = (long long)a.P * (((kY ? w : h) + 31) / 32);
            m = (int)(it / per);
            local = it - (long long)m * per;
            ibase = obase = (long long)m * a.P * w * h;
        }
        const int n = kY ? h : w, lines = kY ? w : h, blocks = (lines + 31) / 32;
        const int k = (int)(local / blocks), l0 = (int)(local - (long long)k * blocks) * 32, line = l0 + lane;
        const bool live = line < lines;
        const long long plane = (long long)k * w * h;
        const float* src = a.in + ibase + plane;
        float* dst = a.out + obase + plane;
        int* place = a.place ? a.place + 2 * (obase + plane) : nullptr;
        const double wa = (double)__ldg(a.deformation + 4 * k + (kY ? 2 : 0)), wb = (double)__ldg(a.deformation + 4 * k + (kY ? 3 : 1));
        // position i of this lane's line, as a float offset from the plane
        auto at = [&](int i) { return kY ? (long long)i * w + line : (long long)line * w + i; };

        // the envelope, candidates in ascending position
        int cnt = 0;
        for (int i0 = 0; i0 < n; i0 += 32) {
            const int len = min(32, n - i0);
            if (!kY) {
                __syncwarp();
                for (int r = 0; r < 32 && l0 + r < lines; ++r)
                    if (lane < len) tile[r * kTileStride + lane] = src[(long long)(l0 + r) * w + i0 + lane];
                __syncwarp();
            }
            if (!live) continue;
            for (int j = 0; j < len; ++j) {
                const int q = i0 + j;
                const float fq = kY ? src[at(q)] : tile[lane * kTileStride + j];
                if (!isfinite(fq)) continue;
                double s = -INFINITY;
                while (cnt > 0) {
                    s = dt_exact_meet(ev[(cnt - 1) * 32], ef[(cnt - 1) * 32], q, fq, wa, wb);
                    if (s > ez[(cnt - 1) * 32]) break;
                    --cnt;
                    s = -INFINITY;
                }
                ez[cnt * 32] = s;
                ev[cnt * 32] = q;
                ef[cnt * 32] = fq;
                if (kY && place) ex[cnt * 32] = place[2 * at(q)];
                ++cnt;
            }
        }

        // the values: position p belongs to the last entry whose z is below p
        int e = 0;
        for (int i0 = 0; i0 < n; i0 += 32) {
            const int len = min(32, n - i0);
            if (!kY) __syncwarp();                                // every lane is done reading the tiles
            if (live)
                for (int j = 0; j < len; ++j) {
                    const int p = i0 + j;
                    float val = -INFINITY;
                    int q = -1;
                    if (cnt > 0) {
                        while (e + 1 < cnt && ez[(e + 1) * 32] < (double)p) ++e;
                        q = ev[e * 32];
                        val = __fsub_rn(ef[e * 32], dt_exact_cost(wa, wb, q - p));
                    }
                    if (kY) {
                        dst[at(p)] = val;
                        if (place) reinterpret_cast<int2*>(place)[at(p)] = q < 0 ? make_int2(-1, -1) : make_int2(ex[e * 32], q);
                    } else {
                        tile[lane * kTileStride + j] = val;
                        otile[lane * kTileStride + j] = q;
                    }
                }
            if (!kY) {
                __syncwarp();
                for (int r = 0; r < 32 && l0 + r < lines; ++r)
                    if (lane < len) {
                        const long long o = (long long)(l0 + r) * w + i0 + lane;
                        dst[o] = tile[r * kTileStride + lane];
                        if (place) place[2 * o] = otile[r * kTileStride + lane];
                    }
                __syncwarp();
            }
        }
    }
}

// ---- the star model's scores --------------------------------------------------------------------------------------------------

struct ScoreArgs {
    const float* root;
    const float* parts;
    float* out;
    const sd_hog_part_map* maps;
    const int32_t* anchors;       // [Q][P][2]
    const long long* tile0;
    int num_maps, Q, P, pad_x, pad_y, part_pad_x, part_pad_y;
    long long total_tiles;
};

__global__ void __launch_bounds__(kThreads) part_scores_kernel(const __grid_constant__ ScoreArgs a)
{
    for (long long t = blockIdx.x; t < a.total_tiles; t += gridDim.x) {
        const int m = sd_find_last_le(0, a.num_maps - 1, t, [&](int i) { return __ldg(a.tile0 + i); });
        const sd_hog_part_map d = a.maps[m];
        const long long plane = (long long)d.width * d.height, n = a.Q * plane;
        const long long e0 = (t - __ldg(a.tile0 + m)) * kScoreTile, e1 = min(e0 + kScoreTile, n);
        const long long pplane = (long long)d.part_width * d.part_height;
        for (long long e = e0 + threadIdx.x; e < e1; e += kThreads) {
            const int q = (int)(e / plane);
            const long long rem = e - q * plane;
            const int y = (int)(rem / d.width), x = (int)(rem - (long long)y * d.width);
            float total = __ldg(a.root + d.root_offset + e);
            bool outside = false;
            for (int p = 0; p < a.P; ++p) {
                const int2 an = __ldg(reinterpret_cast<const int2*>(a.anchors) + q * a.P + p);
                const long long u0 = 2LL * (x - a.pad_x) + an.x + a.part_pad_x, v0 = 2LL * (y - a.pad_y) + an.y + a.part_pad_y;
                if (u0 < 0 || u0 >= d.part_width || v0 < 0 || v0 >= d.part_height) {
                    outside = true;
                    continue;
                }
                total = __fadd_rn(total, __ldg(a.parts + d.part_offset + (long long)(q * a.P + p) * pplane + v0 * d.part_width + u0));
            }
            a.out[d.out_offset + e] = outside ? -INFINITY : total;
        }
    }
}

// ---- the part placements of detections ---------------------------------------------------------------------------------------

struct PlaceArgs {
    const float* parts;           // the part score maps (before the transform)
    const sd_hog_part_map* maps;
    const int32_t* anchors;
    const float* costs;           // [Q * P][2][2R + 1]
    const sd_hog_detection* det;
    const int32_t* count;
    const int32_t* slot_map;      // num_frames x max_det: the table entry of each detection
    sd_hog_part_placement* out;
    int num_frames, max_det, P, R, cell, pfw, pfh, pad_x, pad_y, part_pad_x, part_pad_y;
};

__global__ void __launch_bounds__(kPlaceWarps * 32) part_place_kernel(const __grid_constant__ PlaceArgs a)
{
    extern __shared__ __align__(16) unsigned char smem[];
    const int taps = 2 * a.R + 1, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    float* s_t = reinterpret_cast<float*>(smem) + wid * 2 * taps;  // [taps] row values, then [taps] their dx
    int* s_dx = reinterpret_cast<int*>(s_t + taps);
    const long long items = (long long)a.num_frames * a.max_det * a.P;
    for (long long it = (long long)blockIdx.x * kPlaceWarps + wid; it < items; it += (long long)gridDim.x * kPlaceWarps) {
        const long long slot = it / a.P;
        const int p = (int)(it - slot * a.P);
        const int f = (int)(slot / a.max_det), k = (int)(slot - (long long)f * a.max_det);
        if (k >= __ldg(a.count + f)) continue;                    // uniform over the warp
        const sd_hog_detection det = a.det[slot];
        const sd_hog_part_map d = a.maps[__ldg(a.slot_map + slot)];
        const int q = det.filter, kp = q * a.P + p;
        const int2 an = __ldg(reinterpret_cast<const int2*>(a.anchors) + kp);
        const long long u0 = 2LL * (det.cell_x - a.pad_x) + an.x + a.part_pad_x, v0 = 2LL * (det.cell_y - a.pad_y) + an.y + a.part_pad_y;
        sd_hog_part_placement r;
        r.u = r.v = -1;
        r.term = -INFINITY;
        r.x = r.y = r.w = r.h = 0;
        if (u0 >= 0 && u0 < d.part_width && v0 >= 0 && v0 < d.part_height) {
            const int w = d.part_width, h = d.part_height, u = (int)u0, v = (int)v0;
            const float* plane = a.parts + d.part_offset + (long long)kp * w * h;
            const float* cx = a.costs + (size_t)kp * 2 * taps;
            const float* cy = cx + taps;
            // pass X at column u of each row v + e that the rule reads
            for (int i = lane; i < taps; i += 32) {
                const int y = v + i - a.R;
                if (y < 0 || y >= h) continue;
                const float* row = plane + (long long)y * w + u;
                float best = -INFINITY;
                int arg = kNone;
                for (int dd = -a.R; dd <= a.R; ++dd)
                    if (u + dd >= 0 && u + dd < w) dt_take(__fsub_rn(__ldg(row + dd), __ldg(cx + dd + a.R)), dd, best, arg);
                s_t[i] = best;
                s_dx[i] = arg;
            }
            __syncwarp();
            if (lane == 0) {
                float best = -INFINITY;
                int arg = kNone;
                for (int e = -a.R; e <= a.R; ++e)
                    if (v + e >= 0 && v + e < h) dt_take(__fsub_rn(s_t[e + a.R], __ldg(cy + e + a.R)), e, best, arg);
                r.term = best;
                if (arg != kNone && s_dx[arg + a.R] != kNone) {
                    r.u = u + s_dx[arg + a.R];
                    r.v = v + arg;
                    const sd_box64 b = sd_window_box(r.u, r.v, a.part_pad_x, a.part_pad_y, a.pfw, a.pfh, a.cell, d.frame_w, d.frame_h,
                                                     d.part_level_w, d.part_level_h);
                    r.x = (int)b.x0; r.y = (int)b.y0; r.w = (int)(b.x1 - b.x0); r.h = (int)(b.y1 - b.y0);
                }
            }
            __syncwarp();
        }
        if (lane == 0) a.out[it] = r;
    }
}

struct MappedArgs {
    const float* values;          // the transform's values and (u, v) placements, at the table's part_offset
    const int2* place;
    const sd_hog_part_map* maps;
    const int32_t* anchors;
    const sd_hog_detection* det;
    const int32_t* count;
    const int32_t* slot_map;
    sd_hog_part_placement* out;
    int num_frames, max_det, P, cell, pfw, pfh, pad_x, pad_y, part_pad_x, part_pad_y;
};

__global__ void __launch_bounds__(kThreads) part_mapped_kernel(const __grid_constant__ MappedArgs a)
{
    const long long items = (long long)a.num_frames * a.max_det * a.P;
    for (long long it = (long long)blockIdx.x * kThreads + threadIdx.x; it < items; it += (long long)gridDim.x * kThreads) {
        const long long slot = it / a.P;
        const int p = (int)(it - slot * a.P);
        const int f = (int)(slot / a.max_det), k = (int)(slot - (long long)f * a.max_det);
        if (k >= __ldg(a.count + f)) continue;
        const sd_hog_detection det = a.det[slot];
        const sd_hog_part_map d = a.maps[__ldg(a.slot_map + slot)];
        const int kp = det.filter * a.P + p;
        const int2 an = __ldg(reinterpret_cast<const int2*>(a.anchors) + kp);
        const long long u0 = 2LL * (det.cell_x - a.pad_x) + an.x + a.part_pad_x, v0 = 2LL * (det.cell_y - a.pad_y) + an.y + a.part_pad_y;
        sd_hog_part_placement r;
        r.u = r.v = -1;
        r.term = -INFINITY;
        r.x = r.y = r.w = r.h = 0;
        if (u0 >= 0 && u0 < d.part_width && v0 >= 0 && v0 < d.part_height) {
            const long long o = d.part_offset + ((long long)kp * d.part_height + v0) * d.part_width + u0;
            const int2 pl = a.place[o];
            r.term = a.values[o];
            if (pl.x >= 0) {
                r.u = pl.x;
                r.v = pl.y;
                const sd_box64 b = sd_window_box(r.u, r.v, a.part_pad_x, a.part_pad_y, a.pfw, a.pfh, a.cell, d.frame_w, d.frame_h,
                                                 d.part_level_w, d.part_level_h);
                r.x = (int)b.x0; r.y = (int)b.y0; r.w = (int)(b.x1 - b.x0); r.h = (int)(b.y1 - b.y0);
            }
        }
        a.out[it] = r;
    }
}

// cost tables of num_planes deformations: cx[d] = (float)((double)w0 d^2 + (double)w1 d), cy alike with w2, w3
bool cost_tables(const float* h_def, int num_planes, int R, std::vector<float>& costs)
{
    const int taps = 2 * R + 1;
    costs.resize((size_t)num_planes * 2 * taps);
    for (int k = 0; k < num_planes; ++k)
        for (int axis = 0; axis < 2; ++axis)
            for (int d = -R; d <= R; ++d) {
                const double c = (double)h_def[4 * k + 2 * axis] * d * d + (double)h_def[4 * k + 2 * axis + 1] * d;
                const float f = (float)c;
                if (!std::isfinite(f)) return false;
                costs[((size_t)k * 2 + axis) * taps + d + R] = f;
            }
    return true;
}

int check_model(sd_ctx* ctx, const sd_hog_part_model* m)
{
    SD_REQUIRE(ctx, m && m->d_anchors && sd_aligned(m->d_anchors, 8), "null model or anchors not 8-byte aligned");
    SD_REQUIRE(ctx, m->num_parts >= 1 && m->num_parts <= SD_HOG_PART_MAX_PARTS, "num_parts must be in [1, SD_HOG_PART_MAX_PARTS]");
    SD_REQUIRE(ctx, m->num_components >= 1 && (long long)m->num_components * m->num_parts <= SD_HOG_FILTER_MAX_BANK,
               "num_components must be >= 1 with num_components * num_parts <= SD_HOG_FILTER_MAX_BANK");
    if (const int rc = sd_hog_check_filter(ctx, __func__, m->filter_w, m->filter_h, m->pad_x, m->pad_y)) return rc;
    return sd_hog_check_filter(ctx, __func__, m->part_w, m->part_h, m->part_pad_x, m->part_pad_y);
}

// the score tiles of each map of a part table (first tile per map) and the check every call makes of the table's sizes
int part_tiles(sd_ctx* ctx, const std::vector<sd_hog_part_map>& table, int Q, std::vector<long long>& tile0, long long* total)
{
    tile0.resize(table.size());
    long long tiles = 0;
    for (size_t i = 0; i < table.size(); ++i) {
        const sd_hog_part_map& d = table[i];
        SD_REQUIRE(ctx, d.width >= 0 && d.height >= 0 && d.part_width >= 0 && d.part_height >= 0, "a map's size is negative");
        SD_REQUIRE(ctx, d.root_offset >= 0 && d.part_offset >= 0 && d.out_offset >= 0, "a map's offset is negative");
        tile0[i] = tiles;
        tiles += ((long long)Q * d.width * d.height + kScoreTile - 1) / kScoreTile;
    }
    *total = tiles;
    return SD_OK;
}

// The checks both placement calls make of their table and detections, with the detections read back once: slot_map receives
// each detection's table entry, *work the number of detections.
int placement_slots(sd_ctx* ctx, const sd_hog_part_map* d_maps, int num_maps, const sd_hog_part_model* model, int cell_size,
                    const sd_hog_detection* d_det, const int32_t* d_count, int num_frames, int max_detections,
                    std::vector<int32_t>& slot_map, long long* work)
{
    const int Q = model->num_components;
    std::vector<sd_hog_part_map> table;
    if (num_maps > 0)
        if (const int rc = sd_fetch_table(ctx, d_maps, num_maps, table)) return rc;
    std::vector<long long> tile0;
    long long tiles = 0;
    if (const int rc = part_tiles(ctx, table, Q, tile0, &tiles)) return rc;
    std::map<std::pair<int, int>, int> index;
    for (int i = 0; i < num_maps; ++i) {
        const sd_hog_part_map& d = table[i];
        SD_REQUIRE(ctx, d.frame >= 0 && d.frame < num_frames, "a map's frame is out of range");
        SD_REQUIRE(ctx, d.frame_w >= 1 && d.frame_h >= 1 && d.part_level_w >= 1 && d.part_level_h >= 1,
                   "a map's frame or part level is smaller than 1 x 1");
        SD_REQUIRE(ctx, index.emplace(std::make_pair(d.frame, d.level), i).second, "two maps share one (frame, level)");
        SD_REQUIRE(ctx, sd_window_boxes_fit_int32(d.part_width, d.part_height, model->part_pad_x, model->part_pad_y, model->part_w,
                                                  model->part_h, cell_size, d.frame_w, d.frame_h, d.part_level_w, d.part_level_h),
                   "a map's part boxes do not fit in int32");
    }
    // the detections, read back once: each must come from a map of the table
    const size_t slots = (size_t)num_frames * max_detections;
    std::vector<int32_t> count(num_frames);
    std::vector<sd_hog_detection> det(slots);
    SD_CUDA(ctx, cudaMemcpyAsync(count.data(), d_count, sizeof(int32_t) * num_frames, cudaMemcpyDeviceToHost, ctx->stream));
    SD_CUDA(ctx, cudaMemcpyAsync(det.data(), d_det, sizeof(sd_hog_detection) * slots, cudaMemcpyDeviceToHost, ctx->stream));
    SD_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    slot_map.assign(slots, 0);
    *work = 0;
    for (int f = 0; f < num_frames; ++f) {
        SD_REQUIRE(ctx, count[f] >= 0 && count[f] <= max_detections, "a frame's detection count is outside [0, max_detections]");
        for (int k = 0; k < count[f]; ++k) {
            const sd_hog_detection& r = det[(size_t)f * max_detections + k];
            const auto it = index.find(std::make_pair(f, (int)r.level));
            SD_REQUIRE(ctx, it != index.end(), "a detection's (frame, level) is not in the table");
            const sd_hog_part_map& d = table[it->second];
            SD_REQUIRE(ctx, r.filter >= 0 && r.filter < Q && r.cell_x >= 0 && r.cell_x < d.width && r.cell_y >= 0 && r.cell_y < d.height,
                       "a detection's filter or score position is not one of its map");
            slot_map[(size_t)f * max_detections + k] = it->second;
            ++*work;
        }
    }
    return SD_OK;
}

// the first line block of each map of a table, in pass X (rows) or pass Y (columns)
long long exact_items(const std::vector<sd_hog_grid>& table, int P, bool columns, std::vector<long long>& item0)
{
    long long items = 0;
    item0.resize(table.size());
    for (size_t i = 0; i < table.size(); ++i) {
        item0[i] = items;
        items += (long long)P * sd_div_up(columns ? table[i].width : table[i].height, 32);
    }
    return items;
}

}  // namespace

extern "C" {

int sd_hog_distance_transform(sd_ctx* ctx, const sd_hog_grids* maps, int num_planes, const float* h_deformation, int max_displacement,
                              float* d_values, int32_t* d_place)
{
    if (!ctx) return SD_ERR_INVALID;
    SD_REQUIRE(ctx, maps && h_deformation && d_values, "null argument");
    SD_REQUIRE(ctx, maps->count >= 0, "negative map count");
    SD_REQUIRE(ctx, maps->count == 0 || (maps->d_features && sd_aligned(maps->d_features, 4)), "maps must be non-null and 4-byte aligned");
    SD_REQUIRE(ctx, sd_aligned(d_values, 4) && sd_aligned(d_place, 8), "values must be 4-byte aligned and placements 8-byte aligned");
    SD_REQUIRE(ctx, num_planes >= 1 && num_planes <= SD_HOG_FILTER_MAX_BANK, "num_planes must be in [1, SD_HOG_FILTER_MAX_BANK]");
    SD_REQUIRE(ctx, max_displacement >= 0 && max_displacement <= SD_HOG_PART_MAX_DISPLACEMENT,
               "max_displacement must be in [0, SD_HOG_PART_MAX_DISPLACEMENT]");
    const int R = max_displacement, taps = 2 * R + 1;
    std::vector<float> costs;
    SD_REQUIRE(ctx, cost_tables(h_deformation, num_planes, R, costs), "a cost table entry is not finite");
    if (maps->count == 0) return SD_OK;
    int max_w = 0, max_h = 0;
    std::vector<sd_hog_grid> table;
    if (const int rc = sd_read_hog_grids(ctx, __func__, maps, &max_w, &max_h, maps->d_grids ? &table : nullptr)) return rc;
    std::vector<long long> tile0;
    long long tiles = 0;
    if (maps->d_grids) {
        tile0.resize(table.size());
        for (size_t i = 0; i < table.size(); ++i) {
            tile0[i] = tiles;
            tiles += (long long)num_planes * sd_div_up(table[i].width, kT) * sd_div_up(table[i].height, kT);
        }
    } else {
        tiles = (long long)maps->count * num_planes * sd_div_up(maps->width, kT) * sd_div_up(maps->height, kT);
    }

    const size_t cost_bytes = sd_round16(sizeof(float) * costs.size());
    unsigned char* ws = static_cast<unsigned char*>(sd_workspace(ctx, SD_WS_PARTS, cost_bytes + sizeof(long long) * tile0.size()));
    if (!ws) return SD_ERR_CUDA;
    DtArgs a;
    memset(&a, 0, sizeof(a));
    a.in = maps->d_features;
    a.out = d_values;
    a.place = reinterpret_cast<int2*>(d_place);
    a.grids = maps->d_grids;
    a.width = maps->width;
    a.height = maps->height;
    a.num_maps = maps->count;
    a.P = num_planes;
    a.R = R;
    a.costs = reinterpret_cast<const float*>(ws);
    a.tile0 = reinterpret_cast<const long long*>(ws + cost_bytes);
    a.total_tiles = tiles;
    SD_CUDA(ctx, cudaMemcpyAsync(ws, costs.data(), sizeof(float) * costs.size(), cudaMemcpyHostToDevice, ctx->stream));
    if (!tile0.empty())
        SD_CUDA(ctx, cudaMemcpyAsync(ws + cost_bytes, tile0.data(), sizeof(long long) * tile0.size(), cudaMemcpyHostToDevice, ctx->stream));
    const int span = kT + 2 * R;
    const int smem = (span * span + span * kT + 2 * taps) * (int)sizeof(float) + span * kT;
    SD_CUDA(ctx, cudaFuncSetAttribute(dt_tile_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    const int grid = (int)std::min<long long>(tiles, 16LL * ctx->sm_count);
    dt_tile_kernel<<<grid, kThreads, smem, ctx->stream>>>(a);
    SD_LAUNCH_CHECK(ctx, "dt_tile_kernel");
    return SD_OK;
}

int sd_hog_part_scores(sd_ctx* ctx, const float* d_root, const float* d_parts, const sd_hog_part_map* d_maps, int num_maps,
                       const sd_hog_part_model* model, float* d_out)
{
    if (!ctx) return SD_ERR_INVALID;
    if (const int rc = check_model(ctx, model)) return rc;
    SD_REQUIRE(ctx, num_maps >= 0, "negative map count");
    SD_REQUIRE(ctx, num_maps == 0 || (d_root && d_parts && d_maps && d_out), "null argument");
    SD_REQUIRE(ctx, sd_aligned(d_root, 4) && sd_aligned(d_parts, 4) && sd_aligned(d_out, 4) && sd_aligned(d_maps, 8),
               "scores must be 4-byte aligned and the map table 8-byte aligned");
    if (num_maps == 0) return SD_OK;
    std::vector<sd_hog_part_map> table;
    if (const int rc = sd_fetch_table(ctx, d_maps, num_maps, table)) return rc;
    std::vector<long long> tile0;
    long long tiles = 0;
    if (const int rc = part_tiles(ctx, table, model->num_components, tile0, &tiles)) return rc;
    if (tiles == 0) return SD_OK;
    long long* ws = static_cast<long long*>(sd_workspace(ctx, SD_WS_PARTS, sizeof(long long) * tile0.size()));
    if (!ws) return SD_ERR_CUDA;
    SD_CUDA(ctx, cudaMemcpyAsync(ws, tile0.data(), sizeof(long long) * tile0.size(), cudaMemcpyHostToDevice, ctx->stream));
    ScoreArgs a;
    memset(&a, 0, sizeof(a));
    a.root = d_root;
    a.parts = d_parts;
    a.out = d_out;
    a.maps = d_maps;
    a.anchors = model->d_anchors;
    a.tile0 = ws;
    a.num_maps = num_maps;
    a.Q = model->num_components;
    a.P = model->num_parts;
    a.pad_x = model->pad_x; a.pad_y = model->pad_y;
    a.part_pad_x = model->part_pad_x; a.part_pad_y = model->part_pad_y;
    a.total_tiles = tiles;
    const int grid = (int)std::min<long long>(tiles, 16LL * ctx->sm_count);
    part_scores_kernel<<<grid, kThreads, 0, ctx->stream>>>(a);
    SD_LAUNCH_CHECK(ctx, "part_scores_kernel");
    return SD_OK;
}

int sd_hog_part_placements(sd_ctx* ctx, const float* d_parts, const sd_hog_part_map* d_maps, int num_maps, const sd_hog_part_model* model,
                           const float* h_deformation, int max_displacement, int cell_size, const sd_hog_detection* d_det,
                           const int32_t* d_count, int num_frames, int max_detections, sd_hog_part_placement* d_out)
{
    if (!ctx) return SD_ERR_INVALID;
    if (const int rc = check_model(ctx, model)) return rc;
    SD_REQUIRE(ctx, h_deformation && d_det && d_count && d_out && (num_maps == 0 || (d_parts && d_maps)), "null argument");
    SD_REQUIRE(ctx, sd_aligned(d_parts, 4) && sd_aligned(d_maps, 8) && sd_aligned(d_det, 4) && sd_aligned(d_count, 4) &&
                        sd_aligned(d_out, 4),
               "scores, detections, counts and output must be 4-byte aligned, the map table 8-byte aligned");
    SD_REQUIRE(ctx, num_maps >= 0, "negative map count");
    SD_REQUIRE(ctx, num_frames >= 1, "num_frames must be >= 1");
    SD_REQUIRE(ctx, max_detections >= 1 && max_detections <= SD_HOG_DETECT_MAX_CANDIDATES,
               "max_detections must be in [1, SD_HOG_DETECT_MAX_CANDIDATES]");
    SD_REQUIRE(ctx, cell_size >= 1 && cell_size <= kDenseMaxCell, "cell_size must be in [1,32]");
    SD_REQUIRE(ctx, max_displacement >= 0 && max_displacement <= SD_HOG_PART_MAX_DISPLACEMENT,
               "max_displacement must be in [0, SD_HOG_PART_MAX_DISPLACEMENT]");
    const int Q = model->num_components, P = model->num_parts, R = max_displacement;
    std::vector<float> costs;
    SD_REQUIRE(ctx, cost_tables(h_deformation, Q * P, R, costs), "a cost table entry is not finite");
    std::vector<int32_t> slot_map;
    long long work = 0;
    if (const int rc = placement_slots(ctx, d_maps, num_maps, model, cell_size, d_det, d_count, num_frames, max_detections, slot_map,
                                       &work))
        return rc;
    if (work == 0) return SD_OK;
    const size_t slots = slot_map.size();

    const size_t cost_bytes = sd_round16(sizeof(float) * costs.size());
    unsigned char* ws = static_cast<unsigned char*>(sd_workspace(ctx, SD_WS_PARTS, cost_bytes + sizeof(int32_t) * slots));
    if (!ws) return SD_ERR_CUDA;
    SD_CUDA(ctx, cudaMemcpyAsync(ws, costs.data(), sizeof(float) * costs.size(), cudaMemcpyHostToDevice, ctx->stream));
    SD_CUDA(ctx, cudaMemcpyAsync(ws + cost_bytes, slot_map.data(), sizeof(int32_t) * slots, cudaMemcpyHostToDevice, ctx->stream));
    PlaceArgs a;
    memset(&a, 0, sizeof(a));
    a.parts = d_parts;
    a.maps = d_maps;
    a.anchors = model->d_anchors;
    a.costs = reinterpret_cast<const float*>(ws);
    a.det = d_det;
    a.count = d_count;
    a.slot_map = reinterpret_cast<const int32_t*>(ws + cost_bytes);
    a.out = d_out;
    a.num_frames = num_frames;
    a.max_det = max_detections;
    a.P = P;
    a.R = R;
    a.cell = cell_size;
    a.pfw = model->part_w; a.pfh = model->part_h;
    a.pad_x = model->pad_x; a.pad_y = model->pad_y;
    a.part_pad_x = model->part_pad_x; a.part_pad_y = model->part_pad_y;
    const long long items = (long long)slots * P;
    const int grid = (int)std::min<long long>((items + kPlaceWarps - 1) / kPlaceWarps, 16LL * ctx->sm_count);
    const int smem = kPlaceWarps * 2 * (2 * R + 1) * (int)sizeof(float);
    part_place_kernel<<<grid, kPlaceWarps * 32, smem, ctx->stream>>>(a);
    SD_LAUNCH_CHECK(ctx, "part_place_kernel");
    return SD_OK;
}

int sd_hog_distance_transform_exact(sd_ctx* ctx, const sd_hog_grids* maps, int num_planes, const float* h_deformation, float* d_values,
                                    int32_t* d_place)
{
    if (!ctx) return SD_ERR_INVALID;
    SD_REQUIRE(ctx, maps && h_deformation && d_values, "null argument");
    SD_REQUIRE(ctx, maps->count >= 0, "negative map count");
    SD_REQUIRE(ctx, maps->count == 0 || (maps->d_features && sd_aligned(maps->d_features, 4)), "maps must be non-null and 4-byte aligned");
    SD_REQUIRE(ctx, sd_aligned(d_values, 4) && sd_aligned(d_place, 8), "values must be 4-byte aligned and placements 8-byte aligned");
    SD_REQUIRE(ctx, num_planes >= 1 && num_planes <= SD_HOG_FILTER_MAX_BANK, "num_planes must be in [1, SD_HOG_FILTER_MAX_BANK]");
    for (int i = 0; i < 4 * num_planes; ++i)
        SD_REQUIRE(ctx, std::isfinite(h_deformation[i]) && (i % 2 == 1 || h_deformation[i] > 0),
                   "every deformation weight must be finite, with w0 > 0 and w2 > 0");
    if (maps->count == 0) return SD_OK;
    int max_w = 0, max_h = 0;
    std::vector<sd_hog_grid> table;
    if (const int rc = sd_read_hog_grids(ctx, __func__, maps, &max_w, &max_h, maps->d_grids ? &table : nullptr)) return rc;
    std::vector<long long> item0[2];
    long long items[2];
    for (int y = 0; y < 2; ++y)
        items[y] = maps->d_grids ? exact_items(table, num_planes, y == 1, item0[y])
                                 : (long long)maps->count * num_planes * sd_div_up(y ? maps->width : maps->height, 32);
    if (items[0] == 0) return SD_OK;

    // scratch: the deformations, each pass's first line blocks, then the envelopes of a pass whose lines do not fit in shared
    // memory (kEnvBytes per position of the longest line, for each lane of each warp of the grid; at most kEnvBudget bytes
    // unless one CTA needs more)
    constexpr size_t kEnvBudget = size_t(256) << 20;
    const int nmax[2] = {max_w, max_h};
    int grid[2];
    size_t env_at = sd_round16(sizeof(float) * 4 * num_planes), items_at[2];
    for (int y = 0; y < 2; ++y) {
        items_at[y] = env_at;
        env_at += sd_round16(sizeof(long long) * item0[y].size());
    }
    size_t env_bytes = 0;
    for (int y = 0; y < 2; ++y) {
        const size_t per_cta = (size_t)kExactWarps * 32 * kEnvBytes * nmax[y];
        long long ctas = std::min<long long>(sd_div_up(items[y], kExactWarps), 8LL * ctx->sm_count);
        if (nmax[y] > kEnvShared) {
            ctas = std::max<long long>(1, std::min<long long>(ctas, (long long)(kEnvBudget / per_cta)));
            env_bytes = std::max(env_bytes, (size_t)ctas * per_cta);
        }
        grid[y] = (int)ctas;
    }
    unsigned char* ws = static_cast<unsigned char*>(sd_workspace(ctx, SD_WS_PARTS, env_at + env_bytes));
    if (!ws) return SD_ERR_CUDA;
    SD_CUDA(ctx, cudaMemcpyAsync(ws, h_deformation, sizeof(float) * 4 * num_planes, cudaMemcpyHostToDevice, ctx->stream));
    for (int y = 0; y < 2; ++y)
        if (!item0[y].empty())
            SD_CUDA(ctx, cudaMemcpyAsync(ws + items_at[y], item0[y].data(), sizeof(long long) * item0[y].size(), cudaMemcpyHostToDevice,
                                         ctx->stream));
    for (int y = 0; y < 2; ++y) {
        ExactArgs a;
        memset(&a, 0, sizeof(a));
        a.in = y ? d_values : maps->d_features;
        a.out = d_values;
        a.place = d_place;
        a.grids = maps->d_grids;
        a.width = maps->width;
        a.height = maps->height;
        a.num_maps = maps->count;
        a.P = num_planes;
        a.deformation = reinterpret_cast<const float*>(ws);
        a.item0 = reinterpret_cast<const long long*>(ws + items_at[y]);
        a.total_items = items[y];
        a.nmax = nmax[y];
        a.env = nmax[y] > kEnvShared ? ws + env_at : nullptr;
        const int smem = kExactWarps * ((y ? 0 : 2 * 32 * kTileStride * (int)sizeof(float)) + (a.env ? 0 : kEnvBytes * 32 * nmax[y]));
        if (y) {
            SD_CUDA(ctx, cudaFuncSetAttribute(dt_exact_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
            dt_exact_kernel<true><<<grid[y], kExactWarps * 32, smem, ctx->stream>>>(a);
            SD_LAUNCH_CHECK(ctx, "dt_exact_kernel<Y>");
        } else {
            SD_CUDA(ctx, cudaFuncSetAttribute(dt_exact_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
            dt_exact_kernel<false><<<grid[y], kExactWarps * 32, smem, ctx->stream>>>(a);
            SD_LAUNCH_CHECK(ctx, "dt_exact_kernel<X>");
        }
    }
    return SD_OK;
}

int sd_hog_part_placements_mapped(sd_ctx* ctx, const float* d_values, const int32_t* d_place, const sd_hog_part_map* d_maps,
                                  int num_maps, const sd_hog_part_model* model, int cell_size, const sd_hog_detection* d_det,
                                  const int32_t* d_count, int num_frames, int max_detections, sd_hog_part_placement* d_out)
{
    if (!ctx) return SD_ERR_INVALID;
    if (const int rc = check_model(ctx, model)) return rc;
    SD_REQUIRE(ctx, d_det && d_count && d_out && (num_maps == 0 || (d_values && d_place && d_maps)), "null argument");
    SD_REQUIRE(ctx, sd_aligned(d_values, 4) && sd_aligned(d_place, 8) && sd_aligned(d_maps, 8) && sd_aligned(d_det, 4) &&
                        sd_aligned(d_count, 4) && sd_aligned(d_out, 4),
               "values, detections, counts and output must be 4-byte aligned, the placements and the map table 8-byte aligned");
    SD_REQUIRE(ctx, num_maps >= 0, "negative map count");
    SD_REQUIRE(ctx, num_frames >= 1, "num_frames must be >= 1");
    SD_REQUIRE(ctx, max_detections >= 1 && max_detections <= SD_HOG_DETECT_MAX_CANDIDATES,
               "max_detections must be in [1, SD_HOG_DETECT_MAX_CANDIDATES]");
    SD_REQUIRE(ctx, cell_size >= 1 && cell_size <= kDenseMaxCell, "cell_size must be in [1,32]");
    std::vector<int32_t> slot_map;
    long long work = 0;
    if (const int rc = placement_slots(ctx, d_maps, num_maps, model, cell_size, d_det, d_count, num_frames, max_detections, slot_map,
                                       &work))
        return rc;
    if (work == 0) return SD_OK;
    const size_t slots = slot_map.size();
    int32_t* ws = static_cast<int32_t*>(sd_workspace(ctx, SD_WS_PARTS, sizeof(int32_t) * slots));
    if (!ws) return SD_ERR_CUDA;
    SD_CUDA(ctx, cudaMemcpyAsync(ws, slot_map.data(), sizeof(int32_t) * slots, cudaMemcpyHostToDevice, ctx->stream));
    MappedArgs a;
    memset(&a, 0, sizeof(a));
    a.values = d_values;
    a.place = reinterpret_cast<const int2*>(d_place);
    a.maps = d_maps;
    a.anchors = model->d_anchors;
    a.det = d_det;
    a.count = d_count;
    a.slot_map = ws;
    a.out = d_out;
    a.num_frames = num_frames;
    a.max_det = max_detections;
    a.P = model->num_parts;
    a.cell = cell_size;
    a.pfw = model->part_w; a.pfh = model->part_h;
    a.pad_x = model->pad_x; a.pad_y = model->pad_y;
    a.part_pad_x = model->part_pad_x; a.part_pad_y = model->part_pad_y;
    const long long items = (long long)slots * model->num_parts;
    const int grid = (int)std::min<long long>((items + kThreads - 1) / kThreads, 16LL * ctx->sm_count);
    part_mapped_kernel<<<grid, kThreads, 0, ctx->stream>>>(a);
    SD_LAUNCH_CHECK(ctx, "part_mapped_kernel");
    return SD_OK;
}

}  // extern "C"
