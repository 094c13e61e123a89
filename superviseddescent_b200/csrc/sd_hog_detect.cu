// Detections from HOG filter scores (sd_hog_detections): the candidates of every frame above a threshold, their boxes in frame
// pixels, and greedy non-maximum suppression, for a batch of score maps in one asynchronous call.
//
// Every candidate has a 64-bit key, (order-preserving score key << 32) | ~rank, where rank is its frame-local enumeration rank
// (the map's place in the table, then q, y, x).  Keys are unique within a frame, and a larger key comes first in the rule's
// order, so every step below is an exact integer operation on keys and the result does not depend on tiling or atomics.
//
//   1. det_count_kernel     one pass over all scores: each frame's candidate count (integer atomics).
//   2. det_hist_kernel /    only for frames with more than max_candidates candidates, and only when some frame of the call can
//      det_pick_kernel      have that many: a radix select of the max_candidates-th largest key, 8 bits a pass, at most 8
//                           passes; a frame leaves the select as soon as all keys of its current prefix are taken.
//   3. det_compact_kernel   one pass: the keys >= the frame's cut (all candidates of a frame that does not overflow) go to the
//                           frame's list in scratch, in any order (warp-aggregated slots).
//   4. det_nms_kernel       one CTA per frame: a bitonic sort of the list in shared memory, every box from (map, q, y, x) by
//                           the integer rule, then greedy suppression over a removed-bitmask: the next live candidate is kept
//                           and tests its box against all later ones in parallel, (kept) x (list / threads) box tests in all.
//
// Scratch (SD_WS_DETECT): num_frames x max_candidates keys, a 256-bin histogram, a small state and one int32 per frame, and three
// int32 per map (its first tile, its first rank, and its place in the frame-grouped map list).  It does not grow with the number
// of scores.
#include "sd_internal.cuh"

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>
#include <vector>

namespace {

constexpr int kThreads = 256;                 // select kernels
constexpr int kTile = kThreads * 16;          // scores of one map per tile
constexpr int kNmsThreads = 1024;

struct FrameState {
    unsigned long long above;    // candidates of the frame
    unsigned long long cut;      // keys >= cut are selected
    unsigned long long prefix;   // radix select: the digits decided so far
    unsigned int need;           // radix select: keys still to take below the prefix
    unsigned int fill;           // keys the compaction has written
    int active;                  // radix select still running
};

struct DetArgs {
    const float* scores;
    const sd_hog_score_map* maps;
    int num_maps, num_frames;
    const int* tile0;            // per map: its first tile
    const unsigned* rank0;       // per map: frame-local rank of its first score
    const int* fmaps;            // map indices grouped by frame, in table order
    const int* fmap0;            // num_frames + 1: each frame's first entry of fmaps
    int total_tiles;
    int Q, cell, fw, fh, pad_x, pad_y;
    float threshold;
    double overlap;
    int max_c, max_det;
    FrameState* state;
    unsigned* hist;              // num_frames x 256
    unsigned long long* keys;    // num_frames x max_c
    sd_hog_detection* out;
    int32_t* count;
    int64_t* above;
};

// order-preserving: a larger float gives a larger key; -0 and +0 give one key
__device__ __forceinline__ unsigned score_key(float s)
{
    const unsigned b = __float_as_uint(s == 0.f ? 0.f : s);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

__device__ __forceinline__ unsigned long long cand_key(float s, unsigned rank)
{
    return ((unsigned long long)score_key(s) << 32) | (0xFFFFFFFFu - rank);
}

// the tile's map and its range of scores [e0, e1) in the map
struct TileSpan {
    int m;
    sd_hog_score_map d;
    long long e0, e1;
};

__device__ __forceinline__ TileSpan tile_span(const DetArgs& a, int t)
{
    TileSpan s;
    s.m = sd_find_last_le(0, a.num_maps - 1, t, [&](int i) { return __ldg(a.tile0 + i); });   // the last map whose first tile is <= t
    s.d = a.maps[s.m];
    const long long n = (long long)a.Q * s.d.width * s.d.height;
    s.e0 = (long long)(t - __ldg(a.tile0 + s.m)) * kTile;
    s.e1 = min(s.e0 + kTile, n);
    return s;
}

__global__ void __launch_bounds__(kThreads) det_count_kernel(const __grid_constant__ DetArgs a)
{
    for (int t = blockIdx.x; t < a.total_tiles; t += gridDim.x) {
        const TileSpan s = tile_span(a, t);
        const float* p = a.scores + s.d.offset;
        unsigned c = 0;
        for (long long e = s.e0 + threadIdx.x; e < s.e1; e += kThreads) c += __ldg(p + e) > a.threshold;
        c = __reduce_add_sync(0xFFFFFFFFu, c);
        if ((threadIdx.x & 31) == 0 && c) atomicAdd(&a.state[s.d.frame].above, (unsigned long long)c);
    }
}

__global__ void det_init_kernel(const __grid_constant__ DetArgs a)
{
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= a.num_frames) return;
    FrameState& s = a.state[f];
    if (a.above) a.above[f] = (int64_t)s.above;
    s.active = s.above > (unsigned long long)a.max_c;
    s.need = (unsigned)a.max_c;
    s.prefix = 0;
    s.cut = 0;                       // every candidate key is > 0
    s.fill = 0;
}

// pass p: the histogram of digit p (bits 63 - 8p .. 56 - 8p) of the keys that match the frame's prefix
__global__ void __launch_bounds__(kThreads) det_hist_kernel(const __grid_constant__ DetArgs a, int p)
{
    __shared__ unsigned sh[256];
    const int shift = 56 - 8 * p;
    for (int t = blockIdx.x; t < a.total_tiles; t += gridDim.x) {
        const TileSpan s = tile_span(a, t);
        const FrameState& st = a.state[s.d.frame];
        if (!st.active) continue;                                 // uniform over the CTA
        const unsigned long long prefix = st.prefix;
        for (int i = threadIdx.x; i < 256; i += kThreads) sh[i] = 0;
        __syncthreads();
        const float* p_s = a.scores + s.d.offset;
        const unsigned r0 = __ldg(a.rank0 + s.m);
        for (long long e = s.e0 + threadIdx.x; e < s.e1; e += kThreads) {
            const float v = __ldg(p_s + e);
            if (!(v > a.threshold)) continue;
            const unsigned long long k = cand_key(v, r0 + (unsigned)e);
            if (p > 0 && (k >> (shift + 8)) != prefix) continue;
            atomicAdd(&sh[(k >> shift) & 255], 1u);
        }
        __syncthreads();
        unsigned* h = a.hist + (size_t)s.d.frame * 256;
        for (int i = threadIdx.x; i < 256; i += kThreads)
            if (sh[i]) atomicAdd(h + i, sh[i]);
        __syncthreads();
    }
}

// pass p: each selecting frame takes the digit that holds its need-th largest key
__global__ void det_pick_kernel(const __grid_constant__ DetArgs a, int p)
{
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= a.num_frames) return;
    FrameState& s = a.state[f];
    if (!s.active) return;
    unsigned* h = a.hist + (size_t)f * 256;
    unsigned cum = 0, need = s.need;
    int d = 255;
    for (; d > 0; --d) {
        if (cum + h[d] >= need) break;
        cum += h[d];
    }
    need -= cum;
    const unsigned long long prefix = (s.prefix << 8) | (unsigned)d;
    if (h[d] == need) {                                           // every key of the prefix is taken: the cut is found
        s.cut = prefix << (56 - 8 * p);
        s.active = 0;
    }
    s.need = need;
    s.prefix = prefix;
    for (int i = 0; i < 256; ++i) h[i] = 0;
}

__global__ void __launch_bounds__(kThreads) det_compact_kernel(const __grid_constant__ DetArgs a)
{
    const int lane = threadIdx.x & 31;
    for (int t = blockIdx.x; t < a.total_tiles; t += gridDim.x) {
        const TileSpan s = tile_span(a, t);
        FrameState& st = a.state[s.d.frame];
        const unsigned long long cut = st.cut;
        const float* p = a.scores + s.d.offset;
        const unsigned r0 = __ldg(a.rank0 + s.m);
        unsigned long long* keys = a.keys + (size_t)s.d.frame * a.max_c;
        for (long long eb = s.e0; eb < s.e1; eb += kThreads) {     // uniform trip count: the ballot sees every lane
            const long long e = eb + threadIdx.x;
            unsigned long long k = 0;
            if (e < s.e1) {
                const float v = __ldg(p + e);
                if (v > a.threshold) k = cand_key(v, r0 + (unsigned)e);
            }
            const bool take = k != 0 && k >= cut;
            const unsigned b = __ballot_sync(0xFFFFFFFFu, take);
            if (!b) continue;
            const int leader = __ffs(b) - 1;
            unsigned base = 0;
            if (lane == leader) base = atomicAdd(&st.fill, (unsigned)__popc(b));
            base = __shfl_sync(0xFFFFFFFFu, base, leader);
            if (take) keys[base + __popc(b & ((1u << lane) - 1))] = k;
        }
    }
}

struct Decoded {
    int m;
    long long e;
    int q, y, x;
};

// a frame's candidate from its key: the map (the last of the frame's maps whose first rank is <= the rank) and (q, y, x)
__device__ Decoded decode(const DetArgs& a, int f, unsigned long long k)
{
    const unsigned rank = 0xFFFFFFFFu - (unsigned)(k & 0xFFFFFFFFu);
    const int i = sd_find_last_le(a.fmap0[f], a.fmap0[f + 1] - 1, rank, [&](int j) { return a.rank0[a.fmaps[j]]; });
    Decoded r;
    r.m = a.fmaps[i];
    const sd_hog_score_map& d = a.maps[r.m];
    r.e = rank - a.rank0[r.m];
    const long long row = r.e / d.width;
    r.x = (int)(r.e - row * d.width);
    r.q = (int)(row / d.height);
    r.y = (int)(row - (long long)r.q * d.height);
    return r;
}

// {x0, y0, x1, y1} of a score position in int32 (sd_hog_detections checks that they fit)
__device__ int4 box_of(const DetArgs& a, const sd_hog_score_map& d, int x, int y)
{
    const sd_box64 b = sd_window_box(x, y, a.pad_x, a.pad_y, a.fw, a.fh, a.cell, d.frame_w, d.frame_h, d.level_w, d.level_h);
    return make_int4((int)b.x0, (int)b.y0, (int)b.x1, (int)b.y1);
}

__device__ __forceinline__ long long box_area(int4 b) { return (long long)(b.z - b.x) * (b.w - b.y); }

__global__ void __launch_bounds__(kNmsThreads, 1) det_nms_kernel(const __grid_constant__ DetArgs a, int key_slots)
{
    extern __shared__ __align__(16) unsigned char smem[];
    unsigned long long* s_key = reinterpret_cast<unsigned long long*>(smem);        // [key_slots], a power of two >= max_c, >= 2
    int4* s_box = reinterpret_cast<int4*>(s_key + key_slots);                       // [max_c]
    unsigned* s_rm = reinterpret_cast<unsigned*>(s_box + a.max_c);                  // [max_c / 32 rounded up]: removed
    const int f = blockIdx.x, tid = threadIdx.x, lane = tid & 31;
    const int n = (int)min(a.state[f].above, (unsigned long long)a.max_c);
    int P = 1;
    while (P < n) P <<= 1;
    const unsigned long long* g = a.keys + (size_t)f * a.max_c;
    for (int i = tid; i < P; i += kNmsThreads) s_key[i] = i < n ? g[i] : 0ull;   // 0: below every candidate key
    const int words = (n + 31) >> 5;
    for (int i = tid; i < words; i += kNmsThreads) s_rm[i] = 0;
    __syncthreads();

    // bitonic sort, descending
    for (int k = 2; k <= P; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = tid; i < P; i += kNmsThreads) {
                const int ixj = i ^ j;
                if (ixj > i) {
                    const unsigned long long u = s_key[i], v = s_key[ixj];
                    if ((i & k) == 0 ? u < v : u > v) {
                        s_key[i] = v;
                        s_key[ixj] = u;
                    }
                }
            }
            __syncthreads();
        }

    for (int i = tid; i < n; i += kNmsThreads) {
        const Decoded c = decode(a, f, s_key[i]);
        s_box[i] = box_of(a, a.maps[c.m], c.x, c.y);
    }
    __syncthreads();

    sd_hog_detection* out = a.out + (size_t)f * a.max_det;
    int kept = 0, i = -1;
    while (kept < a.max_det) {
        // the next candidate not removed, the same in every thread (broadcast reads of the bitmask)
        int w = (i + 1) >> 5;
        unsigned live = w < words ? ~s_rm[w] & (0xFFFFFFFFu << ((i + 1) & 31)) : 0u;
        while (!live && ++w < words) live = ~s_rm[w];
        if (!live) break;
        i = (w << 5) + __ffs(live) - 1;
        if (i >= n) break;
        const int4 bi = s_box[i];
        if (tid == 0) {
            const Decoded c = decode(a, f, s_key[i]);
            const sd_hog_score_map& d = a.maps[c.m];
            sd_hog_detection r;
            r.x = bi.x; r.y = bi.y; r.w = bi.z - bi.x; r.h = bi.w - bi.y;
            r.score = a.scores[d.offset + c.e];
            r.filter = c.q; r.level = d.level;
            r.cell_x = c.x; r.cell_y = c.y;
            out[kept] = r;
        }
        ++kept;
        const long long ai = box_area(bi);
        if (ai > 0) {                                             // a box with zero area suppresses nothing
            const int jend = words << 5;
            for (int j = ((i + 1) & ~31) + tid; j < jend; j += kNmsThreads) {   // a warp covers one bitmask word
                bool sup = false;
                if (j > i && j < n) {
                    const int4 bj = s_box[j];
                    const long long aj = box_area(bj);
                    const long long iw = (long long)min(bi.z, bj.z) - max(bi.x, bj.x);
                    const long long ih = (long long)min(bi.w, bj.w) - max(bi.y, bj.y);
                    if (aj > 0 && iw > 0 && ih > 0) {
                        const long long inter = iw * ih;
                        sup = (double)inter > a.overlap * (double)(ai + aj - inter);
                    }
                }
                const unsigned b = __ballot_sync(0xFFFFFFFFu, sup);
                if (lane == 0 && b) s_rm[j >> 5] |= b;
            }
        }
        __syncthreads();
    }
    if (tid == 0) a.count[f] = kept;
}

}  // namespace

bool sd_window_boxes_fit_int32(int width, int height, int pad_x, int pad_y, int fw, int fh, int cell, int frame_w, int frame_h,
                               int level_w, int level_h)
{
    if (width <= 0 || height <= 0) return true;
    // the extreme numerators, those of positions 0 and width - 1 (height - 1), exactly
    const __int128 limit = (__int128)1 << 62;
    const __int128 sx = (__int128)cell * frame_w, sy = (__int128)cell * frame_h;
    const __int128 nx[2] = {(__int128)(-pad_x) * sx, (__int128)(width - 1 - pad_x + fw) * sx};
    const __int128 ny[2] = {(__int128)(-pad_y) * sy, (__int128)(height - 1 - pad_y + fh) * sy};
    for (int k = 0; k < 2; ++k) {
        if (!(nx[k] < limit && nx[k] > -limit && ny[k] < limit && ny[k] > -limit)) return false;
        const long long bx = sd_round_half_up((long long)nx[k], level_w), by = sd_round_half_up((long long)ny[k], level_h);
        if (bx < INT_MIN || bx > INT_MAX || by < INT_MIN || by > INT_MAX) return false;
    }
    return true;
}

extern "C" {

int sd_hog_detections(sd_ctx* ctx, const float* d_scores, const sd_hog_score_map* d_maps, int num_maps, int num_frames,
                      int num_filters, int cell_size, int filter_w, int filter_h, int pad_x, int pad_y, float threshold,
                      double overlap, int max_candidates, int max_detections, sd_hog_detection* d_out, int32_t* d_count,
                      int64_t* d_above)
{
    if (!ctx) return SD_ERR_INVALID;
    SD_REQUIRE(ctx, d_out && d_count && (num_maps == 0 || (d_scores && d_maps)), "null argument");
    SD_REQUIRE(ctx, sd_aligned(d_scores, 4) && sd_aligned(d_maps, 8) && sd_aligned(d_out, 4) && sd_aligned(d_count, 4) &&
                        sd_aligned(d_above, 8),
               "scores, output and counts must be 4-byte aligned, the map table and d_above 8-byte aligned");
    SD_REQUIRE(ctx, num_frames >= 1, "num_frames must be >= 1");
    SD_REQUIRE(ctx, num_maps >= 0, "negative map count");
    SD_REQUIRE(ctx, num_filters >= 1 && num_filters <= SD_HOG_FILTER_MAX_BANK, "num_filters must be in [1, SD_HOG_FILTER_MAX_BANK]");
    SD_REQUIRE(ctx, cell_size >= 1 && cell_size <= kDenseMaxCell, "cell_size must be in [1,32]");
    if (const int rc = sd_hog_check_filter(ctx, __func__, filter_w, filter_h, pad_x, pad_y)) return rc;
    SD_REQUIRE(ctx, !std::isnan(threshold), "threshold is NaN");
    SD_REQUIRE(ctx, overlap >= 0.0 && overlap <= 1.0, "overlap must be in [0, 1]");
    SD_REQUIRE(ctx, max_candidates >= 1 && max_candidates <= SD_HOG_DETECT_MAX_CANDIDATES,
               "max_candidates must be in [1, SD_HOG_DETECT_MAX_CANDIDATES]");
    SD_REQUIRE(ctx, max_detections >= 1 && max_detections <= max_candidates, "max_detections must be in [1, max_candidates]");

    std::vector<sd_hog_score_map> table;
    if (num_maps > 0)
        if (const int rc = sd_fetch_table(ctx, d_maps, num_maps, table)) return rc;
    return sd_hog_detections_table(ctx, d_scores, d_maps, table.data(), num_maps, num_frames, num_filters, cell_size, filter_w, filter_h,
                                   pad_x, pad_y, threshold, overlap, max_candidates, max_detections, d_out, d_count, d_above);
}

}  // extern "C"

#define DET_REQUIRE(cond, msg)                                                         \
    do {                                                                               \
        if (!(cond)) return sd_fail(ctx, SD_ERR_INVALID, "%s: %s", fn, msg);           \
    } while (0)
int sd_hog_detections_table(sd_ctx* ctx, const float* d_scores, const sd_hog_score_map* d_maps, const sd_hog_score_map* table,
                            int num_maps, int num_frames, int num_filters, int cell_size, int filter_w, int filter_h, int pad_x,
                            int pad_y, float threshold, double overlap, int max_candidates, int max_detections,
                            sd_hog_detection* d_out, int32_t* d_count, int64_t* d_above)
{
    const char* fn = "sd_hog_detections";
    // per map: its first tile and first frame-local rank; the maps grouped by frame
    std::vector<int> ints(3 * (size_t)num_maps + num_frames + 1);
    int* tile0 = ints.data();
    unsigned* rank0 = reinterpret_cast<unsigned*>(tile0 + num_maps);
    int* fmaps = tile0 + 2 * num_maps;
    int* fmap0 = fmaps + num_maps;
    std::vector<long long> frame_scores(num_frames, 0);
    long long tiles = 0;
    for (int i = 0; i < num_maps; ++i) {
        const sd_hog_score_map& m = table[i];
        DET_REQUIRE(m.frame >= 0 && m.frame < num_frames, "a map's frame is out of range");
        DET_REQUIRE(m.offset >= 0, "a map's offset is negative");
        DET_REQUIRE(m.frame_w >= 1 && m.frame_h >= 1 && m.level_w >= 1 && m.level_h >= 1, "a map's frame or level is smaller than 1 x 1");
        DET_REQUIRE(m.width >= 0 && m.height >= 0, "a map's size is negative");
        const long long n = (long long)num_filters * m.width * m.height;
        tile0[i] = (int)tiles;
        tiles += (n + kTile - 1) / kTile;
        DET_REQUIRE(tiles <= INT_MAX, "too many score tiles");
        rank0[i] = (unsigned)frame_scores[m.frame];
        frame_scores[m.frame] += n;
        DET_REQUIRE(frame_scores[m.frame] <= (long long)UINT_MAX, "more than 2^32 - 1 scores in one frame");
        DET_REQUIRE(sd_window_boxes_fit_int32(m.width, m.height, pad_x, pad_y, filter_w, filter_h, cell_size, m.frame_w, m.frame_h,
                                              m.level_w, m.level_h),
                    "a map's boxes do not fit in int32");
    }
    {
        std::vector<int> per(num_frames + 1, 0);
        for (int i = 0; i < num_maps; ++i) per[table[i].frame + 1]++;
        for (int f = 0; f < num_frames; ++f) per[f + 1] += per[f];
        std::copy(per.begin(), per.end(), fmap0);
        for (int i = 0; i < num_maps; ++i) fmaps[per[table[i].frame]++] = i;      // stable: table order within a frame
    }
    const bool select = std::any_of(frame_scores.begin(), frame_scores.end(), [&](long long n) { return n > max_candidates; });

    // scratch: keys | frame states | histograms | ints
    const size_t key_bytes = sizeof(unsigned long long) * num_frames * (size_t)max_candidates;
    const size_t state_bytes = sd_round16(sizeof(FrameState) * num_frames);
    const size_t hist_bytes = sizeof(unsigned) * 256 * (size_t)num_frames;
    const size_t int_bytes = sizeof(int) * ints.size();
    unsigned char* ws = static_cast<unsigned char*>(sd_workspace(ctx, SD_WS_DETECT, key_bytes + state_bytes + hist_bytes + int_bytes));
    if (!ws) return SD_ERR_CUDA;

    DetArgs a;
    memset(&a, 0, sizeof(a));
    a.scores = d_scores;
    a.maps = d_maps;
    a.num_maps = num_maps;
    a.num_frames = num_frames;
    a.keys = reinterpret_cast<unsigned long long*>(ws);
    a.state = reinterpret_cast<FrameState*>(ws + key_bytes);
    a.hist = reinterpret_cast<unsigned*>(ws + key_bytes + state_bytes);
    int* d_ints = reinterpret_cast<int*>(ws + key_bytes + state_bytes + hist_bytes);
    a.tile0 = d_ints;
    a.rank0 = reinterpret_cast<const unsigned*>(d_ints + num_maps);
    a.fmaps = d_ints + 2 * num_maps;
    a.fmap0 = d_ints + 3 * num_maps;
    a.total_tiles = (int)tiles;
    a.Q = num_filters; a.cell = cell_size; a.fw = filter_w; a.fh = filter_h; a.pad_x = pad_x; a.pad_y = pad_y;
    a.threshold = threshold;
    a.overlap = overlap;
    a.max_c = max_candidates;
    a.max_det = max_detections;
    a.out = d_out;
    a.count = d_count;
    a.above = d_above;

    SD_CUDA(ctx, cudaMemsetAsync(a.state, 0, state_bytes + hist_bytes, ctx->stream));
    SD_CUDA(ctx, cudaMemcpyAsync(d_ints, ints.data(), int_bytes, cudaMemcpyHostToDevice, ctx->stream));
    const int grid = (int)std::max(1LL, std::min<long long>(tiles, 8LL * ctx->sm_count));
    const int fgrid = sd_div_up(num_frames, 128);
    if (tiles > 0) {
        det_count_kernel<<<grid, kThreads, 0, ctx->stream>>>(a);
        SD_LAUNCH_CHECK(ctx, "det_count_kernel");
    }
    det_init_kernel<<<fgrid, 128, 0, ctx->stream>>>(a);
    SD_LAUNCH_CHECK(ctx, "det_init_kernel");
    if (select)
        for (int p = 0; p < 8; ++p) {
            det_hist_kernel<<<grid, kThreads, 0, ctx->stream>>>(a, p);
            SD_LAUNCH_CHECK(ctx, "det_hist_kernel");
            det_pick_kernel<<<fgrid, 128, 0, ctx->stream>>>(a, p);
            SD_LAUNCH_CHECK(ctx, "det_pick_kernel");
        }
    if (tiles > 0) {
        det_compact_kernel<<<grid, kThreads, 0, ctx->stream>>>(a);
        SD_LAUNCH_CHECK(ctx, "det_compact_kernel");
    }
    int key_slots = 2;                               // an even count keeps the boxes after the keys 16-byte aligned
    while (key_slots < max_candidates) key_slots <<= 1;
    const int smem = key_slots * (int)sizeof(unsigned long long) + max_candidates * (int)sizeof(int4) + (max_candidates + 31) / 32 * 4;
    SD_CUDA(ctx, cudaFuncSetAttribute(det_nms_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    det_nms_kernel<<<num_frames, kNmsThreads, smem, ctx->stream>>>(a, key_slots);
    SD_LAUNCH_CHECK(ctx, "det_nms_kernel");
    return SD_OK;
}
#undef DET_REQUIRE
