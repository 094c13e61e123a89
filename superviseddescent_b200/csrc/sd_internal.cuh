// Internal definitions shared by the .cu translation units of libsd_b200.so.
// Nothing here is part of the C ABI (include/sd_b200.h).
#pragma once

#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <string>
#include <vector>

#include "sd_b200.h"

#define SD_MAX_EYES 4
#define SD_MAX_BINS 16   // undirected orientations K supported by the HOG kernel
constexpr int kDenseMaxCell = 32;   // largest dense cell size: one cell with its halo stays below 227 KB of shared memory at K = 16

enum { SD_WS_GRAM_EXT = 0, SD_WS_FEATURES, SD_WS_SCRATCH, SD_WS_TC_TILES,
       SD_WS_PARTIAL, SD_WS_GEOM, SD_WS_GEMM_PARTIAL, SD_WS_DIAGINV2, SD_WS_PANEL, SD_WS_BIAS, SD_WS_CG, SD_WS_CGMAT,
       SD_WS_UPLOAD /* B,G,R scratch of sd_upload_frames */,
       SD_WS_RANK /* the rank diagnostic's working copy of the D x D system, its panel and state (sd_rank.cu) */,
       SD_WS_LEVEL /* column shift and shifted-row weights of sd_train_level (sd_train.cu) */,
       SD_WS_GATHER /* frame, union, region, record and index tables of the levels on host frames (sd_train.cu) */,
       SD_WS_PYRAMID /* resized levels and level tables of one slice of sd_hog_pyramid (sd_hog_dense.cu) */,
       SD_WS_FILTERS /* first CTA of every grid of sd_hog_correlate (sd_hog_filters.cu) */,
       SD_WS_DETECT /* candidate keys, frame states, histograms and map tables of sd_hog_detections (sd_hog_detect.cu) */,
       SD_WS_SVM /* compacted active rows, margins, column shift and index of sd_learn_squared_hinge (sd_hog_train.cu) */,
       SD_WS_TRAIN_ROWS /* positive rows, negative cache and labels of sd_hog_train_filter (sd_hog_train.cu) */,
       SD_WS_TRAIN_SLICE /* one slice's pyramid, scores, tables and detections of sd_hog_train_filter (sd_hog_train.cu) */,
       SD_WS_COUNT };

// Block-row ownership of the distributed factorisation: the matrix is cut into panels of SD_PANEL_ROWS rows (two 128-row
// Cholesky blocks), and panel p belongs to rank p % nranks.  The Gram exchange delivers each panel's rows to their owner, and
// every step of the solve that splits work over the ranks splits it the same way.
constexpr int SD_PANEL_ROWS = 256;
__host__ __device__ inline int sd_panel_owner(int64_t row, int nranks) { return (int)(row / SD_PANEL_ROWS) % nranks; }

// The rows of a C sub-matrix that this rank owns; first_row = global row of the sub-matrix's first row.
struct sd_row_filter {
    int nranks, rank;
    int64_t first_row;
};

struct sd_comm;   // sd_comm.cu

struct sd_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    cudaStream_t copy_stream = nullptr;   // host->device copies of host frames (sd_detect_faces_host, sd_upload_frames)
    cudaStream_t chain_stream = nullptr;  // Cholesky look-ahead: next panel's diagonal blocks while the trailing update runs
    cudaEvent_t chain_ev[2] = {nullptr, nullptr};
    int syrk_sm_reserve = 0;              // SMs the persistent SYRK leaves free (1 while a look-ahead chain runs beside it)
    std::string err;
    std::vector<int2> tile_scratch;       // host side of the tensor-core tile lists
    int64_t launches = 0;
    int sm_count = 132;
    int gram_mode = 0;
    int solver_mode = 0;           // systems with D > 256: 0 = blocked Cholesky, 1 = conjugate gradients (Cholesky if they stall)
    int cg_iterations = 0;         // of the last solve: +n CG converged, -n CG gave up after n (factorisation answered), 0 not tried
    bool rank_diagnostic = false;  // sd_set_rank_diagnostic: every solve also computes the rank of its regularised system
    int last_rank = -1;            // of the last solve: the rank, or -1 when it was not computed
    cudaEvent_t cg_ev[8] = {};     // convergence read-backs of the CG loop (the host runs a few iterations ahead of them)
    int64_t roi_fallbacks = 0;     // faces repeated from the full frame because a patch left its ROI
    int64_t gathered_bytes = 0;    // host-frame bytes sd_train_level / sd_apply_level read over PCIe
    float timings[4] = {0, 0, 0, 0};
    cudaEvent_t ev[6] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    void* ws[SD_WS_COUNT] = {};
    size_t ws_bytes[SD_WS_COUNT] = {};
    // pinned scratch for small device->host results (lambda, residual, status flags)
    void* h_scratch = nullptr;
    void* d_scratch = nullptr;   // 4 KB
    // staging pair of sd_detect_faces_host and of the levels on host frames (sd_ensure_stage)
    void* d_stage[2] = {nullptr, nullptr};
    size_t stage_bytes[2] = {0, 0};
    cudaEvent_t stage_ev[2] = {nullptr, nullptr};
    cudaEvent_t stage_done[2] = {nullptr, nullptr};
    // the levels on a host projection (sd_train.cu): pinned staging pair the callback fills, one event per half (its upload is
    // done), the chunk buffer's last reader on the stream, and the pinned copy of the level's parameter rows
    void* host_stage[2] = {nullptr, nullptr};
    size_t host_stage_bytes[2] = {0, 0};
    cudaEvent_t host_stage_ev[2] = {nullptr, nullptr};
    cudaEvent_t host_chunk_free = nullptr;
    void* host_x = nullptr;
    size_t host_x_bytes = 0;
};

int sd_fail(sd_ctx* ctx, int code, const char* fmt, ...);
int sd_check_cuda(sd_ctx* ctx, cudaError_t e, const char* what);
// grow-only workspace; returns nullptr (and sets the error) on failure
void* sd_workspace(sd_ctx* ctx, int slot, size_t bytes);

#define SD_CUDA(ctx, call)                                                        \
    do {                                                                          \
        cudaError_t _e = (call);                                                  \
        if (_e != cudaSuccess) return sd_check_cuda((ctx), _e, #call);            \
    } while (0)

#define SD_LAUNCH_CHECK(ctx, name)                                                \
    do {                                                                          \
        (ctx)->launches++;                                                        \
        cudaError_t _e = cudaGetLastError();                                      \
        if (_e != cudaSuccess) return sd_check_cuda((ctx), _e, name);             \
    } while (0)

#define SD_REQUIRE(ctx, cond, msg)                                                \
    do {                                                                          \
        if (!(cond)) return sd_fail((ctx), SD_ERR_INVALID, "%s: %s", __func__, msg); \
    } while (0)

static inline int sd_div_up(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }

// ---- HOG configurations ------------------------------------------------------------------------

// dd, the features per cell of vl_hog_new(variant, num_bins): 3K + 4 for UoCTTI (variant 1), 4K for Dalal-Triggs (variant 0)
inline int sd_hog_dd(int num_bins, int variant) { return variant == 1 ? 3 * num_bins + 4 : 4 * num_bins; }

// The configuration rule of the HOG entry points: variant 0 or 1 and num_bins in [1, SD_MAX_BINS], and for the dense ones, which
// take a cell size, cell_size in [1, kDenseMaxCell].  Returns SD_OK, or SD_ERR_INVALID with the message "fn: ..." in ctx (none
// for ctx == nullptr: the host-only functions report a status only).
inline int sd_hog_check_config(sd_ctx* ctx, const char* fn, int variant, int num_bins)
{
    if (variant != 0 && variant != 1) return sd_fail(ctx, SD_ERR_INVALID, "%s: unknown HOG variant", fn);
    if (num_bins < 1 || num_bins > SD_MAX_BINS) return sd_fail(ctx, SD_ERR_INVALID, "%s: num_bins must be in [1,16]", fn);
    return SD_OK;
}
inline int sd_hog_check_config(sd_ctx* ctx, const char* fn, int variant, int num_bins, int cell_size)
{
    if (const int rc = sd_hog_check_config(ctx, fn, variant, num_bins)) return rc;
    if (cell_size < 1 || cell_size > kDenseMaxCell) return sd_fail(ctx, SD_ERR_INVALID, "%s: cell_size must be in [1,32]", fn);
    return SD_OK;
}

// a device descriptor table of count entries, read back to the host once
template <class T>
int sd_fetch_table(sd_ctx* ctx, const T* d_table, int count, std::vector<T>& table)
{
    table.resize(count);
    SD_CUDA(ctx, cudaMemcpyAsync(table.data(), d_table, sizeof(T) * count, cudaMemcpyDeviceToHost, ctx->stream));
    SD_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return SD_OK;
}

// ---- internal entry points shared between translation units ---------------------------------

// Tensor-core SYRK (sd_gram_tc.cu): C[i,j] = beta*C[i,j] + alpha * sum_{k<K} S[k,i] * S[k,j] for i < MI, j < NJ, on the
// tiles that intersect j >= i.  S: K x NJ row-major (lds), C: MI x NJ (ldc).  passes: 3 = 3xTF32 split, 1 = one TF32 pass;
// unbiased: round the hi part of the split.  rows (optional): only the tiles of rows this rank owns.
int sd_syrk_tc(sd_ctx* ctx, const float* d_S, int64_t lds, int K, int MI, int NJ, float* d_C, int64_t ldc, float alpha, float beta,
               int passes, bool unbiased, const sd_row_filter* rows);
// whether the tensor-core kernel can read S (TMA alignment)
bool sd_syrk_tc_supported(const float* d_S, int64_t lds, int K);
// the driver's cuTensorMapEncodeTiled, looked up once (sd_gram_tc.cu); nullptr when the driver does not provide it
typedef CUresult (*sd_encode_tiled_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                       const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                       CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
sd_encode_tiled_fn sd_encode_tiled();
// the SYRK dispatcher (sd_linalg.cu): the one place that reads the gram mode and picks the tensor-core or the SIMT kernel.
// big: the size rule's verdict (syrk_is_big) for the product the call belongs to.
int syrk_upper(sd_ctx* ctx, const float* d_S, int64_t lds, int K, int MI, int NJ, float* d_C, int64_t ldc, float alpha, float beta,
               bool big, bool unbiased, const sd_row_filter* rows = nullptr);
bool syrk_is_big(int K, int64_t MI, int64_t NJ);

int sd_check_hog_status(sd_ctx* ctx, const char* what);   // sd_api.cu: synchronises, reports and clears the projection's flags
// the grids of an sd_hog_grids call, validated; per-grid descriptors are read back once into *table (if given) (sd_hog_render.cu)
int sd_read_hog_grids(sd_ctx* ctx, const char* fn, const sd_hog_grids* grids, int* max_w, int* max_h, std::vector<sd_hog_grid>* table);

// The learn path of sd_learn_centred in two steps (sd_linalg.cu), so that a training level can add its rows chunk by chunk
// (sd_train.cu).  The Gram lives in the context's workspace (D x sd_learn_ldg floats).
inline int64_t sd_learn_ldg(int D, int M) { return ((int64_t)(D + M) + 3) / 4 * 4; }
// [A^T A | A^T B] of N rows: started (accumulate == false; records the start of "At * A") or added onto (accumulate == true)
int sd_learn_gram(sd_ctx* ctx, const float* d_A, int64_t lda, const float* d_B, int64_t ldb, int N, bool shard, int D, int M,
                  bool accumulate);
// exchange over the ranks and solve with the column shift d_mu, as sd_learn_centred does after its Gram
int sd_learn_centred_solve(sd_ctx* ctx, sd_comm* comm, int D, int M, const sd_regulariser* reg, int n_train_global, int route,
                           const float* d_mu, float* d_X, float* d_Xc, float* lambda_out);
// d_A[:, c] -= d_mu[c] for c < D - 1 on N rows (the centring pass of sd_centre_features)
int sd_shift_rows(sd_ctx* ctx, float* d_A, int64_t lda, int N, int D, const float* d_mu);
constexpr int SD_LU_MAX_DIM = 256;   // systems up to this D keep the reference-order LU on uncentred rows

// numerical rank of the symmetric matrix whose upper triangle is in d_G (blocked pivoted Cholesky on a copy, sd_rank.cu)
int sd_gram_rank(sd_ctx* ctx, const float* d_G, int64_t ldg, int D, int* rank_out, float* first_pivot, float* last_pivot);

// prepared launches of the tensor-core TN-GEMM (sd_gram_tc.cu): plan_storage = SD_TC_PLAN_BYTES bytes, 64-byte aligned
#define SD_TC_PLAN_BYTES 640
int sd_gemm_tn_tc_prepare(sd_ctx* ctx, const float* d_SA, int64_t lda, const float* d_SB, int64_t ldb, int K, int MI, int NJ,
                          float* d_C, int64_t ldc, float alpha, float beta, int passes, bool unbiased, bool upper_only,
                          const sd_row_filter* rows, void* d_tiles_buf, void* plan_storage, bool* empty,
                          bool narrow = false /* a single tile column of <= 192 columns may use the narrow-N kernel variants */,
                          int a_strip_rows = 0 /* > 0: operand A strip-major, see sd_gram_tc.cu */);
int sd_gemm_tn_tc_launch(sd_ctx* ctx, const void* plan_storage);

// multi-GPU helpers (sd_comm.cu); a null communicator is a single rank
int sd_comm_rank_of(const sd_comm* c);
int sd_comm_size_of(const sd_comm* c);
int sd_comm_bcast(sd_ctx* ctx, sd_comm* c, float* d_buf, size_t count, int root, cudaStream_t stream);
int sd_comm_group_start(sd_ctx* ctx);
int sd_comm_group_end(sd_ctx* ctx);
int sd_comm_allreduce_f64(sd_ctx* ctx, sd_comm* c, double* d_buf, size_t count, cudaStream_t stream);
int sd_comm_allreduce_f32(sd_ctx* ctx, sd_comm* c, float* d_buf, size_t count, cudaStream_t stream);
// conjugate gradients on the tensor cores (sd_cg.cu); SD_ERR_NUMERIC = did not converge, use the factorisation
int sd_cg_solve(sd_ctx* ctx, sd_comm* comm, float* G, int64_t ldg, int n, int col0, int M, float** W_out, int* ldw_out, int* iters);
// rows [k0, k1) of the n x n system whose part of the product S P rank `me` computes in the shared CG route (multiples of 16 rows)
inline void sd_cg_slab(int n, int nranks, int me, int* k0, int* k1)
{
    *k0 = 0; *k1 = n;
    if (nranks > 1) {
        const int per = ((n + nranks - 1) / nranks + 15) / 16 * 16;
        *k0 = me * per < n ? me * per : n;
        *k1 = (me + 1) * per < n ? (me + 1) * per : n;
    }
}
// true when sd_reduce_scatter_gram leaves the rows block-row-cyclic (large, 16-byte aligned systems); smaller ones are all-reduced
bool sd_gram_is_scattered(int D, int64_t ldg, const float* d_G);

// device-side normalisation factors, shared by the HOG and cascade kernels
struct sd_eyes_dev {
    int kind;
    int n_right, n_left;
    int right_idx[SD_MAX_EYES];
    int left_idx[SD_MAX_EYES];
};
int sd_eyes_to_dev(sd_ctx* ctx, const sd_normalisation* n, int num_landmarks, sd_eyes_dev* out);

// ---- host frames read in place (sd_model.cu) ---------------------------------------------------------------------------------
// One region of a pinned host frame for roi_gather_kernel: the SMs pull its rows zero-copy into a packed grey device buffer
// (16-byte vectors; colour pixels converted on the way).  The region's x is a multiple of 16 pixels and its rows lie inside the
// frame's row_stride.
struct GatherRec {
    const uint8_t* src;          // device-mapped address of the region's first pixel in the caller's frame
    int64_t src_stride;          // bytes between the frame's rows
    int64_t dst_offset;          // of the grey region in the staging buffer; its rows are 16 * vec_per_row bytes apart
    int32_t vec_per_row, rows;   // region size in steps of 16 pixels x rows
};
// the one gather: n_grey records of grey frames, then n_colour records of B,G,R frames, into dst, on `stream`
int sd_roi_gather(sd_ctx* ctx, const GatherRec* d_grey, int n_grey, const GatherRec* d_colour, int n_colour, uint8_t* dst,
                  cudaStream_t stream);
// Device-mapped address of a pinned host frame, or nullptr.  Frames inside the last pinned allocation seen are mapped by
// offset instead of one driver query each.
struct PinnedRange {
    uintptr_t lo = 0, hi = 0;    // host addresses of the allocation
    intptr_t delta = 0;          // device address - host address
};
const uint8_t* sd_mapped_frame(const uint8_t* p, size_t bytes, PinnedRange& last);
// what every entry point that reads sd_host_frame requires of frame f; fn names the entry point in the message
int sd_check_host_frame(sd_ctx* ctx, const char* fn, const sd_host_frame& fr, int f);
// grey bytes per staging half by default: detect's ROI chunks and the levels' gather batches
constexpr size_t SD_STAGE_HALF_BYTES = size_t(48) << 20;
// the context's staging pair (d_stage) holds at least `bytes` each (grow-only; a buffer that grows is freed after both streams drain)
int sd_ensure_stage(sd_ctx* ctx, size_t bytes);
inline size_t sd_host_frame_bytes(const sd_host_frame& f) { return (size_t)(f.height - 1) * f.row_stride + (size_t)f.width * f.channels; }
inline size_t sd_round16(size_t v) { return (v + 15) & ~(size_t)15; }
// grey bytes of a frame at a 16-byte pitch: no region of it is larger
inline size_t sd_gray_bytes(const sd_host_frame& f) { return (size_t)f.height * sd_round16(f.width); }

#ifdef __CUDACC__
// Inter-eye distance exactly as helpers.hpp:136-160 evaluates it: eye centres are float sums
// scaled by the float reciprocal of the count (cv::Vec /= float), the difference is taken in float,
// squares are accumulated in double (cv::norm NORM_L2) and the root is a double sqrt.
__device__ __forceinline__ double sd_device_ied(const float* __restrict__ row, int L, const sd_eyes_dev& e)
{
    float rx = 0.f, ry = 0.f, lx = 0.f, ly = 0.f;
    for (int i = 0; i < e.n_right; ++i) {
        rx = __fadd_rn(rx, row[e.right_idx[i]]);
        ry = __fadd_rn(ry, row[e.right_idx[i] + L]);
    }
    const float ir = __fdiv_rn(1.0f, (float)e.n_right);
    rx = __fmul_rn(rx, ir);
    ry = __fmul_rn(ry, ir);
    for (int i = 0; i < e.n_left; ++i) {
        lx = __fadd_rn(lx, row[e.left_idx[i]]);
        ly = __fadd_rn(ly, row[e.left_idx[i] + L]);
    }
    const float il = __fdiv_rn(1.0f, (float)e.n_left);
    lx = __fmul_rn(lx, il);
    ly = __fmul_rn(ly, il);
    const double dx = (double)__fsub_rn(rx, lx);
    const double dy = (double)__fsub_rn(ry, ly);
    return sqrt(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)));
}

// Half patch size of one sample (adaptive_vlhog.hpp:123): std::round(float rel * double IED / 2), or fixed_half > 0 for the
// non-adaptive HogTransform (examples/landmark_detection.cpp:213).  A half below 1 (cv::resize would throw on the empty ROI)
// becomes 1 and sets *degenerate.  hog_geometry_kernel (sd_hog.cu) and roi_plan_kernel (sd_train.cu) both call it, so the
// window a training gather plans is the window the HOG kernel reads.
__device__ __forceinline__ int sd_patch_half(const float* __restrict__ row, int L, const sd_eyes_dev& eyes, float rel, int fixed_half,
                                             bool* degenerate)
{
    *degenerate = false;
    if (fixed_half > 0) return fixed_half;
    const double ied = sd_device_ied(row, L, eyes);
    int half = (int)round(__dmul_rn(__dmul_rn((double)rel, ied), 0.5));
    if (half < 1) {
        half = 1;
        *degenerate = true;
    }
    return half;
}

// cv::cvtColor(BGR2GRAY) of one 8-bit pixel, OpenCV >= 3 fixed point (15-bit coefficients, SURVEY.md 8c).  The only spelling of
// the conversion: bgr2gray_kernel (sd_hog.cu) and the colour ROI gather (sd_model.cu) both call it.
__device__ __forceinline__ uint32_t sd_bgr_to_gray(uint32_t b, uint32_t g, uint32_t r)
{
    return (3735u * b + 19235u * g + 9798u * r + (1u << 14)) >> 15;
}
#endif
