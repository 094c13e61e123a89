// Cascade levels of the HOG optimiser in chunks of rows (include/sd_b200.h, "training and testing in chunks").
//
//   sd_level_chunk_rows  rows of one chunk that fit beside what the level's solve allocates
//   sd_train_level       superviseddescent.hpp:173-217: HOG, targets, shift, Gram accumulation, exchange, solve, update
//   sd_apply_level       superviseddescent.hpp:262-306, 323-344: HOG, templates, update
//
// [A^T A | A^T b] is a sum over rows, so a level never needs all of its feature rows at once.  The rows are shifted by the column
// means of the first chunk (the pilot p, over all ranks) before they enter the Gram: with n0 rows in that chunk p is within about
// sigma / sqrt(n0) of the true mean, so the shifted Gram keeps the digits that centring saves (DESIGN 4.3), and the solve
// (solve_gram_impl) is exact for any shift -- it rebuilds the norm of the unshifted matrix from the shift, eliminates the bias
// column first (the exact centring of any shifted Gram) and shifts the bias back.  With one chunk p IS the mean and the call
// sequence is sd_train's one-shot sequence, kernel for kernel.
#include "sd_internal.cuh"

#include <climits>

namespace {

constexpr int kMinChunkRows = 256;                       // below this a chunk is all launch overhead
constexpr size_t kReserveBytes = size_t(512) << 20;      // small workspaces, tile lists, allocator granularity

// The batch as seen from sample r0 on: sample i of the view reads the frame sample r0 + i reads in the whole batch.
sd_image_batch batch_from(const sd_image_batch& b, int r0)
{
    sd_image_batch v = b;
    if (r0 == 0) return v;
    v.count = b.count - r0;
    if (b.d_frames) v.d_frames = b.d_frames + r0;
    if (b.d_roi) v.d_roi = b.d_roi + r0;
    if (b.d_roi_miss) v.d_roi_miss = b.d_roi_miss + r0;
    if (!b.d_frames && !b.d_roi) v.d_data = b.d_data + (int64_t)r0 * b.image_stride;
    return v;
}

// HOG rows of samples [r0, r0 + rows) into the chunk buffer
int hog_rows(sd_ctx* ctx, const sd_image_batch* images, const int32_t* d_image_index, const float* d_x, int r0, int rows, int L,
             const sd_normalisation* eyes, const sd_hog_param* p, float* d_chunk, int64_t ld)
{
    const int P = 2 * L;
    const sd_image_batch view = d_image_index ? *images : batch_from(*images, r0);
    return sd_hog_batch(ctx, &view, d_image_index ? d_image_index + r0 : nullptr, d_x + (int64_t)r0 * P, P, rows, L, eyes, p,
                        d_chunk, ld);
}

size_t round_up(size_t v, size_t m) { return (v + m - 1) / m * m; }

}  // namespace

extern "C" {

int sd_level_chunk_rows(sd_ctx* ctx, sd_comm* comm, int64_t N_local, int D, int M, int route, size_t free_bytes, int* rows_out)
{
    if (!ctx) return SD_ERR_INVALID;
    SD_REQUIRE(ctx, rows_out && N_local >= 0 && D >= 1 && M >= 1, "bad argument");
    if (free_bytes == 0) {
        size_t total = 0;
        SD_CUDA(ctx, cudaSetDevice(ctx->device));
        SD_CUDA(ctx, cudaMemGetInfo(&free_bytes, &total));
    }
    const int64_t ld = sd_learn_ldg(D, M);
    const int nranks = sd_comm_size_of(comm);
    // what the level's solve will still allocate with the context's settings, less what the context already holds
    size_t need = 0;
    auto add = [&](int slot, size_t bytes) { if (bytes > ctx->ws_bytes[slot]) need += bytes - ctx->ws_bytes[slot]; };
    const size_t gram = (size_t)D * ld * sizeof(float);
    add(SD_WS_SCRATCH, gram);
    add(SD_WS_LEVEL, (size_t)D * (M + 1) * sizeof(float));
    if (nranks > 1) add(SD_WS_GRAM_EXT, gram);                                          // band buffer of the exchange (at most G)
    if (ctx->rank_diagnostic && !(nranks > 1 && route == 1))                            // the rank's copy of the system
        add(SD_WS_RANK, (size_t)(D + 130) * round_up(D, 4) * sizeof(float) + 4096);
    if (D > SD_LU_MAX_DIM) {
        const size_t n = (size_t)D - 1;
        add(SD_WS_BIAS, (size_t)(D + M) * sizeof(double) + n * (M + 1) * sizeof(float));
        add(SD_WS_DIAGINV2, round_up(n, 128) / 128 * 2 * 128 * 128 * sizeof(float));    // the Cholesky's inverse diagonal blocks
        if (ctx->solver_mode == 1 || (nranks > 1 && route == 2))                        // CG's strip-major copy of the system
            add(SD_WS_CGMAT, round_up(n, 128) * round_up(n, 16) * sizeof(float));
    }
    // per row: the caller's chunk row and the update's partial sums (sd_cascade_update)
    const size_t per_row = (size_t)ld * sizeof(float) + (size_t)M * sizeof(double);
    const size_t fixed = need + kReserveBytes;
    const int64_t fit = free_bytes > fixed ? (int64_t)((free_bytes - fixed) / per_row) : 0;
    const int64_t least = N_local < kMinChunkRows ? N_local : kMinChunkRows;
    if (fit < least)
        return sd_fail(ctx, SD_ERR_CUDA, "sd_level_chunk_rows: D = %d: the solve needs %.2f GB and %lld rows of %.1f KB do not fit beside it "
                       "in %.2f GB", D, need / 1e9, (long long)least, per_row / 1e3, free_bytes / 1e9);
    int64_t rows = fit < N_local ? fit : N_local;
    if (rows > INT_MAX) rows = INT_MAX;
    *rows_out = rows < 1 ? 1 : (int)rows;
    return SD_OK;
}

int sd_train_level(sd_ctx* ctx, sd_comm* comm, const sd_image_batch* images, const int32_t* d_image_index, const float* d_x,
                   const float* d_x_gt, int N_local, int L, int64_t n_global, const sd_normalisation* hog_eyes, const sd_hog_param* p,
                   const sd_normalisation* norm, const float* d_templates, int64_t ldt, const sd_regulariser* reg, int route,
                   float* d_chunk, int64_t ld, int chunk_rows, float* d_X, float* d_x_next, float* lambda_out)
{
    if (!ctx) return SD_ERR_INVALID;
    SD_REQUIRE(ctx, images && d_x && d_x_gt && p && reg && d_chunk && d_X && d_x_next, "null argument");
    SD_REQUIRE(ctx, N_local >= 0 && L >= 1 && n_global >= 1 && n_global <= INT_MAX, "bad sample / landmark count");
    SD_REQUIRE(ctx, chunk_rows >= 1, "chunk_rows must be >= 1");
    SD_REQUIRE(ctx, reg->type == 0 || reg->type == 1, "unknown regularisation type");
    const int D = sd_hog_feature_length(L, p), P = 2 * L;
    SD_REQUIRE(ctx, D >= 2, "bad HOG parameters");
    SD_REQUIRE(ctx, ld >= (int64_t)D + P, "ld < D + 2L");
    SD_REQUIRE(ctx, !d_templates || (chunk_rows >= N_local && ldt >= D), "templates need one chunk (chunk_rows >= N_local) and ldt >= D");
    SD_REQUIRE(ctx, d_x_next != d_x, "x_next must not alias x");
    float* mu = (float*)sd_workspace(ctx, SD_WS_LEVEL, (size_t)D * (P + 1) * sizeof(float));
    if (!mu) return SD_ERR_CUDA;
    float* Xc = mu + D;                                   // weights for the shifted rows: what the update multiplies them with
    sd_comm* c = sd_comm_size_of(comm) > 1 ? comm : nullptr;
    float* B = d_chunk + D;                               // [A | b] side by side: the Gram reads both in one pass
    const int chunks = N_local > 0 ? sd_div_up(N_local, chunk_rows) : 1;
    // the pilot shift is the mean of every rank's first chunk (sd_centre_features also checks the all-ones bias column there)
    int64_t n0 = N_local < chunk_rows ? N_local : chunk_rows;
    int rc = c ? sd_comm_sum_int64(ctx, c, &n0) : SD_OK;
    if (rc) return rc;
    if (n0 < 1) return sd_fail(ctx, SD_ERR_INVALID, "sd_train_level: no samples on any rank");
    const bool shifted = D > SD_LU_MAX_DIM && !reg->regularise_last_row;     // otherwise sd_centre_features leaves mu = 0
    for (int k = 0; k < chunks; ++k) {
        const int r0 = k * chunk_rows, rows = N_local - r0 < chunk_rows ? N_local - r0 : chunk_rows;
        rc = hog_rows(ctx, images, d_image_index, d_x, r0, rows, L, hog_eyes, p, d_chunk, ld);                         // :173-189
        if (!rc && d_templates) rc = sd_subtract_templates(ctx, d_chunk, ld, d_templates, ldt, rows, D);             // :191-197
        if (!rc) rc = sd_cascade_targets(ctx, d_x + (int64_t)r0 * P, d_x_gt + (int64_t)r0 * P, rows, P, norm, B, ld); // :199-205
        if (!rc) rc = k == 0 ? sd_centre_features(ctx, c, d_chunk, ld, rows, D, (int)n0, reg, mu)
                             : (shifted ? sd_shift_rows(ctx, d_chunk, ld, rows, D, mu) : SD_OK);
        if (!rc) rc = sd_learn_gram(ctx, d_chunk, ld, B, ld, rows, true, D, P, k > 0);
        if (rc) return rc;
    }
    rc = sd_learn_centred_solve(ctx, c, D, P, reg, (int)n_global, route, mu, d_X, Xc, lambda_out);                    // :207
    if (rc) return rc;
    // :209-215 -- the last chunk is still in the buffer; the others are projected and shifted again
    const int last = (chunks - 1) * chunk_rows;
    rc = sd_cascade_update(ctx, d_chunk, ld, N_local - last, D, Xc, P, d_x + (int64_t)last * P, norm, d_x_next + (int64_t)last * P);
    for (int k = 0; !rc && k + 1 < chunks; ++k) {
        const int r0 = k * chunk_rows;
        rc = hog_rows(ctx, images, d_image_index, d_x, r0, chunk_rows, L, hog_eyes, p, d_chunk, ld);
        if (!rc && shifted) rc = sd_shift_rows(ctx, d_chunk, ld, chunk_rows, D, mu);
        if (!rc) rc = sd_cascade_update(ctx, d_chunk, ld, chunk_rows, D, Xc, P, d_x + (int64_t)r0 * P, norm, d_x_next + (int64_t)r0 * P);
    }
    return rc;
}

int sd_apply_level(sd_ctx* ctx, const sd_image_batch* images, const int32_t* d_image_index, const float* d_x, int N, int L,
                   const sd_normalisation* hog_eyes, const sd_hog_param* p, const sd_normalisation* norm, const float* d_templates,
                   int64_t ldt, const float* d_X, float* d_chunk, int64_t ld, int chunk_rows, float* d_x_next)
{
    if (!ctx) return SD_ERR_INVALID;
    SD_REQUIRE(ctx, images && d_x && p && d_X && d_chunk && d_x_next, "null argument");
    SD_REQUIRE(ctx, N >= 0 && L >= 1, "bad sample / landmark count");
    SD_REQUIRE(ctx, chunk_rows >= 1, "chunk_rows must be >= 1");
    const int D = sd_hog_feature_length(L, p), P = 2 * L;
    SD_REQUIRE(ctx, D >= 2, "bad HOG parameters");
    SD_REQUIRE(ctx, ld >= D, "ld < D");
    SD_REQUIRE(ctx, !d_templates || ldt >= D, "ldt < D");
    SD_REQUIRE(ctx, d_x_next != d_x, "x_next must not alias x");
    int rc = SD_OK;
    for (int r0 = 0; !rc && r0 < N; r0 += chunk_rows) {
        const int rows = N - r0 < chunk_rows ? N - r0 : chunk_rows;
        rc = hog_rows(ctx, images, d_image_index, d_x, r0, rows, L, hog_eyes, p, d_chunk, ld);
        if (!rc && d_templates) rc = sd_subtract_templates(ctx, d_chunk, ld, d_templates + (int64_t)r0 * ldt, ldt, rows, D);
        if (!rc) rc = sd_cascade_update(ctx, d_chunk, ld, rows, D, d_X, P, d_x + (int64_t)r0 * P, norm, d_x_next + (int64_t)r0 * P);
    }
    return rc;
}

}  // extern "C"
