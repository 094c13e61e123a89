// Aligned face chips (include/sd_b200.h, sd_face_chips): a similarity fitted to each face's landmarks, then the face's frame warped
// by cv::warpAffine's fixed-point bilinear rule into a chip.  Two kernels: the fit (one thread per face, float64) and the warp (one
// CTA per tile of a chip, its row and column terms in shared memory).
#include <algorithm>
#include <climits>
#include <cstring>

#include "sd_internal.cuh"
#include "sd_warp.cuh"

namespace {

constexpr int kFitThreads = 128;
constexpr int kTileW = 64, kTileH = 16, kWarpThreads = 256;   // a warp CTA's chip tile: 64 columns x 16 rows
constexpr int kMaxFaces = 65535;                              // faces per warp launch (grid.z)

// One face's fit: M (chip to frame) and its inverse, row-major 2 x 3, and whether the face is valid (valid 0: both zero).
struct ChipFit {
    double m[6], inv[6];
    int32_t valid, frame;
};

__global__ void __launch_bounds__(kFitThreads) face_chip_fit_kernel(
    const int32_t* __restrict__ face_frame, const float* __restrict__ landmarks, int64_t ldl, int num_faces, int L,
    const int32_t* __restrict__ idx, const double* __restrict__ tmpl, int n, const sd_hog_image* __restrict__ frames, int count,
    int w, int h, ChipFit* __restrict__ out, int* __restrict__ status)
{
    const int i = blockIdx.x * kFitThreads + threadIdx.x;
    if (i >= num_faces) return;
    ChipFit r = {};
    const int f = face_frame[i];
    if (f < 0 || f >= count) {
        atomicOr(status, 2);   // the HOG status word's bad image index
        out[i] = r;
        return;
    }
    r.frame = f;
    const float* x = landmarks + (size_t)i * ldl;
    double sux = 0, suy = 0, sxx = 0, sxy = 0;
    bool finite = true;
    for (int j = 0; j < n; ++j) {
        const double px = x[idx[j]], py = x[idx[j] + L];
        finite = finite && isfinite(px) && isfinite(py);
        sux = __dadd_rn(sux, tmpl[2 * j]);
        suy = __dadd_rn(suy, tmpl[2 * j + 1]);
        sxx = __dadd_rn(sxx, px);
        sxy = __dadd_rn(sxy, py);
    }
    const double dn = (double)n;
    const double ux = __ddiv_rn(sux, dn), uy = __ddiv_rn(suy, dn), mx = __ddiv_rn(sxx, dn), my = __ddiv_rn(sxy, dn);
    double den = 0, na = 0, nb = 0;
    for (int j = 0; j < n; ++j) {
        const double dux = __dsub_rn(tmpl[2 * j], ux), duy = __dsub_rn(tmpl[2 * j + 1], uy);
        const double dx = __dsub_rn((double)x[idx[j]], mx), dy = __dsub_rn((double)x[idx[j] + L], my);
        den = __dadd_rn(den, __dadd_rn(__dmul_rn(dux, dux), __dmul_rn(duy, duy)));
        na = __dadd_rn(na, __dadd_rn(__dmul_rn(dux, dx), __dmul_rn(duy, dy)));
        nb = __dadd_rn(nb, __dsub_rn(__dmul_rn(dux, dy), __dmul_rn(duy, dx)));
    }
    if (finite && den != 0) {
        const double a = __ddiv_rn(na, den), b = __ddiv_rn(nb, den), s = __dadd_rn(__dmul_rn(a, a), __dmul_rn(b, b));
        const double tx = __dsub_rn(mx, __dsub_rn(__dmul_rn(a, ux), __dmul_rn(b, uy)));
        const double ty = __dsub_rn(my, __dadd_rn(__dmul_rn(b, ux), __dmul_rn(a, uy)));
        const double m[6] = {a, -b, tx, b, a, ty};
        const sd_hog_image& fr = frames[f];
        if (s != 0 && sd_warp_fits(m, w, h, fr.width > 32767 || fr.height > 32767)) {
            const double ia = __ddiv_rn(a, s), ib = __ddiv_rn(b, s);
            const double inv[6] = {ia, ib, -__dadd_rn(__dmul_rn(ia, tx), __dmul_rn(ib, ty)),
                                   -ib, ia, __dsub_rn(__dmul_rn(ib, tx), __dmul_rn(ia, ty))};
            for (int k = 0; k < 6; ++k) { r.m[k] = m[k]; r.inv[k] = inv[k]; }
            r.valid = 1;
        }
    }
    out[i] = r;
}

// The pixel of tap (x, y), channel c, or 0 outside the frame
template <class T>
__device__ __forceinline__ T tap(const T* __restrict__ src, const sd_hog_image& fr, int x, int y, int c)
{
    if (x < 0 || y < 0 || x >= fr.width || y >= fr.height) return T(0);
    return __ldg(src + fr.offset + (int64_t)y * fr.row_stride + (int64_t)x * fr.pixel_stride + (int64_t)c * fr.channel_stride);
}

// CTA (tile x, tile y, face f0 + z): the tile's kTileH rows x kTileW columns x C channels of the chip, each output row of the tile
// stored as one contiguous run of elements.  The CTA of tile (0, 0) also writes the face's transforms and valid byte.
template <class T>
__global__ void __launch_bounds__(kWarpThreads) face_chip_warp_kernel(
    const T* __restrict__ src, const sd_hog_image* __restrict__ frames, const ChipFit* __restrict__ fits, int f0, int w, int h, int C,
    T* __restrict__ chips, double* __restrict__ c2f, double* __restrict__ f2c, uint8_t* __restrict__ valid)
{
    __shared__ int s_ad[kTileW], s_bd[kTileW], s_x0[kTileH], s_y0[kTileH];
    const int face = f0 + blockIdx.z;
    const ChipFit& fit = fits[face];
    const int tx0 = blockIdx.x * kTileW, ty0 = blockIdx.y * kTileH;
    const int tw = min(kTileW, w - tx0), th = min(kTileH, h - ty0);
    const bool ok = fit.valid != 0;
    if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x < 13) {
        const int k = threadIdx.x;
        if (k < 6) c2f[(size_t)face * 6 + k] = fit.m[k];
        else if (k < 12) f2c[(size_t)face * 6 + k - 6] = fit.inv[k - 6];
        else valid[face] = (uint8_t)fit.valid;
    }
    if (ok) {
        // the per-column and per-row terms, once per tile (valid faces fit int32: sd_warp_fits)
        if (threadIdx.x < kTileW && threadIdx.x < tw) {
            const double X = (double)(tx0 + threadIdx.x);
            const int2 d = sd_warp_col(fit.m, X);
            s_ad[threadIdx.x] = d.x;
            s_bd[threadIdx.x] = d.y;
        } else if (threadIdx.x >= 128 && threadIdx.x - 128 < th) {
            const int r = threadIdx.x - 128;
            const double Y = (double)(ty0 + r);
            const int2 t = sd_warp_row(fit.m, Y);
            s_x0[r] = t.x;
            s_y0[r] = t.y;
        }
        __syncthreads();
    }
    const sd_hog_image fr = frames[fit.frame];
    const int run = tw * C;   // elements of one tile row
    T* out = chips + ((size_t)face * h + ty0) * w * C + (size_t)tx0 * C;
    for (int e = threadIdx.x; e < th * run; e += kWarpThreads) {
        const int r = e / run, q = e - r * run, col = q / C, c = q - col * C;
        T v = T(0);
        if (ok) {
            const int sx = (s_x0[r] + s_ad[col]) >> 5, sy = (s_y0[r] + s_bd[col]) >> 5;
            v = sd_warp_sample<T>(sx, sy, [&](int x, int y) { return tap(src, fr, x, y, c); });
        }
        out[(size_t)r * w * C + q] = v;
    }
}

}  // namespace

int sd_face_chip_template(const sd_model* m, int width, int height, double padding, int n, const int32_t* h_landmark, double* h_template)
{
    if (!m || !h_template || width < 1 || height < 1 || !std::isfinite(padding) || padding <= -0.5 || n < 1) return SD_ERR_INVALID;
    const int L = sd_model_num_landmarks(m);
    if (!h_landmark && n != L) return SD_ERR_INVALID;
    for (int j = 0; h_landmark && j < n; ++j)
        if (h_landmark[j] < 0 || h_landmark[j] >= L) return SD_ERR_INVALID;
    std::vector<float> mean(2 * (size_t)L);
    if (const int rc = sd_model_get_mean(m, mean.data())) return rc;
    const double den = 1.0 + 2.0 * padding;
    for (int j = 0; j < n; ++j) {
        const int k = h_landmark ? h_landmark[j] : j;
        volatile double x = (double)mean[k] + 0.5;   // volatile: each operation rounded on its own on any host compiler
        x = x + padding;
        x = x / den;
        h_template[2 * j] = x * (double)width;
        volatile double y = (double)mean[k + L] + 0.5;
        y = y + padding;
        y = y / den;
        h_template[2 * j + 1] = y * (double)height;
    }
    return SD_OK;
}

int sd_face_chips(sd_ctx* ctx, const sd_hog_images* frames, const int32_t* d_face_frame, const float* d_landmarks, int64_t ldl,
                  int num_faces, int num_landmarks, const sd_face_chip_param* p, void* d_chips, double* d_chip_to_frame,
                  double* d_frame_to_chip, uint8_t* d_valid)
{
    if (!ctx) return SD_ERR_INVALID;
    SD_REQUIRE(ctx, frames && p && p->h_landmark && p->h_template, "null pointer");
    SD_REQUIRE(ctx, num_faces >= 0, "num_faces < 0");
    SD_REQUIRE(ctx, num_faces == 0 || (d_face_frame && d_landmarks && d_chips && d_chip_to_frame && d_frame_to_chip && d_valid),
               "null pointer");
    SD_REQUIRE(ctx, num_landmarks >= 1 && ldl >= 2 * (int64_t)num_landmarks, "need num_landmarks >= 1 and ldl >= 2 num_landmarks");
    SD_REQUIRE(ctx, p->n >= 2, "need at least 2 landmarks");
    std::vector<char> used(num_landmarks, 0);
    for (int j = 0; j < p->n; ++j) {
        const int k = p->h_landmark[j];
        SD_REQUIRE(ctx, k >= 0 && k < num_landmarks, "landmark index out of range");
        SD_REQUIRE(ctx, !used[k], "landmark index listed twice");
        used[k] = 1;
    }
    SD_REQUIRE(ctx, p->width >= 1 && p->height >= 1, "chip size below 1 x 1");
    SD_REQUIRE(ctx, (int64_t)p->width * p->height <= INT32_MAX, "chip of more than INT32_MAX pixels");
    SD_REQUIRE(ctx, sd_div_up(p->height, kTileH) <= 65535, "chip taller than 1,048,560 px");
    SD_REQUIRE(ctx, frames->dtype == SD_HOG_U8 || frames->dtype == SD_HOG_F32, "unknown dtype");
    SD_REQUIRE(ctx, frames->channels >= 1 && frames->channels <= 16, "channels must be in [1, 16]");
    SD_REQUIRE(ctx, frames->count >= 1 && frames->d_data, "no frames");
    const int C = frames->channels, es = frames->dtype == SD_HOG_F32 ? 4 : 1;
    const int64_t chip_elems = (int64_t)p->width * p->height * C;
    SD_REQUIRE(ctx, num_faces == 0 || chip_elems * es <= INT64_MAX / num_faces, "chip bytes overflow int64");
    SD_REQUIRE(ctx, sd_aligned(d_landmarks, 4) && sd_aligned(d_face_frame, 4) && sd_aligned(d_chip_to_frame, 8) &&
                    sd_aligned(d_frame_to_chip, 8) && (es == 1 || (sd_aligned(frames->d_data, 4) && sd_aligned(d_chips, 4))),
               "unaligned pointer");
    HogPyramidFrames fr;
    if (const int rc = sd_hog_read_image_frames(ctx, __func__, frames, 0, &fr)) return rc;
    if (num_faces == 0) return SD_OK;

    // scratch: [fits | frame table | indices | template], each part 16-byte aligned
    const int n = p->n, count = frames->count;
    const size_t fit_bytes = sd_round16(sizeof(ChipFit) * (size_t)num_faces), tab_bytes = sd_round16(sizeof(sd_hog_image) * (size_t)count),
                 idx_bytes = sd_round16(sizeof(int32_t) * (size_t)n);
    uint8_t* ws = static_cast<uint8_t*>(sd_workspace(ctx, SD_WS_CHIPS, fit_bytes + tab_bytes + idx_bytes + sizeof(double) * 2 * n));
    if (!ws) return SD_ERR_CUDA;
    ChipFit* fits = reinterpret_cast<ChipFit*>(ws);
    sd_hog_image* d_tab = reinterpret_cast<sd_hog_image*>(ws + fit_bytes);
    int32_t* d_idx = reinterpret_cast<int32_t*>(ws + fit_bytes + tab_bytes);
    double* d_tmpl = reinterpret_cast<double*>(ws + fit_bytes + tab_bytes + idx_bytes);
    SD_CUDA(ctx, cudaMemcpyAsync(d_tab, fr.frames.data(), sizeof(sd_hog_image) * count, cudaMemcpyHostToDevice, ctx->stream));
    SD_CUDA(ctx, cudaMemcpyAsync(d_idx, p->h_landmark, sizeof(int32_t) * n, cudaMemcpyHostToDevice, ctx->stream));
    SD_CUDA(ctx, cudaMemcpyAsync(d_tmpl, p->h_template, sizeof(double) * 2 * n, cudaMemcpyHostToDevice, ctx->stream));

    int* d_status = reinterpret_cast<int*>(ctx->d_scratch) + 1;
    face_chip_fit_kernel<<<sd_div_up(num_faces, kFitThreads), kFitThreads, 0, ctx->stream>>>(
        d_face_frame, d_landmarks, ldl, num_faces, num_landmarks, d_idx, d_tmpl, n, d_tab, count, p->width, p->height, fits, d_status);
    SD_LAUNCH_CHECK(ctx, "face_chip_fit_kernel");
    int* h_status = reinterpret_cast<int*>(ctx->h_scratch) + 1;
    SD_CUDA(ctx, cudaMemcpyAsync(h_status, d_status, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    SD_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (*h_status & 2) {
        SD_CUDA(ctx, cudaMemsetAsync(d_status, 0, sizeof(int), ctx->stream));
        return sd_fail(ctx, SD_ERR_INVALID, "sd_face_chips: a face's frame index is out of range");
    }

    const dim3 block(kWarpThreads);
    for (int f0 = 0; f0 < num_faces; f0 += kMaxFaces) {
        const dim3 grid(sd_div_up(p->width, kTileW), sd_div_up(p->height, kTileH), (unsigned)std::min(num_faces - f0, kMaxFaces));
        if (es == 4)
            face_chip_warp_kernel<float><<<grid, block, 0, ctx->stream>>>(
                static_cast<const float*>(frames->d_data), d_tab, fits, f0, p->width, p->height, C, static_cast<float*>(d_chips),
                d_chip_to_frame, d_frame_to_chip, d_valid);
        else
            face_chip_warp_kernel<uint8_t><<<grid, block, 0, ctx->stream>>>(
                static_cast<const uint8_t*>(frames->d_data), d_tab, fits, f0, p->width, p->height, C, static_cast<uint8_t*>(d_chips),
                d_chip_to_frame, d_frame_to_chip, d_valid);
        SD_LAUNCH_CHECK(ctx, "face_chip_warp_kernel");
    }
    return SD_OK;
}
