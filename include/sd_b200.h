/*
 * sd_b200.h -- C ABI of the H100-native cascaded-regression engine.
 *
 * This is the drop-in boundary for the hot path of patrikhuber/superviseddescent
 * (HOG projection -> LinearRegressor::learn -> predict/detect cascade).  Plain C:
 * opaque handles, raw pointers, explicit sizes, int status codes.  No C++ / torch
 * types cross this boundary.  The C++14 header shells in
 * superviseddescent_b200/include/ (same class names and call signatures as the
 * reference) and the ctypes binding in superviseddescent_b200/ sit on top of it.
 *
 * Conventions (reference: SURVEY.md 8b)
 *   - matrices are row-major float32, one sample per row (cv::Mat CV_32FC1 as the
 *     reference uses it, regressors.hpp:202-206); `ld` = row stride in floats.
 *   - landmark rows are [x_0..x_{L-1}, y_0..y_{L-1}] (adaptive_vlhog.hpp:96-97).
 *   - device images are 8-bit single channel (adaptive_vlhog.hpp:115-120 grey path); host frames (sd_host_frame) are
 *     8UC1 or 8UC3 B,G,R and reach the device as grey frames (sd_upload_frames, sd_detect_faces_host).
 *   - pointers named d_* are DEVICE pointers, h_* are HOST pointers.
 *   - every call is asynchronous on the context's stream unless it returns host
 *     data; sd_sync() waits.  Functions are re-entrant on distinct contexts.
 *   - return value 0 = SD_OK; otherwise an sd_status and sd_last_error(ctx) holds
 *     a message.  There is NO CPU fallback: without a usable GPU every compute
 *     entry point fails with SD_ERR_CUDA.
 *
 * Citations are file:line under the reference tree (/root/reference).
 */
#ifndef SD_B200_H
#define SD_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define SD_API __attribute__((visibility("default")))
#else
#define SD_API
#endif

typedef enum {
    SD_OK = 0,
    SD_ERR_INVALID = 1,    /* bad argument / shape (the reference asserts) */
    SD_ERR_CUDA = 2,       /* CUDA runtime / driver failure, or no GPU */
    SD_ERR_IO = 3,         /* model file could not be opened/parsed (model.hpp:199 throws) */
    SD_ERR_MISSING_ID = 4, /* eye identifier not among the landmarks (helpers.hpp:144,153 throws) */
    SD_ERR_NUMERIC = 5,    /* non-finite result / non-positive pivot */
    SD_ERR_UNSUPPORTED = 6
} sd_status;

typedef struct sd_ctx sd_ctx;       /* one per host thread / stream */
typedef struct sd_model sd_model;   /* rcr::detection_model resident on the device */
typedef struct sd_comm sd_comm;     /* multi-GPU communicator (see "multi-GPU training" below) */

/* rcr::HoGParam (adaptive_vlhog.hpp:41-60); same field order as its cereal archive */
typedef struct {
    int32_t variant;             /* 0 = VlHogVariantDalalTriggs, 1 = VlHogVariantUoctti (hog.h:70) */
    int32_t num_cells;
    int32_t cell_size;
    int32_t num_bins;            /* undirected orientations K */
    float relative_patch_size;   /* patch width as a fraction of the inter-eye distance */
} sd_hog_param;

/* superviseddescent::Regulariser (regressors.hpp:87-169) */
typedef struct {
    int32_t type;                /* 0 = Manual, 1 = MatrixNorm (regressors.hpp:93-97) */
    float param;                 /* lambda, or the factor applied to ||AtA||_F / N */
    int32_t regularise_last_row; /* 0: the bias row gets no lambda (regressors.hpp:143-146) */
} sd_regulariser;

/* NormalisationStrategy of the optimiser: NoNormalisation (superviseddescent.hpp:60-74)
 * or rcr::InterEyeDistanceNormalisation (model.hpp:84-116).  Eye landmarks are given as
 * row indices into the landmark list (the host shells resolve the string ids). */
typedef struct {
    int32_t kind;                /* 0 = none, 1 = inter-eye distance */
    int32_t n_right, n_left;     /* 1..4 each */
    int32_t right_idx[4];
    int32_t left_idx[4];
} sd_normalisation;

/* Region of interest of one frame that is resident on the device (see sd_image_batch.d_roi). */
typedef struct {
    int32_t x, y, w, h;          /* in frame coordinates */
    int32_t row_stride;          /* bytes between ROI rows in the packed buffer (multiple of 4) */
    int32_t reserved;
    int64_t offset;              /* byte offset of the ROI's first pixel from d_data */
} sd_roi;

/* One frame of a batch whose frames differ in size (the reference's HogTransform takes a std::vector<cv::Mat> of arbitrary
 * sizes: rcr-train and examples/landmark_detection.cpp train on photographs of different resolutions). */
typedef struct {
    int32_t width, height;       /* defines where the zero padding of a patch starts for THIS frame */
    int32_t row_stride;          /* bytes */
    int32_t reserved;
    int64_t offset;              /* byte offset of the frame's first pixel from d_data */
} sd_frame;

/* A batch of 8UC1 images resident on the device: equally sized (width/height/strides below), or -- d_frames != NULL -- one
 * descriptor per frame. */
typedef struct {
    const uint8_t* d_data;
    int32_t width, height;       /* frame size: defines where the zero padding of a patch starts */
    int32_t row_stride;          /* bytes */
    int64_t image_stride;        /* bytes between consecutive images */
    int32_t count;
    /* Optional (NULL = whole frames are resident): only a region of interest of every frame was uploaded.
     * d_roi[i] locates it inside d_data; a patch that needs frame pixels outside its ROI sets d_roi_miss[i]
     * (sd_detect_faces_host then repeats that face from the full frame). */
    const sd_roi* d_roi;
    uint8_t* d_roi_miss;
    /* Optional (NULL = equally sized frames): per-frame size / pitch / position; width, height, row_stride and image_stride
     * above are then ignored.  Together with d_roi, d_frames[i] supplies only the width and height of frame i (where its zero
     * padding starts): the pixels are where d_roi[i] says. */
    const sd_frame* d_frames;
} sd_image_batch;

/* One host frame (sd_detect_faces_host, sd_upload_frames): 8UC1, or 8UC3 with interleaved B,G,R (converted exactly as
 * sd_bgr2gray does). */
typedef struct {
    const uint8_t* h_data;
    int32_t width, height;
    int32_t row_stride;          /* bytes, >= width * channels */
    int32_t channels;            /* 1 or 3 */
} sd_host_frame;

/* ---- context --------------------------------------------------------------------------- */
/* stream: a cudaStream_t owned by the caller (e.g. torch's current stream); NULL is the CUDA default
 * stream (which is also torch's default stream); SD_STREAM_OWN lets the context create and own a
 * non-blocking stream. */
#define SD_STREAM_OWN ((void*)(intptr_t)-1)
SD_API int sd_ctx_create(int device, void* stream, sd_ctx** out);
SD_API void sd_ctx_destroy(sd_ctx* ctx);
SD_API const char* sd_last_error(const sd_ctx* ctx);
SD_API int sd_sync(sd_ctx* ctx);
/* the cudaStream_t the context runs on (what sd_ctx_create was given, or the stream it created) */
SD_API void* sd_ctx_stream(const sd_ctx* ctx);
SD_API const char* sd_version(void);
/* number of kernels of THIS library launched on ctx since creation (bench.py's gpu_launches) */
SD_API int64_t sd_launch_count(const sd_ctx* ctx);
/* faces that sd_detect_faces_host (and sd_detect_batch_host through it) had to repeat from their full frame (a patch left the
 * uploaded ROI) */
SD_API int64_t sd_roi_fallback_count(const sd_ctx* ctx);

/* device / pinned-host memory for hosts that do not bring their own allocator */
SD_API int sd_malloc(sd_ctx* ctx, size_t bytes, void** d_ptr);
SD_API int sd_free(sd_ctx* ctx, void* d_ptr);
SD_API int sd_host_alloc(sd_ctx* ctx, size_t bytes, void** h_ptr);   /* pinned */
SD_API int sd_host_free(sd_ctx* ctx, void* h_ptr);
SD_API int sd_memcpy_h2d(sd_ctx* ctx, void* d_dst, const void* h_src, size_t bytes);  /* async */
SD_API int sd_memcpy_d2h(sd_ctx* ctx, void* h_dst, const void* d_src, size_t bytes);  /* async */
SD_API int sd_memset(sd_ctx* ctx, void* d_dst, int value, size_t bytes);
/* strided rows in one call (cv::Mat rows with a step, or [A | B] side by side on the device): `rows` rows of `row_bytes`
 * bytes, pitches in bytes; async on the context's stream */
SD_API int sd_memcpy2d_h2d(sd_ctx* ctx, void* d_dst, size_t dst_pitch, const void* h_src, size_t src_pitch, size_t row_bytes, size_t rows);
SD_API int sd_memcpy2d_d2h(sd_ctx* ctx, void* h_dst, size_t dst_pitch, const void* d_src, size_t src_pitch, size_t row_bytes, size_t rows);
SD_API int sd_memcpy2d_d2d(sd_ctx* ctx, void* d_dst, size_t dst_pitch, const void* d_src, size_t src_pitch, size_t row_bytes, size_t rows);

/* ---- projection h: rcr::HogTransform::operator() batched (adaptive_vlhog.hpp:109-185) -- */
/* D = L * num_cells^2 * (3K+4 | 4K) + 1 */
SD_API int sd_hog_feature_length(int num_landmarks, const sd_hog_param* p);
/* Asynchronous.  A degenerate sample (inter-eye distance too small for a patch: the reference's cv::resize would throw) or an
 * image index out of range raises a flag on the device that the NEXT synchronising call on the context reports as
 * SD_ERR_INVALID: sd_sync, sd_hog_debug, sd_detect_batch_device / _host.
 * For sample i: image = images[d_image_index ? d_image_index[i] : i], landmarks = d_x[i, 0:2L].
 * Writes the reference's feature row (per landmark [dim][cell col][cell row], then bias 1)
 * to d_A[i*ld .. i*ld + D).  Columns [D, ld) are left untouched.  hog.c:174-204,595-728,857-1062
 * run fused with the crop / zero-pad / cv::resize glue of adaptive_vlhog.hpp:123-176.
 * eyes == NULL (or eyes->kind == 0) selects the NON-adaptive HogTransform of the hello-world example
 * (examples/landmark_detection.cpp:195-261): patch half-size = num_cells * (cell_size / 2), no resize,
 * relative_patch_size ignored; cell_size must be even.  That functor has no bias column: use the first D - 1 columns. */
SD_API int sd_hog_batch(sd_ctx* ctx, const sd_image_batch* images, const int32_t* d_image_index,
                        const float* d_x, int64_t ldx, int num_samples, int num_landmarks,
                        const sd_normalisation* eyes, const sd_hog_param* p,
                        float* d_A, int64_t ld);
/* parity taps (integer results that must match the reference exactly): per (sample, landmark)
 * patch centre/half size, and optionally the resized u8 patches and per-pixel orientation bins. */
SD_API int sd_hog_debug(sd_ctx* ctx, const sd_image_batch* images, const int32_t* d_image_index,
                        const float* d_x, int64_t ldx, int num_samples, int num_landmarks,
                        const sd_normalisation* eyes, const sd_hog_param* p,
                        int32_t* d_geometry /* N*L*3: cx, cy, half */,
                        uint8_t* d_patches /* N*L*fs*fs or NULL */,
                        int8_t* d_bins /* N*L*fs*fs or NULL, -1 on border / zero gradient */);

/* Colour frames: HogTransform::operator() converts 3-channel images with cv::cvtColor(BGR2GRAY) before anything else
 * (adaptive_vlhog.hpp:114-120).  Same conversion on the device, once per frame instead of once per call:
 *   gray = (3735 B + 19235 G + 9798 R + 2^14) >> 15      (OpenCV >= 3 fixed point; SURVEY.md 8c, pinned against cv2)
 * d_bgr: count frames of height x width interleaved B,G,R bytes; strides in bytes. */
SD_API int sd_bgr2gray(sd_ctx* ctx, const uint8_t* d_bgr, int width, int height, int64_t bgr_row_stride,
                       int64_t bgr_image_stride, int count, uint8_t* d_gray, int64_t gray_row_stride,
                       int64_t gray_image_stride);
/* Host frames (8UC1 or 8UC3 B,G,R, any sizes and row strides) -> one grey batch for sd_hog_batch, the upload of
 * HogTransform's images.  d_buf == NULL: *bytes receives the size d_buf needs and nothing else happens.  Otherwise d_buf
 * (16-byte aligned, *bytes long) receives the grey frames at a 16-byte pitch, followed by the sd_frame table if the sizes
 * differ; *out describes the batch (plain strided batch when all frames share one size).  Colour is converted as
 * sd_bgr2gray does, through context-owned scratch (never d_buf).  Returns when the copies are done.
 * A bad frame (as for sd_detect_faces_host), count < 1, an unaligned d_buf or a *bytes below the size query's are
 * SD_ERR_INVALID before any work is queued (d_buf is not written). */
SD_API int sd_upload_frames(sd_ctx* ctx, const sd_host_frame* frames, int count, void* d_buf, size_t* bytes, sd_image_batch* out);

/* ---- dense HOG of whole frames: vl_hog_put_image (one channel) + vl_hog_extract (hog.c:595-728, :857-1062) -------------
 * The general HOG API the reference ships (hog.h:104-139) on every 8-bit grey frame of a batch, e.g. the input of a
 * sliding-window detector.  Output per frame: VLFeat's planar layout [dd][hogH][hogW], x fastest, with
 *   hogW = (width + cell_size / 2) / cell_size, hogH = (height + cell_size / 2) / cell_size     (hog.c:542-543)
 *   dd   = 3 * num_bins + 4 (variant 1, UoCTTI) or 4 * num_bins (variant 0, Dalal-Triggs).
 * Valid arguments: width and height > 3 with hogW, hogH > 0 (hog.c:545-548), num_bins in [1, 16], cell_size in [1, 32],
 * variant 0 or 1.  Orientations are assigned to the nearest bin (no bilinear orientation assignment), as rcr::HogTransform
 * uses vl_hog; sd_hog_dense_images below adds float and multi-channel frames and bilinear assignment.  Each feature lies within its float64 error bar, a median
 * 50 to 80 units of 2^-24 of its value (the votes of a cell are summed in a different, fixed order than hog.c's; at most 0.78 of
 * that bar on an H100); a
 * frame of num_cells * cell_size pixels square gives bit for bit the features sd_hog_batch computes for the same fixed patch.
 *
 * sd_hog_dense_shape: host only.  Writes hogW, hogH and dd, or returns SD_ERR_INVALID for an invalid configuration. */
SD_API int sd_hog_dense_shape(int width, int height, int cell_size, int num_bins, int variant, int* hog_w, int* hog_h, int* dd);
/* sd_hog_dense: asynchronous on the context's stream.  Frame i's features start at d_out + d_out_offset[i] (offsets in floats,
 * a device array of images->count int64), or, with d_out_offset == NULL (allowed only when all frames have one size), at
 * d_out + i * dd * hogH * hogW.  Frames of different sizes (images->d_frames) need the offsets, computed with
 * sd_hog_dense_shape; the call then reads the frame table back once before it queues work.  Each frame's features depend on
 * that frame alone: the same in any batch, and the same in every run.  A batch with d_roi, an invalid configuration, or a
 * frame that breaks the size rule is SD_ERR_INVALID before any work is queued (d_out is not written). */
SD_API int sd_hog_dense(sd_ctx* ctx, const sd_image_batch* images, int cell_size, int num_bins, int variant, float* d_out,
                        const int64_t* d_out_offset);

/* ---- dense HOG pyramid: every frame of a batch at every scale, in one call --------------------------------------------------
 * The level of a width x height frame at scale s is level_w x level_h px with level_w = floor(width * s + 0.5) and
 * level_h = floor(height * s + 0.5), in double.  Each level is resized from the frame itself (not from another level) by
 * cv::resize INTER_LINEAR's 8-bit fixed-point rule, the resize of sd_hog_batch's patches, with the per-axis scale
 * 1 / (level_w / width) in double; a level of the frame's own size is the frame.  Its features are bit for bit sd_hog_dense's
 * of the resized frame, [dd][hog_h][hog_w] at d_out + d_out_offset[frame * num_scales + s] (floats; a device array of
 * count * num_scales int64).  A level narrower or lower than 4 px, or whose cell grid is empty, is empty: hog_w = hog_h = 0,
 * nothing is written and its offset is not read.  Scales must be finite and in (0, 4], and levels at most 2^28 px per side.
 * Cell (x, y) of a level starts at pixel (x * cell_size * width / level_w, y * cell_size * height / level_h) of the frame.
 *
 * sd_hog_pyramid_shape: host only.  Writes the level's size, its hog_w, hog_h (0 for an empty level) and dd, or returns
 * SD_ERR_INVALID for a frame smaller than 1 x 1, an invalid scale or an invalid configuration. */
SD_API int sd_hog_pyramid_shape(int width, int height, double scale, int cell_size, int num_bins, int variant,
                                int* level_w, int* level_h, int* hog_w, int* hog_h, int* dd);
/* sd_hog_pyramid: asynchronous on the context's stream; h_scales is a host array of num_scales scales.  Frames are an
 * sd_image_batch as for sd_hog_dense: equally sized, or per-frame d_frames (the call then reads the table back once); host
 * and colour frames reach the device through sd_upload_frames.  The resized levels go through context scratch, one slice of
 * the batch at a time (about 64 MB of levels per slice), so the scratch does not grow with the batch.  Each level's features
 * depend on its frame and scale alone.  Null pointers, a batch with d_roi, num_scales < 1, an invalid scale or configuration,
 * or a frame smaller than 1 x 1 is SD_ERR_INVALID before any work is queued (d_out is not written). */
SD_API int sd_hog_pyramid(sd_ctx* ctx, const sd_image_batch* images, const double* h_scales, int num_scales,
                          int cell_size, int num_bins, int variant, float* d_out, const int64_t* d_out_offset);

/* ---- dense HOG of 8-bit or float frames with 1..16 channels: every input of vl_hog_put_image (hog.c:595-728) ----------------
 * One frame: element (x, y, c) at offset + y * row_stride + x * pixel_stride + c * channel_stride, in ELEMENTS of the batch's
 * dtype.  VLFeat's planar layout is pixel_stride = 1, channel_stride = height * row_stride; the interleaved layout of OpenCV
 * and numpy (H, W, C) is pixel_stride = C, channel_stride = 1.  Offset and strides are non-negative. */
typedef struct {
    int32_t width, height;
    int64_t offset, row_stride, pixel_stride, channel_stride;
} sd_hog_image;
#define SD_HOG_U8 0
#define SD_HOG_F32 1
/* A batch of frames resident on the device: equally sized (frame i at frame.offset + i * image_stride elements), or --
 * d_frames != NULL -- one device descriptor per frame (frame and image_stride are then ignored). */
typedef struct {
    const void* d_data;          /* SD_HOG_F32: 4-byte aligned */
    int32_t dtype;               /* SD_HOG_U8 or SD_HOG_F32 */
    int32_t channels;            /* 1..16, the same for every frame */
    int32_t count;
    sd_hog_image frame;
    int64_t image_stride;        /* elements */
    const sd_hog_image* d_frames;
} sd_hog_images;
/* sd_hog_dense_images: vl_hog_new(variant, num_bins) + vl_hog_set_use_bilinear_orientation_assignments(bilinear_orientations)
 * + vl_hog_put_image(frame, channels, cell_size) + vl_hog_extract on every frame, asynchronous on the context's stream.  At each
 * pixel the gradient comes from the channel with the largest squared modulus (the first on a tie; hog.c:631-644); channels are
 * taken as given (no colour conversion).  bilinear_orientations = 1: each pixel votes into its two nearest orientation bins
 * (hog.c:674-678), each vote weighted by the orientation weight squared, as hog.c:706-714 does.  Output, offsets, size rule
 * and frame independence as sd_hog_dense (sd_hog_dense_shape gives the shape).  Nearest-bin features of 8-bit frames are bit
 * for bit those of sd_hog_dense on the same pixels, and those of float frames holding the same values.  An unknown dtype,
 * channels outside [1, 16], an unaligned float buffer, a negative offset or stride, a frame that breaks the size rule, or an
 * invalid configuration is SD_ERR_INVALID before any work is queued (d_out is not written). */
SD_API int sd_hog_dense_images(sd_ctx* ctx, const sd_hog_images* images, int cell_size, int num_bins, int variant,
                               int bilinear_orientations, float* d_out, const int64_t* d_out_offset);

/* ---- dense HOG of a caller's gradient fields: vl_hog_put_polar_field + vl_hog_extract (hog.c:746-845, :857-1062) ----------
 * Each field is a modulus and an angle per pixel, e.g. the gradient of another operator, colour gradients combined by the
 * caller, or an optical flow's magnitude and direction (histograms of flow).  One sd_hog_image places element (x, y) at
 * offset + y * row_stride + x * pixel_stride of BOTH buffers: two separate planes, or an interleaved (H, W, 2) array with
 * d_angle = d_modulus + 1 and pixel_stride = 2.  channel_stride is not read (it must not be negative, as everywhere). */
typedef struct {
    const float* d_modulus;          /* 4-byte aligned */
    const float* d_angle;            /* 4-byte aligned; same element layout as d_modulus */
    int32_t count;
    sd_hog_image frame;              /* equally sized fields: field i at frame.offset + i * image_stride */
    int64_t image_stride;            /* elements */
    const sd_hog_image* d_frames;    /* optional: one descriptor per field, as in sd_hog_images */
} sd_hog_polar_fields;
/* sd_hog_dense_polar: vl_hog_new(variant, num_bins) + vl_hog_set_use_bilinear_orientation_assignments(bilinear_orientations)
 * + vl_hog_put_polar_field(modulus, angle, directed, width, height, cell_size) + vl_hog_extract on every field, asynchronous on
 * the context's stream.  Every pixel votes, the border rows and columns included; a modulus <= 0 does not (a NaN modulus
 * does, as in hog.c).  ho = angle / (pi / num_bins) selects the bin floor(ho) or floor(ho) + 1 (nearest, a tie to the second),
 * or both, weighted 1 - frac(ho) and frac(ho) (bilinear), each taken modulo 2 * num_bins (directed = 1) or num_bins
 * (directed = 0); a vote carries modulus * wx * wy * w_o^2 as in hog.c.  Two cases hog.c leaves undefined have a defined
 * result: a pixel whose ho is not a finite float (a NaN or infinite angle, or a quotient that overflows float) does not vote,
 * and the residue is computed exactly without hog.c's loop, so angles of any magnitude (|ho| >= 2^63 included) vote into
 * the exact bin.  Output, offsets, size rule and frame independence as sd_hog_dense_images (sd_hog_dense_shape gives the
 * shape).  Null or unaligned field pointers, directed or bilinear_orientations outside {0, 1}, a negative offset or stride, a
 * field that breaks the size rule, an invalid configuration, or fields of different sizes without d_out_offset is
 * SD_ERR_INVALID before any work is queued (d_out is not written). */
SD_API int sd_hog_dense_polar(sd_ctx* ctx, const sd_hog_polar_fields* fields, int cell_size, int num_bins, int variant,
                              int directed, int bilinear_orientations, float* d_out, const int64_t* d_out_offset);

/* ---- render, flip and transpose of planar HOG features: vl_hog_render, vl_hog_get_permutation (hog.c:225-312, :428-495) ----
 * Features are VLFeat's planar layout [dd][h][w] of a grid of w x h cells (what the dense HOG calls above write), with dd and
 * the variant as there.  A rendered grid is an image of h * 21 rows of w * 21 floats, row-major: cell (x, y) owns the 21 x 21
 * tile at column 21 x, row 21 y.  sd_hog_permutation and sd_hog_glyphs are host only: the tables vl_hog_new builds. */
#define SD_HOG_GLYPH_SIZE 21
/* One grid of a batch: its features at d_features + offset, its result at d_out + out_offset (floats, non-negative). */
typedef struct {
    int32_t width, height;           /* cells, >= 1 */
    int64_t offset, out_offset;
} sd_hog_grid;
/* A batch of grids on the device: equally sized (width x height cells; grid i's features at d_features + i * dd * h * w, its
 * result packed the same way: i * h * w * 441 floats for a render, i * dd * h * w for a relayout), or -- d_grids != NULL --
 * one device descriptor per grid (width and height are then ignored; the call reads the table back once). */
typedef struct {
    const float* d_features;
    int32_t count;
    int32_t width, height;
    const sd_hog_grid* d_grids;
} sd_hog_grids;
/* sd_hog_permutation: writes the dd entries of vl_hog_get_permutation: the features of a left-right mirrored image are
 * flipped[i] = features[perm[i]] at the mirrored cell.  sd_hog_glyphs: writes the num_bins x 21 x 21 glyphs of vl_hog_new
 * (each value 0 or 1, glyph k row-major; transposed = 1 gives the column-major glyphs of a transposed VlHog).  Either returns
 * SD_ERR_INVALID for a null pointer, num_bins outside [1, 16], or variant / transposed outside {0, 1}. */
SD_API int sd_hog_permutation(int num_bins, int variant, int64_t* perm);
SD_API int sd_hog_glyphs(int num_bins, int transposed, float* glyphs);
/* sd_hog_render: vl_hog_render of every grid into d_image, asynchronous on the context's stream.  Read-modify-write, as hog.c
 * adds into the caller's buffer: zero the image first for a fresh render.  Per cell, weight k is the sum of the orientation's 3
 * (UoCTTI) or 4 (Dalal-Triggs) planes in hog.c's order; each pixel adds weight_k * glyph_k for k ascending in float without
 * FMA and is then clamped to [min(0, weights), max(0, weights)] with hog.c's comparisons, so the image is bit for bit hog.c's
 * (NaN included) for the same features and starting image.  transposed selects the glyphs of a transposed VlHog.  Null
 * pointers, an invalid configuration, or a grid smaller than 1 x 1 or with a negative offset is SD_ERR_INVALID before any work
 * is queued (d_image is not written). */
SD_API int sd_hog_render(sd_ctx* ctx, const sd_hog_grids* grids, int num_bins, int variant, int transposed, float* d_image);
/* sd_hog_relayout: a gather of every grid's planes into d_out, asynchronous on the context's stream, out of place (d_out must
 * not overlap the input).  flip = 1: plane i of the result is plane perm[i] (sd_hog_permutation) with its columns mirrored,
 * out[i][y][x] = in[perm[i]][y][w - 1 - x] -- the features of the left-right mirrored image.  transpose = 1: each (flipped)
 * plane is then stored transposed, [w][h] -- the features of a transposed VlHog.  Validation as sd_hog_render. */
SD_API int sd_hog_relayout(sd_ctx* ctx, const sd_hog_grids* grids, int num_bins, int variant, int flip, int transpose, float* d_out);

/* ---- HOG filters: a bank of templates scored over a batch of HOG grids (the score maps of a sliding-window detector) ---------
 * Filters are [Q][dd][fh][fw], the layout of the features of a grid of fw x fh cells: sd_hog_dense of a template image gives a
 * filter, sd_hog_render draws one and sd_hog_relayout(flip = 1) mirrors one.  For grid g ([dd][h][w] as in sd_hog_grids),
 * filter q and output (y, x):
 *   S = bias[q] + sum_{c < dd} sum_{dy < fh} sum_{dx < fw} F[q][c][dy][dx] * M[c][y + dy - pad_y][x + dx - pad_x]
 * with M = 0 outside the grid, over oh = h + 2 pad_y - fh + 1 rows and ow = w + 2 pad_x - fw + 1 columns, written [Q][oh][ow] at
 * d_scores + out_offset of the grid's descriptor, or at d_scores + i * Q * oh * ow for equally sized grids.  A grid with
 * oh <= 0 or ow <= 0 (smaller than the filter) has no scores and is valid.  Arithmetic: float32 FMAs (no TF32) in one fixed
 * order -- per (channel, dy) ascending, dx ascending, a chain from 0; the bias added last -- so each score depends on its grid,
 * filter and bias alone: the same in any batch and in every run.  Score (x, y) of a pyramid level covers the cells from
 * (x - pad_x, y - pad_y), which start at pixel (x - pad_x) * cell_size * width / level_w of the frame (rows alike).
 * Limits: fw, fh in [1, SD_HOG_FILTER_MAX_SIDE], num_filters in [1, SD_HOG_FILTER_MAX_BANK], pad_x in [0, fw - 1] and pad_y
 * in [0, fh - 1].  Null pointers (d_bias may be NULL: no bias), pointers that are not 4-byte aligned, an invalid configuration,
 * a grid smaller than 1 x 1 or with a negative offset, or anything outside the limits is SD_ERR_INVALID before any work is
 * queued (d_scores is not written). */
#define SD_HOG_FILTER_MAX_SIDE 32
#define SD_HOG_FILTER_MAX_BANK 256
SD_API int sd_hog_correlate(sd_ctx* ctx, const sd_hog_grids* maps, int num_bins, int variant,
                            const float* d_filters, int num_filters, int filter_w, int filter_h,
                            const float* d_bias /* num_filters floats or NULL */, int pad_x, int pad_y, float* d_scores);

/* ---- detections from HOG filter scores: thresholded boxes in frame pixels and greedy non-maximum suppression ----------------
 * One score map of sd_hog_correlate's output: the [Q][height][width] scores of one pyramid level of one frame. */
typedef struct {
    int32_t frame;              /* in [0, num_frames): the frame whose detection list receives the map's detections */
    int32_t level;              /* reported with each detection; not otherwise interpreted */
    int32_t frame_w, frame_h;   /* the frame, px */
    int32_t level_w, level_h;   /* the level, px (sd_hog_pyramid_shape); level_w == frame_w for an unscaled map */
    int32_t width, height;      /* ow x oh score positions (either may be 0: no scores) */
    int64_t offset;             /* floats: the map's scores at d_scores + offset */
} sd_hog_score_map;
typedef struct {
    int32_t x, y, w, h;         /* box in frame pixels, the argument layout of sd_detect_faces_* */
    float score;
    int32_t filter, level;      /* filter index q, the map's level */
    int32_t cell_x, cell_y;     /* score position in the map */
} sd_hog_detection;
/* sd_hog_detections: the detections of every frame of a batch, asynchronous on the context's stream.
 *   Candidates.  Score (x, y) of filter q in a map is a candidate of the map's frame when score > threshold (a NaN score never
 *     is).  d_above[f] (d_above may be NULL) receives frame f's candidate count before any cap.
 *   Box.  Exact integer arithmetic in int64, rh(n, d) = floor((2n + d) / (2d)) (round half up, floor division),
 *     sx = cell_size * frame_w, sy = cell_size * frame_h:
 *       x0 = rh((x - pad_x) * sx, level_w),  x1 = rh((x - pad_x + filter_w) * sx, level_w),  rows alike with sy and level_h;
 *     the box is (x0, y0, x1 - x0, y1 - y0), not clipped to the frame.  This is sd_hog_correlate's mapping of a score to pixels,
 *     (x - pad_x) * cell_size * width / level_w, rounded.
 *   Order.  A frame's candidates by score descending (scores compare as floats: -0 == +0), then in enumeration order: the map's
 *     index in the table, then q, y, x.  The order is total.
 *   Cap.  Only the first max_candidates candidates of a frame, in that order, go on to suppression.
 *   Suppression.  Greedy over the capped list in order: a candidate is kept unless a kept candidate overlaps it with
 *     (double)inter > overlap * (double)union, inter and union int64 pixel areas (torchvision's nms rule on these boxes); a box
 *     of zero area never suppresses and is never suppressed.  overlap = 1 keeps every candidate.  Suppression stops when
 *     max_detections candidates are kept.
 *   Output.  Frame f's kept detections, in order, at d_out + f * max_detections; d_count[f] says how many.  Slots past the count
 *     are not written.
 *   Classes.  All filters of one call form one class (a filter and its mirror, mixture components).  Per-class suppression is one
 *     call per class: a map's offset may point at filter q0's plane, with num_filters that class's filter count.
 * A frame's result depends only on its own maps, in their table order: bit for bit the same in any batch and in every run.  The
 * call reads the map table back once and queues its work; scratch is num_frames x max_candidates 8-byte keys, a small state per
 * frame and three int32 per map.  Null pointers (d_scores and d_maps may be NULL when num_maps = 0), d_scores, d_out or d_count
 * not 4-byte aligned, d_maps or d_above not 8-byte aligned, num_frames < 1, num_maps < 0, a map whose frame is out of range,
 * whose offset is negative, whose frame or level is smaller than 1 x 1, whose size is negative or whose boxes do not fit in int32,
 * more than 2^32 - 1 scores in one frame, overlap outside [0, 1], a NaN threshold, num_filters, cell_size (1..32), filter sides or
 * pads outside sd_hog_correlate's limits, max_candidates outside [1, SD_HOG_DETECT_MAX_CANDIDATES], or max_detections outside
 * [1, max_candidates] is SD_ERR_INVALID before any work is queued (nothing is written).  num_maps = 0 writes zero counts. */
#define SD_HOG_DETECT_MAX_CANDIDATES 8192
SD_API int sd_hog_detections(sd_ctx* ctx, const float* d_scores, const sd_hog_score_map* d_maps, int num_maps,
                             int num_frames, int num_filters, int cell_size, int filter_w, int filter_h, int pad_x, int pad_y,
                             float threshold, double overlap, int max_candidates, int max_detections,
                             sd_hog_detection* d_out /* num_frames x max_detections */, int32_t* d_count /* num_frames */,
                             int64_t* d_above /* num_frames, or NULL */);

/* ---- training HOG filters: window rows, a squared-hinge linear SVM and hard-negative mining ---------------------------------
 * One window of a batch of grids: score position (x, y) of sd_hog_correlate on grid `grid`; flip = 1 reads the window of the
 * left-right mirrored image. */
typedef struct {
    int32_t grid, x, y, flip;
} sd_hog_window;
/* sd_hog_windows: the feature row of every window, asynchronous on the context's stream.  With D = dd * fh * fw + 1, row r holds
 * what score (x, y) of sd_hog_correlate reads, in the filter layout:
 *   rows[r * ldr + (c * fh + dy) * fw + dx] = M[c][y + dy - pad_y][x + dx - pad_x]      (M = 0 outside the grid)
 * and rows[r * ldr + D - 1] = 1.0, the bias column of the centred learn path; columns D .. ldr - 1 are not written.  A flipped
 * window is sd_hog_relayout(flip = 1) of the fh x fw block it reads: plane perm[c] (sd_hog_permutation), columns mirrored.  A
 * pure gather: row . [F | b] in float64 is sd_hog_correlate's score of [F | b] within that call's float32 rounding.  The call
 * reads the grid table (if any) and the window table back once.  Null or unaligned pointers (4 bytes), an invalid configuration,
 * filter sides or pads outside sd_hog_correlate's limits, ldr < D, a window whose grid is out of range, whose (x, y) is not a
 * score position of its grid, or whose flip is not 0 or 1 is SD_ERR_INVALID before any work is queued (d_rows is not written). */
SD_API int sd_hog_windows(sd_ctx* ctx, const sd_hog_grids* maps, int num_bins, int variant, int filter_w, int filter_h, int pad_x,
                          int pad_y, const sd_hog_window* d_windows, int count, float* d_rows, int64_t ldr);
/* sd_hog_box_windows: host only.  For each ground-truth box (boxes[4 b ..] = x, y, w, h in pixels of a frame_w x frame_h frame)
 * the window that covers it best over the frame's pyramid at the given scales: the candidates are every score position of every
 * non-empty level (sd_hog_pyramid_shape), each with the exact integer box sd_hog_detections reports for it; the best has the
 * largest IoU over int64 areas, compared exactly as rationals, ties to the lower level, then y, then x.  out[b] = (level, x, y,
 * 0) and iou[b] = its IoU as a double; a box whose best window fails (double) inter >= positive_overlap * (double) union gets
 * grid = -1.  SD_ERR_INVALID for null pointers, a frame smaller than 1 x 1, an invalid scale or configuration, filter sides or
 * pads outside sd_hog_correlate's limits, positive_overlap outside [0, 1], or a box with w or h < 1. */
SD_API int sd_hog_box_windows(int frame_w, int frame_h, const double* scales, int num_scales, int cell_size, int num_bins,
                              int variant, int filter_w, int filter_h, int pad_x, int pad_y, double positive_overlap,
                              const int32_t* boxes, int num_boxes, sd_hog_window* out, double* iou);
/* sd_learn_squared_hinge: the linear SVM with squared hinge loss,
 *   minimise f(w) = lambda / 2 * sum_{j < D-1} w_j^2 + 1/2 * sum_i max(0, 1 - y_i a_i . w)^2,
 * rows a_i of A (N x D, the last column the all-ones bias, which is not regularised), labels y_i = +1 or -1.  The primal finite
 * Newton method (Keerthi & DeCoste 2005): from w = 0 (every row active), each step solves the ridge system on the active rows
 * S = {i : y_i a_i . w < 1}, (lambda I' + A_S^T A_S) w = A_S^T y_S, with sd_learn_centred (Manual lambda, bias unregularised) on
 * rows shifted by one column mean fixed for the whole solve (sd_centre_features on the first step's rows, which are all of them).
 * The margins of the Newton point are computed in float64 on the device; if its active set is S it is the optimum, otherwise an
 * exact line search on the host (phi(t) = f(w + t d) is a convex piecewise quadratic, minimised in float64 over its sorted
 * breakpoints) gives the next point.  It stops when the active set after a step equals the set the step was solved on
 * (SD_SVM_CONVERGED), when f does not decrease (SD_SVM_NO_DECREASE: the last point that decreased f is kept), or after
 * max_iterations steps.  The context's solver and Gram settings apply as for sd_learn_centred.  d_A is not modified; the scratch
 * is N x roundup4(D + 1) floats of compacted rows and N doubles of margins, plus the learn path's own workspace.  Each step reads
 * back the N margins and synchronises.  The result is the same in every run.  Null or unaligned (4 bytes) pointers, a label
 * other than +1 or -1, lambda <= 0 or not finite, N < 1, D < 2, lda < D or max_iterations < 1 is SD_ERR_INVALID before any work
 * is queued (d_w is not written). */
#define SD_SVM_CONVERGED 0
#define SD_SVM_NO_DECREASE 1
#define SD_SVM_ITERATION_CAP 2
typedef struct {
    int32_t iterations;          /* Newton steps taken */
    int32_t active;              /* |S| at the returned w */
    int32_t stop;                /* SD_SVM_* */
    int32_t reserved;
    double objective;            /* f at the returned w, float64 */
} sd_svm_report;
SD_API int sd_learn_squared_hinge(sd_ctx* ctx, const float* d_A, int64_t lda, const float* d_y, int N, int D, float lambda,
                                  int max_iterations, float* d_w /* D */, sd_svm_report* report /* may be NULL */);
/* sd_hog_train_filter: a HOG filter for the sliding-window detector (sd_hog_pyramid + sd_hog_correlate + sd_hog_detections),
 * trained by a squared-hinge SVM with hard-negative mining.  The rule:
 *   Positives.  Each box is assigned its window by sd_hog_box_windows with positive_overlap = (double) p->positive_overlap (the
 *     float widened, so a threshold such as 0.7 is the float nearest to it); with flip_positives each assigned box
 *     also adds its mirrored window.  Rows are in box order, each unflipped row followed by its mirror.  Unassigned boxes are
 *     counted and skipped.  The positive set is fixed across rounds.
 *   Round 0.  The filter is the mean of the unflipped positive rows (feature columns, float64 sums rounded to float) minus its
 *     own scalar mean (float64, rounded to float), bias 0.  Each frame gives its detections under this filter: sd_hog_detections
 *     over all its levels with threshold -FLT_MAX, max_candidates SD_HOG_DETECT_MAX_CANDIDATES, overlap mine_overlap and
 *     max_detections negatives_per_frame; a window whose box overlaps a box of its frame with (double) inter > negative_overlap *
 *     (double) union is excluded.  Then the first solve runs.
 *   Rounds 1 .. rounds.  The same mining with the current filter and bias at threshold -1 (the windows that violate the margin).
 *   Cache.  Windows already cached, by (frame, level, x, y), are not new.  New windows take the next empty slot of the cache;
 *     when it is full, the slots of cached negatives that are inactive under the round's filter (margin >= 1), in slot order;
 *     when those are used up, the round's remaining new windows are truncated.  New windows come in frame order and, within a
 *     frame, in the detection order.  A round after round 0 that adds no window ends the training, and its solve is skipped.
 *   Solve.  sd_learn_squared_hinge (lambda, max_iterations) on the positive rows (+1) followed by the cache in slot order (-1).
 *   Frames without boxes are pure negative frames.  The pyramids are computed a slice of frames at a time (about 256 MB of
 *   features each) and each slice is mined and gathered while it is resident; the scratch does not grow with the number of
 *   frames, apart from per-frame and per-box tables and the (positives + max_negatives) x D rows.  The result depends only on the
 *   frames, boxes and parameters, bit for bit the same in every run.
 * Output: d_filter (device, dd * fh * fw floats, the [dd][fh][fw] layout of sd_hog_correlate), *h_bias, one report per round in
 * h_rounds[0 .. rounds] (entries after an early stop are zero), the cache in slot order in h_negatives (max_negatives entries, or
 * NULL; grid = frame * num_scales + level, flip 0) and its size in *h_num_negatives.  The frames are an sd_image_batch as for
 * sd_hog_pyramid (no d_roi).  Null pointers, an invalid configuration, scale, filter side or pad, a box whose frame is out of
 * range or whose w or h < 1, lambda <= 0, overlaps outside [0, 1], flip_positives outside {0, 1}, rounds < 0, negatives_per_frame
 * outside [1, SD_HOG_DETECT_MAX_CANDIDATES], max_negatives < 1, max_iterations < 1, D above SD_HOG_TRAIN_MAX_DIM or no assigned
 * box is SD_ERR_INVALID, and rows, Gram and one slice that would not fit in device memory SD_ERR_CUDA, before any work is
 * queued. */
#define SD_HOG_TRAIN_MAX_DIM 8192   /* D = dd * fh * fw + 1: 31 x 16 x 16 + 1 = 7937 fits; the Gram is 256 MB at the cap */
typedef struct {
    int32_t frame, x, y, w, h;
} sd_hog_box;
typedef struct {
    float lambda;                 /* on the filter, not the bias */
    float positive_overlap;       /* e.g. 0.5: minimum IoU of a box's window (sd_hog_box_windows) */
    float negative_overlap;       /* e.g. 0.3: a mined window overlapping a box of its frame by more is not a negative */
    int32_t flip_positives;       /* 1: every positive also as its mirrored window */
    int32_t rounds;               /* mining rounds after round 0 */
    int32_t negatives_per_frame;  /* per frame and round (sd_hog_detections' max_detections) */
    float mine_overlap;           /* suppression among one frame's mined windows; 1 = none */
    int32_t max_negatives;        /* rows of the negative cache */
    int32_t max_iterations;       /* Newton iterations per solve */
} sd_hog_train_param;
typedef struct {
    int32_t positives;            /* positive rows (mirrors included) */
    int32_t unassigned;           /* boxes no window covers at positive_overlap */
    int32_t cache;                /* cached negatives after the round's mining */
    int32_t mined;                /* windows the round's detections gave, after the box exclusion */
    int32_t excluded;             /* windows excluded for overlapping a box */
    int32_t added;                /* new windows that entered the cache */
    int32_t evicted;              /* inactive cached negatives whose slots new windows took */
    int32_t truncated;            /* new windows dropped because the cache was full */
    int32_t solved;               /* 1: the round's solve ran */
    int32_t reserved;
    sd_svm_report solve;
    /* the round's phases: CUDA events around the pyramids, the scores, the detections and the window gathers (kernel only; its
     * tables are uploaded before), the host clock around the host filtering (the detections' download and the box exclusion)
     * and around the solve (which ends synchronised); round 0 includes the pass that gathers the positives */
    float pyramid_ms, scores_ms, detect_ms, host_ms, gather_ms, solve_ms;
    double gathered_bytes;        /* rows read and written by the round's gathers: 2 x rows x D x 4 */
} sd_hog_train_report;
SD_API int sd_hog_train_filter(sd_ctx* ctx, const sd_image_batch* images, const sd_hog_box* h_boxes, int num_boxes,
                               const double* h_scales, int num_scales, int cell_size, int num_bins, int variant, int filter_w,
                               int filter_h, int pad_x, int pad_y, const sd_hog_train_param* p, float* d_filter, float* h_bias,
                               sd_hog_train_report* h_rounds, sd_hog_window* h_negatives, int* h_num_negatives);

/* ---- regressor: LinearRegressor<Solver> (regressors.hpp:318-400) ------------------------ */
/* Solver::solve (regressors.hpp:199-234 == verbose_solver.hpp:53-111):
 *   X = (A^T A + Lambda)^-1 A^T B ;  A: N x D, B: N x M, X: D x M (ldx_out = M).
 * lambda_out (host, may be NULL) receives the lambda actually applied (regressors.hpp:126-148).
 * n_train_global: the N used in the MatrixNorm rule (== N on one GPU; the global sample count
 * when the Gram was summed over ranks).  Phase timings (ms) of the last call, named as the
 * reference's VerbosePartialPivLUSolver prints them, are available from sd_solver_timings. */
SD_API int sd_learn(sd_ctx* ctx, const float* d_A, int64_t lda, const float* d_B, int64_t ldb,
                    int N, int D, int M, const sd_regulariser* reg, float* d_X, float* lambda_out);
/* The training path on CENTRED feature rows (what the shells' and the Python mirror's train() use for D > 256).
 * HOG features are non-negative, so A^T A is dominated by n mu mu^T and the covariance that decides the weights sits several
 * digits down; a float32 Gram matrix -- the reference's as much as this one -- then loses three digits of the weights (the
 * reference's own arithmetic is 2e-3 away from the float64 solution on RCR features).  Subtracting the column means before the
 * Gram is the same least-squares problem (A w + c 1 = (A - 1 mu^T) w + (c + mu.w) 1) without that loss:
 *   sd_centre_features : d_mu[c] = mean of column c over ALL ranks' rows (0 for the last = bias column); d_A[:, c] -= d_mu[c]
 *                        in place.  The shift is only the same problem when the last column is exactly all ones and is not
 *                        regularised (regressors.hpp:143-146): otherwise -- and for D <= 256 (reference-order LU) -- the rows are
 *                        left untouched and d_mu = 0, with which sd_learn_centred is sd_learn / sd_learn_dist.
 *   sd_learn_centred   : Gram of the centred rows, exchange (comm may be NULL; route as in sd_learn_dist), lambda from the norm
 *                        of the UNcentred A^T A (regressors.hpp:135: reconstructed from the centred Gram and mu), solve.
 *                        d_X  : D x M weights for uncentred features -- the model (bias shifted back: c' - mu.w);
 *                        d_Xc : (optional) the weights that go with the centred buffer, for sd_cascade_update on it. */
SD_API int sd_centre_features(sd_ctx* ctx, sd_comm* comm, float* d_A, int64_t lda, int N_local, int D, int n_global,
                              const sd_regulariser* reg, float* d_mu);
SD_API int sd_learn_centred(sd_ctx* ctx, sd_comm* comm, const float* d_Ac, int64_t lda, const float* d_B, int64_t ldb,
                            int N_local, int D, int M, const sd_regulariser* reg, int n_train_global, int route,
                            const float* d_mu, float* d_X, float* d_Xc, float* lambda_out);

/* ColPivHouseholderQRSolver::solve (regressors.hpp:264-305): the same system, plus the one diagnostic that solver exists for --
 * the numerical rank of the regularised A^T A (regressors.hpp:288-293 prints it and asks for a larger lambda).  A^T A + Lambda is
 * symmetric positive semi-definite, so the rank comes from a diagonally pivoted Cholesky (threshold eps * D relative to the
 * largest pivot, Eigen's default rule) at any D.  It factors a copy of the D x D matrix in its own workspace: 1.16 GB at
 * D = 17,051 and 11.1 GB at D = 52,701, where a one-GPU train then holds about 44 GB (features 21 + Gram 11 + copy 11).  Like
 * the reference the call goes on to solve when the matrix is rank deficient; if the solve itself then breaks down the status is
 * SD_ERR_NUMERIC and sd_last_error carries the reference's message with the rank. */
SD_API int sd_learn_rank_revealing(sd_ctx* ctx, const float* d_A, int64_t lda, const float* d_B, int64_t ldb,
                                   int N, int D, int M, const sd_regulariser* reg, float* d_X, float* lambda_out, int* rank_out);
/* The same, split at the multi-GPU exchange point (superviseddescent.hpp:207 / SURVEY 8e):
 *   1. sd_gram      : d_G[Dx(D+M)] = [A^T A | A^T B] of the local rows (upper triangle of the
 *                     D x D part is valid; row stride ldg >= D+M)
 *   2. (caller)     : allreduce d_G over ranks
 *   3. sd_solve_gram: regularise with n_train_global and solve, replicated on every rank */
SD_API int sd_gram(sd_ctx* ctx, const float* d_A, int64_t lda, const float* d_B, int64_t ldb,
                   int N, int D, int M, float* d_G, int64_t ldg);
SD_API int sd_solve_gram(sd_ctx* ctx, float* d_G, int64_t ldg, int D, int M,
                         const sd_regulariser* reg, int n_train_global, float* d_X, float* lambda_out);
/* LinearRegressor::predict (regressors.hpp:377-381): out[N x M] = values[N x D] * X[D x M] */
SD_API int sd_predict(sd_ctx* ctx, const float* d_values, int64_t ldv, int N, int D,
                      const float* d_X, int M, float* d_out, int64_t ldo);
/* LinearRegressor::test (regressors.hpp:361-369): ||values X - labels||_2 / ||labels||_2 */
SD_API int sd_test_residual(sd_ctx* ctx, const float* d_values, int64_t ldv, const float* d_labels,
                            int64_t ldl, int N, int D, const float* d_X, int M, double* residual_out);
/* timings of the last sd_learn / sd_solve_gram: [0] "At * A", [1] "AtA + Reg", [2] "Decomposition",
 * [3] "solve()" in milliseconds (verbose_solver.hpp:66-103) */
SD_API int sd_solver_timings(sd_ctx* ctx, float ms_out[4]);
/* precision of the Gram and of the Cholesky trailing updates (both run the same SYRK kernels):
 * 0 = 3xTF32 split on the truncated operand (default: Gram ~2e-7),
 * 3 = 3xTF32 split with the hi part rounded in shared memory (unbiased: Gram ~7e-8, ~15 % slower),
 * 1 = single TF32 pass (~7e-5), also for the trailing updates, 2 = force the fp32 SIMT kernel (~3e-7) everywhere.
 * The trailing updates always round the hi part; the product inside conjugate gradients is always 3xTF32 with rounded hi. */
SD_API int sd_set_gram_mode(sd_ctx* ctx, int mode);

/* ---- multi-GPU training: the exchange at superviseddescent.hpp:207 (SURVEY 8e) ----------------------------------------
 * One process per GPU, samples (rows of A) sharded over the ranks.  [A^T A | A^T b] is a sum over the shards, so per cascade
 * level there is ONE collective on it; lambda uses the global sample count.  The collectives are NCCL (bound at run time:
 * libnccl.so.2 must be loadable when nranks > 1).  Three routes:
 *   replicated : sd_gram -> sd_allreduce_gram -> sd_solve_gram on every rank (small systems; the solve does not scale)
 *   shared CG  : sd_gram -> sd_allreduce_gram -> conjugate gradients whose product S P is split over the ranks by slabs of the
 *                contraction, one all-reduce of 2L x D floats per iteration (sd_learn_dist / sd_learn_centred with
 *                distributed_solve = 2); falls back to the replicated factorisation when CG does not converge
 *   distributed: sd_gram -> sd_reduce_scatter_gram -> sd_solve_gram_dist: the 256-row panels of [AtA|Atb] are owned
 *                block-row-cyclically (panel p by rank p % nranks); the owner factors its panel, broadcasts it, every rank
 *                updates the block rows it owns (blocked right-looking Cholesky, same kernels as on one GPU); every rank
 *                ends with the same X.  sd_learn_dist runs any of the routes from the local rows.
 * Determinism: for a fixed nranks the result is reproducible bit for bit; it differs from the one-GPU result only by the
 * summation order of the partial Gram matrices (~1e-7 relative). */
#define SD_COMM_ID_BYTES 128
/* rank 0 obtains an id and hands it to the other ranks by any means the host has (MPI, torch.distributed, a file) */
SD_API int sd_comm_get_unique_id(uint8_t* id_out /* SD_COMM_ID_BYTES */);
SD_API int sd_comm_create(sd_ctx* ctx, const uint8_t* id, int rank, int nranks, sd_comm** out);   /* collective */
/* adopt a ncclComm_t the host already owns (it is not destroyed by sd_comm_destroy) */
SD_API int sd_comm_adopt(sd_ctx* ctx, void* nccl_comm, int rank, int nranks, sd_comm** out);
SD_API void sd_comm_destroy(sd_comm* comm);
SD_API int sd_comm_rank(const sd_comm* comm);
SD_API int sd_comm_size(const sd_comm* comm);
/* sum of one host integer over the ranks (the N of the MatrixNorm rule, regressors.hpp:135) */
SD_API int sd_comm_sum_int64(sd_ctx* ctx, sd_comm* comm, int64_t* h_value);
/* d_recv[r * bytes_per_rank ..] = rank r's d_send (current landmarks for a training callback, superviseddescent.hpp:217) */
SD_API int sd_comm_allgather(sd_ctx* ctx, sd_comm* comm, const void* d_send, size_t bytes_per_rank, void* d_recv);
/* in place on d_G (D x ldg, as written by sd_gram): sums over the ranks the part the solve reads -- every 256-row band from
 * its diagonal column to the end of its rows (the upper triangle and the right-hand sides; about half of the buffer) */
SD_API int sd_allreduce_gram(sd_ctx* ctx, sd_comm* comm, float* d_G, int64_t ldg, int D, int M);
/* the same sums, but band p is only delivered to rank p % nranks (what sd_solve_gram_dist expects) */
SD_API int sd_reduce_scatter_gram(sd_ctx* ctx, sd_comm* comm, float* d_G, int64_t ldg, int D, int M);
/* sd_solve_gram on a reduce-scattered d_G; collective, every rank receives X (and the same lambda) */
SD_API int sd_solve_gram_dist(sd_ctx* ctx, sd_comm* comm, float* d_G, int64_t ldg, int D, int M,
                              const sd_regulariser* reg, int n_train_global, float* d_X, float* lambda_out);
/* LinearRegressor::learn on sharded rows: local Gram, exchange, solve.  distributed_solve: 0 = all-reduce, every rank solves
 * alone; 1 = reduce to the panel owners + distributed factorisation; 2 = all-reduce + conjugate gradients shared by the ranks
 * (see sd_set_solver).  N_local may be 0. */
SD_API int sd_learn_dist(sd_ctx* ctx, sd_comm* comm, const float* d_A, int64_t lda, const float* d_B, int64_t ldb,
                         int N_local, int D, int M, const sd_regulariser* reg, int n_train_global, int distributed_solve,
                         float* d_X, float* lambda_out);

/* Solver of the systems with D > 256 (smaller ones always take the reference-order partial-pivot LU):
 *   0 = blocked Cholesky (default): the direct solve that stands in for Eigen::PartialPivLU (regressors.hpp:224-225);
 *   1 = conjugate gradients on the tensor cores: after the bias column has been eliminated the regularised Gram matrix of the
 *       centred features is very well conditioned under the MatrixNorm rule (condition number ~ N / 350 for RCR features), so a
 *       few dozen products with the D x D matrix replace the D^3 / 3 factorisation; it stops at a relative residual of 2e-6 and
 *       falls back to the Cholesky if the recurrence breaks down or stalls (ill-conditioned systems, tiny lambda).
 * sd_learn_dist: distributed_solve 2 = the ranks share the CG iterations (rows of the matrix sharded, one all-reduce of
 * 2L x D floats per iteration).  sd_solver_iterations, of the last solve: +n = CG converged after n iterations and its answer
 * was used; -n = CG ran n iterations, gave up, and the factorisation answered; 0 = CG was not tried. */
SD_API int sd_set_solver(sd_ctx* ctx, int mode);
SD_API int sd_solver_iterations(const sd_ctx* ctx);

/* The rank diagnostic of sd_learn_rank_revealing for every solve: with on != 0, sd_learn, sd_learn_centred, sd_solve_gram and
 * sd_learn_dist (routes 0 and 2) also compute the numerical rank of the regularised system (what the optimisers' train() needs
 * for ColPivHouseholderQRSolver levels).  sd_last_rank, of the last solve: the rank, or -1 when it was not computed.  With
 * centred features the matrix factored is the centred Gram + Lambda; it is congruent to the uncentred one (T^T (A^T A + Lambda) T
 * with a unit-triangular T, and T^T Lambda T = Lambda because the bias is not regularised), so its exact rank is the same, and
 * the relative cut is applied to the better-conditioned matrix.  Route 1 (distributed factorisation) holds no rank's whole
 * matrix: -1 there. */
SD_API int sd_set_rank_diagnostic(sd_ctx* ctx, int on);
SD_API int sd_last_rank(const sd_ctx* ctx);

/* ---- cascade steps: SupervisedDescentOptimiser (superviseddescent.hpp:165-344) ---------- */
/* b_i = (x_i - x_gt_i) (.) norm(x_i)     (superviseddescent.hpp:199-205) */
SD_API int sd_cascade_targets(sd_ctx* ctx, const float* d_x, const float* d_x_gt, int N, int P,
                              const sd_normalisation* norm, float* d_B, int64_t ldb);
/* x_next_i = x_i - (A_i X) (.) (1 / norm(x_i))   (superviseddescent.hpp:209-215, 296-301, 336-339)
 * d_x_next must not alias d_x. */
SD_API int sd_cascade_update(sd_ctx* ctx, const float* d_A, int64_t lda, int N, int D,
                             const float* d_X, int P, const float* d_x, const sd_normalisation* norm,
                             float* d_x_next);
/* observed = features - templates (superviseddescent.hpp:191-197), in place on A */
SD_API int sd_subtract_templates(sd_ctx* ctx, float* d_A, int64_t lda, const float* d_T, int64_t ldt,
                                 int N, int D);

/* ---- cascade levels: one HogTransform cascade level per call, in chunks of rows ---------------------------------------------
 * A level's feature rows [A | b] (ld = roundup4(D + 2L) floats per sample: 68 KB at D = 17,051, 211 KB at D = 52,701) need not
 * be resident at once: [A^T A | A^T b] is a sum over rows.  The caller owns one buffer of chunk_rows x ld floats; the level runs
 * through it chunk by chunk.
 *
 * Where a level's frames are (sd_level_frames): exactly one of images and host_frames is non-NULL, anything else is SD_ERR_INVALID
 * before any work is queued.
 *   - images: frames resident on the device, as for sd_hog_batch.
 *   - host_frames: num_host_frames host frames (sd_host_frame: grey or B,G,R, any sizes), each in pinned, device-mapped memory with
 *     a 16-byte aligned base and row_stride (the ROI route of sd_detect_faces_host), and row_stride >= channels * (width rounded up
 *     to 16).  Only frames a sample refers to are read or checked; they are read in place while the call runs.  Per chunk of rows
 *     the HOG rows are produced in gather batches that fit one half of the context's staging pair: the exact union of the windows
 *     of the batch's patches is planned per frame on the device (samples of one frame in one batch share one region), gathered
 *     zero-copy over PCIe (colour converted to grey on the way) on the context's copy stream while the previous batch's HOG runs,
 *     and read by the unchanged HOG kernel.  One small read-back per batch is the only synchronisation the plan adds, and the call
 *     reads d_sample_frame back once before it queues work.  Each half holds max(stage_half_bytes, the largest referenced frame's
 *     grey bytes at a 16-byte pitch) rounded up to 16; the context keeps the pair (it is the pair sd_detect_faces_host uses) and
 *     grows it when a call needs more.  X, lambda and x_next are bit for bit what the same frames uploaded by sd_upload_frames give.
 *     Frames that break these rules are SD_ERR_INVALID before any work is queued.  Every rank passes its own frames.
 *   - d_sample_frame (device, N ints, may be NULL = frame i): sample i reads frame d_sample_frame[i].  An index out of range raises
 *     the projection's status flag (reported by the next synchronising call, as for sd_hog_batch); on the host route the sample
 *     then reads frame 0. */
typedef struct {
    const sd_image_batch* images;      /* frames resident on the device, or NULL */
    const sd_host_frame* host_frames;  /* frames in pinned host memory, or NULL */
    int32_t num_host_frames;
    const int32_t* d_sample_frame;     /* sample i reads frame d_sample_frame[i]; NULL = frame i, on either route */
    size_t stage_half_bytes;           /* host route: bytes per staging half; 0 = the library's default (48 MB) */
} sd_level_frames;
/* sd_level_chunk_rows: the largest r <= N_local such that r rows of the caller's chunk buffer (r * ld * 4 bytes, with the update's
 * r * M * 8 bytes of partial sums) fit in free_bytes beside everything the level will still allocate with the context's current
 * settings -- G (D x ld), the rank copy if the diagnostic is on, CG's copy of the system if CG may run (sd_set_solver 1, or route 2
 * on several ranks), the band buffer of the exchange on several ranks, the bias / inverse workspaces and, for host frames, the
 * staging pair (sized by the largest frame of the table) -- less what the context already holds, and a reserve of 512 MB for small
 * workspaces.  frames may be NULL (no staging).  free_bytes == 0: cudaMemGetInfo.  Returns N_local (at least 1) when everything
 * fits; SD_ERR_CUDA, with a message naming D, when not even min(N_local, 256) rows fit.  M = the parameter width P (2L for HOG
 * levels).  It serves the projected levels below unchanged: D = feature_length, M = P, frames = NULL.
 *
 * sd_train_level: one training level (superviseddescent.hpp:173-217) for the HOG projection (frames as above, hog_eyes as in
 * sd_hog_batch).  d_x, d_x_gt: N_local x 2L current / ground-truth landmarks; norm: the optimiser's normalisation; d_templates:
 * optional N_local x D (row pitch ldt); reg / route / comm as in sd_learn_centred (comm may be NULL); n_global: the samples of all
 * ranks.  Writes the model d_X (D x 2L, for uncentred features), the updated landmarks d_x_next (N_local x 2L) and *lambda_out (may
 * be NULL).
 *   - one chunk (chunk_rows >= N_local): sd_hog_batch, sd_subtract_templates, sd_cascade_targets, sd_centre_features,
 *     sd_learn_centred and sd_cascade_update (on the centred rows with their weights) -- bit for bit what those calls give.
 *   - several chunks: chunk 0 is centred by sd_centre_features over every rank's first chunk; its column means p (the pilot
 *     shift) are subtracted from every later chunk too, and every chunk's [A - 1 p^T | b] is added onto one Gram.  The solve is
 *     exact for any shift (DESIGN 4.3); p only has to be close enough to the mean to avoid the float32 cancellation.  The update
 *     projects and shifts every chunk but the last (still resident) again.
 *   The rank diagnostic (sd_set_rank_diagnostic), solver, gram mode and sd_solver_timings keep their meaning; with several chunks
 *   "At * A" spans the whole accumulation, the projection of the later chunks included.  For a fixed chunk_rows and rank count
 *   the result is reproducible bit for bit.  Every rank makes the same collectives whatever its chunk count.
 *   SD_ERR_INVALID before any work is queued (outputs unwritten): chunk_rows < 1, ld < D + 2L, templates with
 *   chunk_rows < N_local (a chunked level would check the all-ones bias column on chunk 0 only, and T is as large as the
 *   features), d_x_next == d_x, null pointers, bad frames.
 *
 * sd_apply_level: one test / predict level (superviseddescent.hpp:262-306, 323-344) in chunks of chunk_rows rows (ld >= D):
 * HOG rows, optional templates (N x D, pitch ldt), x_next = x - (A X) (.) 1 / norm(x).  With ld a multiple of 4 and a 16-byte
 * aligned d_chunk each row's result does not depend on the chunking.  Same argument errors as sd_train_level, with ld >= D. */
SD_API int sd_level_chunk_rows(sd_ctx* ctx, sd_comm* comm, const sd_level_frames* frames, int64_t N_local, int D, int M, int route,
                               size_t free_bytes, int* rows_out);
SD_API int sd_train_level(sd_ctx* ctx, sd_comm* comm, const sd_level_frames* frames,
                          const float* d_x, const float* d_x_gt, int N_local, int L, int64_t n_global,
                          const sd_normalisation* hog_eyes, const sd_hog_param* p, const sd_normalisation* norm,
                          const float* d_templates, int64_t ldt, const sd_regulariser* reg, int route,
                          float* d_chunk, int64_t ld, int chunk_rows, float* d_X, float* d_x_next, float* lambda_out);
SD_API int sd_apply_level(sd_ctx* ctx, const sd_level_frames* frames, const float* d_x, int N, int L,
                          const sd_normalisation* hog_eyes, const sd_hog_param* p, const sd_normalisation* norm,
                          const float* d_templates, int64_t ldt, const float* d_X,
                          float* d_chunk, int64_t ld, int chunk_rows, float* d_x_next);

/* ---- cascade levels on the caller's projection ------------------------------------------------------------------------------
 * The reference's ProjectionFunction is any h(x_row, level, index) (examples/simple_function.cpp, pose_estimation.cpp).  A
 * projection that can run on the device hands the level its feature rows through a callback; everything after the rows --
 * templates, targets, the pilot shift, the Gram in chunks, the exchange, the solve and the update -- is the loop of sd_train_level /
 * sd_apply_level, with the same rules:
 *   - targets go in columns [D, D + P) of the chunk buffer (ld >= D + P in training, ld >= D in apply);
 *   - centring and the pilot shift apply only when D > 256, the last column is exactly ones and the bias is not regularised;
 *   - templates need one chunk; route and comm as in sd_train_level, and every rank makes the same collectives (on several ranks
 *     two more than sd_train_level: the failure agreement below);
 *   - for a fixed chunk_rows and rank count the result is reproducible bit for bit (given a deterministic callback).
 * P is any parameter width (6 for the pose example).  norm->kind == 1 (inter-eye distance) needs an even P and eye indices below
 * P / 2.
 *
 * The callback writes the features of parameter rows [first_row, first_row + rows) of this rank into columns [0, feature_length)
 * of d_out (row pitch ld floats); d_x points at row first_row (pitch ldx floats).  It returns 0, or non-zero to fail the level.
 *   - Its work must be ordered on sd_ctx_stream(ctx): it enqueues there, or synchronises its own stream before it returns.
 *   - It must not write outside columns [0, feature_length) of its `rows` rows of d_out.
 *   - It may call sd_hog_batch, sd_bgr2gray and the memcpy / memset entry points on ctx.  It must not call any learn, solve, level
 *     or detect entry point on ctx: those share the level's workspaces.
 *   - In training it is called twice for every chunk but the last (once for the Gram, once for the update), so it must be
 *     deterministic.  It is never called with rows == 0.
 *   - Its own device memory is not counted by sd_level_chunk_rows, which leaves it only the 512 MB reserve: a callback that
 *     needs scratch per row should pass free_bytes less that scratch to the query, or choose chunk_rows itself.
 * Errors: a non-zero return fails the level with SD_ERR_INVALID and the message "projection callback returned N".  On several
 * ranks a callback that fails on one rank fails the level on every rank (the others report "the projection callback failed on
 * another rank"): the failing rank still takes part in the collectives up to the exchange, and the ranks agree on failures
 * before the exchange and at the end of the level (one host integer each).  Any other error on one rank is, as for
 * sd_train_level, not agreed on: the other ranks may wait in a collective.  A NULL fn,
 * feature_length < 1, P < 1, a normalisation P cannot carry, ld below the rule above, and the argument errors of sd_train_level /
 * sd_apply_level are SD_ERR_INVALID before any work is queued (outputs unwritten, the callback not called). */
typedef int (*sd_project_fn)(void* user, sd_ctx* ctx, int level, const float* d_x, int64_t ldx, int64_t first_row, int rows,
                             float* d_out, int64_t ld);
typedef struct {
    sd_project_fn fn;
    void* user;                  /* passed to fn unchanged */
    int32_t level;               /* passed to fn: the reference's regressorLevel */
    int32_t feature_length;      /* D */
} sd_level_projection;
SD_API int sd_train_level_projected(sd_ctx* ctx, sd_comm* comm, const sd_level_projection* proj,
                                    const float* d_x, const float* d_x_gt, int N_local, int P, int64_t n_global,
                                    const sd_normalisation* norm, const float* d_templates, int64_t ldt,
                                    const sd_regulariser* reg, int route, float* d_chunk, int64_t ld, int chunk_rows,
                                    float* d_X, float* d_x_next, float* lambda_out);
SD_API int sd_apply_level_projected(sd_ctx* ctx, const sd_level_projection* proj, const float* d_x, int N, int P,
                                    const sd_normalisation* norm, const float* d_templates, int64_t ldt, const float* d_X,
                                    float* d_chunk, int64_t ld, int chunk_rows, float* d_x_next);

/* ---- cascade levels on the caller's host projection -------------------------------------------------------------------------
 * The reference's own projections (examples/simple_function.cpp, pose_estimation.cpp, the hello-world HogTransform) and CPU
 * descriptors run on the host.  Such a projection hands the level its feature rows through a host callback; the library copies
 * them up in a pipeline and everything after the rows is the loop of sd_train_level_projected / sd_apply_level_projected, with
 * the same rules (targets in [D, D + P), the pilot shift, templates in one chunk, the exchange and the failure agreement on
 * several ranks, the rank diagnostic, reproducibility for a fixed chunk_rows and rank count).
 *
 * Inputs of the callback:
 *   - h_x points at row first_row of a pinned host copy of this rank's d_x (pitch ldx = P floats).  The library makes that copy
 *     once per level call, before the first callback; the callback must not write it.
 *   - it writes columns [0, feature_length) of `rows` rows into h_out, a pinned staging half (pitch ld_out = roundup4(D) floats),
 *     and returns 0, or non-zero to fail the level.
 * Batches: within a chunk the callback is called in ascending row order, each call for min(rows left in the chunk, rows that fit
 * one staging half) rows and never for 0 rows.  A half holds stage_half_bytes (0 = 48 MB), at least one row.
 * The pipeline: each filled half goes up on the context's copy stream (one 2-D copy of columns [0, D) into the chunk buffer at the
 * batch's row offset) while the callback fills the other half; the host waits on a half's copy before it refills it.  The first
 * copy of a chunk waits for the previous chunk's last reader on the context's stream, and the stream waits for the chunk's last
 * copy before templates, targets, centring and the Gram.  So the host fills chunk k + 1 while the GPU works on chunk k.  The
 * context keeps the pinned staging pair and the pinned copy of x (grow-only, freed by sd_ctx_destroy); sd_level_chunk_rows is
 * unchanged (frames = NULL): the staging is host memory.
 * The contract:
 *   - in training the callback is called twice for every chunk but the last, so it must be deterministic;
 *   - it runs on the calling thread, and must not call into ctx;
 *   - when it writes the rows a device callback (sd_level_projection) writes, X, lambda and x_next are bit for bit those of
 *     sd_train_level_projected / sd_apply_level_projected for the same chunk_rows, whatever the staging-half size.
 * Errors: a non-zero return fails the level with SD_ERR_INVALID and the message "projection callback returned N"; on several
 * ranks the failure is agreed on as for sd_level_projection.  A NULL fn, feature_length < 1 and the argument errors of
 * sd_train_level_projected / sd_apply_level_projected are SD_ERR_INVALID before any work is queued (outputs unwritten, the
 * callback not called). */
typedef int (*sd_host_project_fn)(void* user, int level, const float* h_x, int64_t ldx, int64_t first_row, int rows,
                                  float* h_out, int64_t ld_out);
typedef struct {
    sd_host_project_fn fn;
    void* user;                  /* passed to fn unchanged */
    int32_t level;               /* passed to fn: the reference's regressorLevel */
    int32_t feature_length;      /* D */
    size_t stage_half_bytes;     /* bytes per pinned staging half; 0 = the library's default (48 MB) */
} sd_level_host_projection;
SD_API int sd_train_level_host_projected(sd_ctx* ctx, sd_comm* comm, const sd_level_host_projection* proj,
                                         const float* d_x, const float* d_x_gt, int N_local, int P, int64_t n_global,
                                         const sd_normalisation* norm, const float* d_templates, int64_t ldt,
                                         const sd_regulariser* reg, int route, float* d_chunk, int64_t ld, int chunk_rows,
                                         float* d_X, float* d_x_next, float* lambda_out);
SD_API int sd_apply_level_host_projected(sd_ctx* ctx, const sd_level_host_projection* proj, const float* d_x, int N, int P,
                                         const sd_normalisation* norm, const float* d_templates, int64_t ldt, const float* d_X,
                                         float* d_chunk, int64_t ld, int chunk_rows, float* d_x_next);

/* host-frame bytes (region bytes x channels) the levels on host frames have read over PCIe on ctx since creation */
SD_API int64_t sd_gathered_bytes(const sd_ctx* ctx);
/* *in_place = 1 when the levels can read a host frame where it is (pinned and device-mapped, 16-byte aligned base and
 * row_stride, row_stride >= channels * roundup16(width)), else 0; a bad frame (as for sd_upload_frames) is SD_ERR_INVALID.  The
 * HogTransform front ends pack the other frames once into pinned memory. */
SD_API int sd_host_frame_in_place(sd_ctx* ctx, const sd_host_frame* frame, int* in_place);
/* free and total memory of the context's device (cudaMemGetInfo): what the HogTransform front ends choose their route by */
SD_API int sd_device_memory(sd_ctx* ctx, size_t* free_bytes, size_t* total_bytes);

/* ---- rcr::detection_model (model.hpp:122-219) -------------------------------------------- */
/* load_detection_model / save_detection_model (model.hpp:192-219): cereal binary, byte compatible */
SD_API int sd_model_load(sd_ctx* ctx, const char* path, sd_model** out);
SD_API int sd_model_save(sd_ctx* ctx, const sd_model* m, const char* path);
/* build a model from trained parts (detection_model ctor, model.hpp:128-129); weights are host
 * pointers, one D_s x 2L matrix per level; ids are NUL-terminated strings. */
SD_API int sd_model_create(sd_ctx* ctx, int num_levels, int num_landmarks,
                           const float* const* h_weights, const sd_regulariser* regs,
                           const sd_hog_param* hog_params, const float* h_mean,
                           const char* const* landmark_ids,
                           const char* const* right_eye_ids, int n_right,
                           const char* const* left_eye_ids, int n_left, sd_model** out);
SD_API void sd_model_destroy(sd_model* m);
SD_API int sd_model_num_levels(const sd_model* m);
SD_API int sd_model_num_landmarks(const sd_model* m);
SD_API int sd_model_hog_param(const sd_model* m, int level, sd_hog_param* out);
SD_API int sd_model_regulariser(const sd_model* m, int level, sd_regulariser* out);
SD_API int sd_model_normalisation(const sd_model* m, sd_normalisation* out);
SD_API int sd_model_get_mean(const sd_model* m, float* h_mean /* 2L */);            /* get_mean, model.hpp:159 */
SD_API int sd_model_get_weights(const sd_model* m, int level, float* h_w /* D x 2L */, int* rows, int* cols);
SD_API const char* sd_model_landmark_id(const sd_model* m, int i);
/* rcr::align_mean (model.hpp:64-76); host-side, a few flops */
SD_API int sd_align_mean(const float* h_mean, int num_landmarks, int box_x, int box_y, int box_w, int box_h,
                         float scaling_x, float scaling_y, float translation_x, float translation_y,
                         float* h_out);
/* Training front end of apps/rcr/rcr-train.cpp.
 * perturb (:130-146): translate a face box by fractions of its size and scale it about its centre (float arithmetic,
 * truncation toward zero like cv::Rect(int)); host-side, a few flops. */
SD_API int sd_perturb_box(int box_x, int box_y, int box_w, int box_h, float translation_x, float translation_y,
                          float scaling, int32_t out_box[4]);
/* calculate_normalised_landmark_errors (:149-212): d_err[r, i] = || pred[r, i] - gt[r, i] ||_2 / IED(pred[r]) for N rows of
 * 2L landmarks each ([x.., y..]); d_err: N x L, row pitch lde. */
SD_API int sd_normalised_landmark_errors(sd_ctx* ctx, const float* d_pred, int64_t ldp, const float* d_gt, int64_t ldgt,
                                         int N, int num_landmarks, const sd_normalisation* eyes, float* d_err, int64_t lde);
/* detection_model::detect(image, initialisation) batched, everything on the device
 * (model.hpp:147-157 -> superviseddescent.hpp:323-344).  d_x0: B x 2L initial landmarks. */
SD_API int sd_detect_batch_device(sd_ctx* ctx, const sd_model* m, const sd_image_batch* images,
                                  const float* d_x0, int count, float* d_landmarks);
/* detection_model::detect(image, facebox) batched with HOST buffers (model.hpp:132-144): aligns the
 * mean to each box, copies the frames host->device in chunks overlapped with compute, runs the cascade
 * and copies the B x 2L landmarks back.  h_images: count x height x row_stride bytes (8UC1; pinned
 * memory makes the copies asynchronous); h_boxes: count x 4 (x, y, w, h). */
SD_API int sd_detect_batch_host(sd_ctx* ctx, const sd_model* m, const uint8_t* h_images, int count,
                                int width, int height, int row_stride, const int32_t* h_boxes,
                                float* h_landmarks);
/* detect(image, facebox) / detect(image, initialisation) (model.hpp:132-157) for num_faces faces in num_frames host frames of
 * any sizes, grey or colour, any number of faces per frame.  Face f lies in frames[h_face_frame[f]].  Exactly one of h_boxes
 * (num_faces x 4: x, y, w, h -> align_mean) and h_x0 (num_faces x 2L initial landmarks, e.g. the previous video frame's) is
 * non-NULL.  h_landmarks: num_faces x 2L, in the caller's face order.  Frames that no face refers to are never read.
 * A face index out of range, channels not 1 or 3, row_stride < width * channels, or both / neither of h_boxes and h_x0 are
 * SD_ERR_INVALID before any work is queued (h_landmarks is not written); so is a degenerate face, as in sd_detect_batch_device.
 * Routes:
 *   - every referenced frame in pinned, device-mapped host memory with a 16-byte aligned base and row_stride: the SMs gather a
 *     neighbourhood of each face (one per face, also for several faces of one frame) straight from the frame, converting
 *     colour pixels to grey on the way; a face whose cascade leaves its neighbourhood is repeated from its whole frame
 *     (sd_roi_fallback_count);
 *   - otherwise each referenced frame is copied to the device once (colour frames then converted there) in chunks
 *     overlapped with the cascade.
 * Both routes give bit-identical landmarks. */
SD_API int sd_detect_faces_host(sd_ctx* ctx, const sd_model* m, const sd_host_frame* frames, int num_frames,
                                const int32_t* h_face_frame, int num_faces, const int32_t* h_boxes, const float* h_x0,
                                float* h_landmarks);
/* sd_detect_batch_device with a face -> frame index: face i lies in images[d_face_frame[i]] (d_face_frame may be NULL: face i
 * in frame i), so a frame with several faces is resident once.  An index out of range is SD_ERR_INVALID. */
SD_API int sd_detect_faces_device(sd_ctx* ctx, const sd_model* m, const sd_image_batch* images, const int32_t* d_face_frame,
                                  const float* d_x0, int num_faces, float* d_landmarks);

#ifdef __cplusplus
}
#endif
#endif /* SD_B200_H */
