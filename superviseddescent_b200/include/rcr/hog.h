// H100 drop-in for include/rcr/hog.h: VLFeat's VlHog object API (hog.h:104-139) with the reference's names and signatures,
// header-only over the C ABI (include/sd_b200.h).  Code written against hog.h -- the reference's examples, and callers of
// vl_hog_put_image / vl_hog_extract on one patch at a time -- compiles against this file unchanged, whether it includes it
// directly or inside extern "C" { } as the reference's own headers do.
//
//   vl_hog_put_image / vl_hog_put_polar_field   upload the caller's buffer, compute the features on the device
//                                               (sd_hog_dense_images / sd_hog_dense_polar) and return once the buffer has
//                                               been read: the caller may overwrite it at once
//   vl_hog_extract                              downloads the features of the last put and synchronises
//   vl_hog_render                               sd_hog_render with the object's glyphs, into the caller's image (read-modify-write)
//   transposed = VL_TRUE                        column-major buffers: the device reads the buffer through swapped strides and
//                                               transposes every feature plane (sd_hog_relayout); width, height and the
//                                               features are in the caller's memory coordinates, as in hog.c
//
// Each call does its work through sd_b200::context(), one context per thread, so objects can be used from a thread pool, one
// object per thread.  Where hog.c asserts, and outside this project's range (cellSize 1..32, numOrientations 1..16, 1..16
// channels), the functions throw std::runtime_error.  One call is one round trip to the device: this is the drop-in for
// existing per-patch code; sd_hog_dense_images and sd_hog_render batch many images per call.  vl_hog_process is declared and
// not defined, as in the reference.
#ifndef VL_HOG_H
#define VL_HOG_H

extern "C++" {

#include <climits>
#include <cstdint>
#include <stdexcept>
#include <string>
#include <vector>

#include "sd_b200/device.hpp"

typedef unsigned long long vl_size;
typedef int vl_bool;
typedef long long vl_index;
typedef unsigned long long vl_uindex;
#define VL_TRUE 1
#define VL_FALSE 0

enum VlHogVariant_ { VlHogVariantDalalTriggs, VlHogVariantUoctti };
typedef enum VlHogVariant_ VlHogVariant;

// This project's object.  Callers use the functions only; the fields are not part of the interface.
struct VlHog_ {
    VlHogVariant variant;
    vl_size numOrientations;
    vl_size dimension;
    vl_bool transposed;
    vl_bool bilinear;
    std::vector<vl_index> permutation;
    vl_size hogWidth, hogHeight;                         // cells of the last put, in the caller's memory coordinates
    bool ready;                                          // a put has run
    mutable sd_b200::DeviceBuffer input, angle, scratch; // device copies of the caller's buffers, grown as needed
    sd_b200::DeviceBuffer features;                      // [dimension][hogHeight][hogWidth] of the last put
};
typedef struct VlHog_ VlHog;

VlHog* vl_hog_new(VlHogVariant variant, vl_size numOrientations, vl_bool transposed);
void vl_hog_delete(VlHog* self);
void vl_hog_process(VlHog* self, float* features, float const* image, vl_size width, vl_size height, vl_size numChannels,
                    vl_size cellSize);
void vl_hog_put_image(VlHog* self, float const* image, vl_size width, vl_size height, vl_size numChannels, vl_size cellSize);
void vl_hog_put_polar_field(VlHog* self, float const* modulus, float const* angle, vl_bool directed, vl_size width, vl_size height,
                            vl_size cellSize);
void vl_hog_extract(VlHog* self, float* features);
vl_size vl_hog_get_height(VlHog* self);
vl_size vl_hog_get_width(VlHog* self);
void vl_hog_render(VlHog const* self, float* image, float const* features, vl_size width, vl_size height);
vl_size vl_hog_get_dimension(VlHog const* self);
vl_index const* vl_hog_get_permutation(VlHog const* self);
vl_size vl_hog_get_glyph_size(VlHog const* self);
vl_bool vl_hog_get_use_bilinear_orientation_assignments(VlHog const* self);
void vl_hog_set_use_bilinear_orientation_assignments(VlHog* self, vl_bool x);

namespace vl_hog_detail {

inline void require(bool ok, const std::string& what)
{
    if (!ok) throw std::runtime_error(what);
}

// The frame of a put as the device reads it: the caller's width x height buffer (x fastest), or -- transposed -- the image whose
// columns are the buffer's rows: height x width pixels, one element apart down a column and width elements apart along a row.
inline sd_hog_image frame(const VlHog* self, vl_size width, vl_size height, int64_t channel_stride)
{
    sd_hog_image f{};
    const int w = static_cast<int>(width), h = static_cast<int>(height);
    if (self->transposed) { f.width = h; f.height = w; f.row_stride = 1; f.pixel_stride = w; }
    else { f.width = w; f.height = h; f.row_stride = w; f.pixel_stride = 1; }
    f.channel_stride = channel_stride;
    return f;
}

// hog.c's asserts (self and the buffers set, width and height > 3, at least half a cell) and this project's range.
inline void check_put(const VlHog* self, const void* a, const void* b, vl_size width, vl_size height, vl_size cellSize, const char* fn)
{
    require(self && a && b, std::string(fn) + ": null argument");
    int w = 0, h = 0, dd = 0;
    const bool ok = width <= INT_MAX && height <= INT_MAX && cellSize >= 1 && cellSize <= 32 &&
                    sd_hog_dense_shape(static_cast<int>(width), static_cast<int>(height), static_cast<int>(cellSize),
                                       static_cast<int>(self->numOrientations), self->variant, &w, &h, &dd) == SD_OK;
    require(ok, std::string(fn) + ": a " + std::to_string(width) + " x " + std::to_string(height) + " buffer with cell size " +
                    std::to_string(cellSize) + " is outside the supported range: width and height > 3 and at least half a cell, "
                    "cellSize 1..32");
}

// Runs launch(d_out) for the frame f, which writes the true-orientation features [dd][h][w]; in transposed mode they go to the
// scratch buffer and every plane is transposed into the object's features.  Returns after the device has finished, so the
// caller's buffers have been read.
template <class Launch>
void compute(VlHog* self, sd_ctx* ctx, const sd_hog_image& f, vl_size cellSize, Launch launch, const char* fn)
{
    int w = 0, h = 0, dd = 0;
    sd_b200::check(ctx, sd_hog_dense_shape(f.width, f.height, static_cast<int>(cellSize), static_cast<int>(self->numOrientations),
                                           self->variant, &w, &h, &dd), fn);
    const size_t bytes = static_cast<size_t>(dd) * w * h * sizeof(float);
    self->ready = false;
    self->features.allocate(bytes);
    if (!self->transposed) {
        sd_b200::check(ctx, launch(self->features.as<float>()), fn);
        self->hogWidth = static_cast<vl_size>(w);
        self->hogHeight = static_cast<vl_size>(h);
    } else {
        self->scratch.allocate(bytes);
        sd_b200::check(ctx, launch(self->scratch.as<float>()), fn);
        sd_hog_grids g{};
        g.d_features = self->scratch.as<float>();
        g.count = 1;
        g.width = w;
        g.height = h;
        sd_b200::check(ctx, sd_hog_relayout(ctx, &g, static_cast<int>(self->numOrientations), self->variant, 0, 1,
                                            self->features.as<float>()), fn);
        self->hogWidth = static_cast<vl_size>(h);
        self->hogHeight = static_cast<vl_size>(w);
    }
    sd_b200::check(ctx, sd_sync(ctx), fn);
    self->ready = true;
}

}  // namespace vl_hog_detail

inline VlHog* vl_hog_new(VlHogVariant variant, vl_size numOrientations, vl_bool transposed)
{
    vl_hog_detail::require(variant == VlHogVariantDalalTriggs || variant == VlHogVariantUoctti, "vl_hog_new: unknown HOG variant");
    vl_hog_detail::require(numOrientations >= 1 && numOrientations <= 16,
                           "vl_hog_new: numOrientations is " + std::to_string(numOrientations) + ", the supported range is 1..16");
    const int K = static_cast<int>(numOrientations);
    VlHog* self = new VlHog();
    self->variant = variant;
    self->numOrientations = numOrientations;
    self->dimension = static_cast<vl_size>(sd_b200::hog_dimension(variant, K));
    self->transposed = transposed ? VL_TRUE : VL_FALSE;
    self->bilinear = VL_FALSE;
    self->hogWidth = self->hogHeight = 0;
    self->ready = false;
    std::vector<int64_t> perm(self->dimension);
    sd_hog_permutation(K, variant, perm.data());
    self->permutation.assign(perm.begin(), perm.end());
    return self;
}

inline void vl_hog_delete(VlHog* self) { delete self; }

inline void vl_hog_put_image(VlHog* self, float const* image, vl_size width, vl_size height, vl_size numChannels, vl_size cellSize)
{
    vl_hog_detail::check_put(self, image, image, width, height, cellSize, "vl_hog_put_image");
    vl_hog_detail::require(numChannels >= 1 && numChannels <= 16,
                           "vl_hog_put_image: numChannels is " + std::to_string(numChannels) + ", the supported range is 1..16");
    sd_ctx* ctx = sd_b200::context();
    const size_t n = static_cast<size_t>(width) * height * numChannels;
    self->input.allocate(n * sizeof(float));
    sd_b200::check(ctx, sd_memcpy_h2d(ctx, self->input.as<float>(), image, n * sizeof(float)), "vl_hog_put_image");
    sd_hog_images im{};
    im.d_data = self->input.as<float>();
    im.dtype = SD_HOG_F32;
    im.channels = static_cast<int32_t>(numChannels);
    im.count = 1;
    im.frame = vl_hog_detail::frame(self, width, height, static_cast<int64_t>(width) * height);
    const int cs = static_cast<int>(cellSize), K = static_cast<int>(self->numOrientations), bil = self->bilinear ? 1 : 0;
    vl_hog_detail::compute(self, ctx, im.frame, cellSize, [&](float* d_out) {
        return sd_hog_dense_images(ctx, &im, cs, K, self->variant, bil, d_out, nullptr);
    }, "vl_hog_put_image");
}

inline void vl_hog_put_polar_field(VlHog* self, float const* modulus, float const* angle, vl_bool directed, vl_size width, vl_size height,
                                   vl_size cellSize)
{
    vl_hog_detail::check_put(self, modulus, angle, width, height, cellSize, "vl_hog_put_polar_field");
    sd_ctx* ctx = sd_b200::context();
    const size_t bytes = static_cast<size_t>(width) * height * sizeof(float);
    self->input.allocate(bytes);
    self->angle.allocate(bytes);
    sd_b200::check(ctx, sd_memcpy_h2d(ctx, self->input.as<float>(), modulus, bytes), "vl_hog_put_polar_field");
    sd_b200::check(ctx, sd_memcpy_h2d(ctx, self->angle.as<float>(), angle, bytes), "vl_hog_put_polar_field");
    sd_hog_polar_fields pf{};
    pf.d_modulus = self->input.as<float>();
    pf.d_angle = self->angle.as<float>();
    pf.count = 1;
    pf.frame = vl_hog_detail::frame(self, width, height, 0);
    const int cs = static_cast<int>(cellSize), K = static_cast<int>(self->numOrientations), bil = self->bilinear ? 1 : 0;
    vl_hog_detail::compute(self, ctx, pf.frame, cellSize, [&](float* d_out) {
        return sd_hog_dense_polar(ctx, &pf, cs, K, self->variant, directed ? 1 : 0, bil, d_out, nullptr);
    }, "vl_hog_put_polar_field");
}

inline void vl_hog_extract(VlHog* self, float* features)
{
    vl_hog_detail::require(self && features, "vl_hog_extract: null argument");
    vl_hog_detail::require(self->ready, "vl_hog_extract: no features: call vl_hog_put_image or vl_hog_put_polar_field first");
    sd_ctx* ctx = sd_b200::context();
    const size_t bytes = static_cast<size_t>(self->dimension * self->hogWidth * self->hogHeight) * sizeof(float);
    sd_b200::check(ctx, sd_memcpy_d2h(ctx, features, self->features.as<float>(), bytes), "vl_hog_extract");
    sd_b200::check(ctx, sd_sync(ctx), "vl_hog_extract");
}

inline vl_size vl_hog_get_height(VlHog* self) { return self->hogHeight; }
inline vl_size vl_hog_get_width(VlHog* self) { return self->hogWidth; }

inline void vl_hog_render(VlHog const* self, float* image, float const* features, vl_size width, vl_size height)
{
    vl_hog_detail::require(self && image && features, "vl_hog_render: null argument");
    vl_hog_detail::require(width > 0 && height > 0 && width <= INT_MAX / SD_HOG_GLYPH_SIZE && height <= INT_MAX / SD_HOG_GLYPH_SIZE,
                           "vl_hog_render: a " + std::to_string(width) + " x " + std::to_string(height) +
                               " grid of cells is outside the supported range: 1.." + std::to_string(INT_MAX / SD_HOG_GLYPH_SIZE) +
                               " cells per side");
    sd_ctx* ctx = sd_b200::context();
    const size_t cells = static_cast<size_t>(width) * height;
    const size_t in_bytes = static_cast<size_t>(self->dimension) * cells * sizeof(float);
    const size_t img_bytes = cells * SD_HOG_GLYPH_SIZE * SD_HOG_GLYPH_SIZE * sizeof(float);
    self->input.allocate(in_bytes);
    self->scratch.allocate(img_bytes);
    sd_b200::check(ctx, sd_memcpy_h2d(ctx, self->input.as<float>(), features, in_bytes), "vl_hog_render");
    sd_b200::check(ctx, sd_memcpy_h2d(ctx, self->scratch.as<float>(), image, img_bytes), "vl_hog_render");
    sd_hog_grids g{};
    g.d_features = self->input.as<float>();
    g.count = 1;
    g.width = static_cast<int32_t>(width);
    g.height = static_cast<int32_t>(height);
    sd_b200::check(ctx, sd_hog_render(ctx, &g, static_cast<int>(self->numOrientations), self->variant, self->transposed ? 1 : 0,
                                      self->scratch.as<float>()), "vl_hog_render");
    sd_b200::check(ctx, sd_memcpy_d2h(ctx, image, self->scratch.as<float>(), img_bytes), "vl_hog_render");
    sd_b200::check(ctx, sd_sync(ctx), "vl_hog_render");
}

inline vl_size vl_hog_get_dimension(VlHog const* self) { return self->dimension; }
inline vl_index const* vl_hog_get_permutation(VlHog const* self) { return self->permutation.data(); }
inline vl_size vl_hog_get_glyph_size(VlHog const*) { return SD_HOG_GLYPH_SIZE; }
inline vl_bool vl_hog_get_use_bilinear_orientation_assignments(VlHog const* self) { return self->bilinear; }
inline void vl_hog_set_use_bilinear_orientation_assignments(VlHog* self, vl_bool x) { self->bilinear = x; }

}  // extern "C++"

#endif  // VL_HOG_H
