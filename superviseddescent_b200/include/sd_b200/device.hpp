// Glue between the C++14 header shells and the C ABI (include/sd_b200.h): one lazily created context
// per host thread, RAII device buffers, and translation of status codes into the exception types the
// reference throws (std::runtime_error, SURVEY.md 8b "Errors").
#pragma once

#include <cstdlib>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "sd_b200.h"
#include "sd_b200/mat.hpp"

namespace sd_b200 {

inline void check(sd_ctx* ctx, int rc, const char* what)
{
    if (rc == SD_OK) return;
    std::string msg = ctx ? sd_last_error(ctx) : "no CUDA device / context (the engine has no CPU fallback)";
    throw std::runtime_error(std::string(what) + ": " + msg);
}

// One context per host thread (re-entrant on distinct contexts, SURVEY 8b "Threading").
// The device ordinal comes from SD_B200_DEVICE (default 0).
inline sd_ctx* context()
{
    struct Holder {
        sd_ctx* ctx = nullptr;
        Holder()
        {
            const char* env = std::getenv("SD_B200_DEVICE");
            const int dev = env ? std::atoi(env) : 0;
            const int rc = sd_ctx_create(dev, nullptr, &ctx);
            if (rc != SD_OK) throw std::runtime_error("sd_ctx_create failed: no usable CUDA device (the engine has no CPU fallback)");
        }
        ~Holder() { sd_ctx_destroy(ctx); }
    };
    static thread_local Holder holder;
    return holder.ctx;
}

class DeviceBuffer {
public:
    DeviceBuffer() = default;
    explicit DeviceBuffer(size_t bytes) { allocate(bytes); }
    DeviceBuffer(const DeviceBuffer&) = delete;
    DeviceBuffer& operator=(const DeviceBuffer&) = delete;
    DeviceBuffer(DeviceBuffer&& o) noexcept : ptr_(o.ptr_), bytes_(o.bytes_) { o.ptr_ = nullptr; o.bytes_ = 0; }
    DeviceBuffer& operator=(DeviceBuffer&& o) noexcept { std::swap(ptr_, o.ptr_); std::swap(bytes_, o.bytes_); return *this; }
    ~DeviceBuffer() { if (ptr_) sd_free(context(), ptr_); }
    void allocate(size_t bytes)
    {
        if (bytes <= bytes_) return;
        if (ptr_) { sd_free(context(), ptr_); ptr_ = nullptr; }
        check(context(), sd_malloc(context(), bytes, &ptr_), "sd_malloc");
        bytes_ = bytes;
    }
    template <class T> T* as() const { return static_cast<T*>(ptr_); }
    size_t bytes() const { return bytes_; }

private:
    void* ptr_ = nullptr;
    size_t bytes_ = 0;
};

// pinned host memory (sd_host_alloc), e.g. frames the HogTransform keeps in host memory
class HostBuffer {
public:
    HostBuffer() = default;
    HostBuffer(const HostBuffer&) = delete;
    HostBuffer& operator=(const HostBuffer&) = delete;
    ~HostBuffer() { if (ptr_) sd_host_free(context(), ptr_); }
    void allocate(size_t bytes)
    {
        if (ptr_) { sd_host_free(context(), ptr_); ptr_ = nullptr; }
        check(context(), sd_host_alloc(context(), bytes, &ptr_), "sd_host_alloc");
    }
    template <class T> T* as() const { return static_cast<T*>(ptr_); }

private:
    void* ptr_ = nullptr;
};

// packed float32 cv::Mat -> device (row stride ld floats, ld >= cols)
inline void upload(const cv::Mat& m, DeviceBuffer& dst, int64_t ld)
{
    dst.allocate(static_cast<size_t>(m.rows) * ld * sizeof(float));
    sd_ctx* ctx = context();
    if (m.isContinuous() && ld == m.cols) {
        check(ctx, sd_memcpy_h2d(ctx, dst.as<float>(), m.ptr<float>(0), static_cast<size_t>(m.rows) * m.cols * sizeof(float)), "upload");
    } else {   // strided on either side: one 2-D copy
        check(ctx, sd_memcpy2d_h2d(ctx, dst.as<float>(), static_cast<size_t>(ld) * sizeof(float), m.ptr<float>(0), m.step(),
                                   static_cast<size_t>(m.cols) * sizeof(float), static_cast<size_t>(m.rows)), "upload");
    }
    check(ctx, sd_sync(ctx), "upload");   // the host Mat may go away after this call
}

// 8UC1 / 8UC3 (B,G,R) frames as the C ABI's host frames: the pixels stay where they are, Mat::step() is the row stride
inline std::vector<sd_host_frame> host_frames(const std::vector<cv::Mat>& images)
{
    std::vector<sd_host_frame> frames(images.size());
    for (size_t i = 0; i < images.size(); ++i) {
        const cv::Mat& im = images[i];
        frames[i] = sd_host_frame{im.ptr<unsigned char>(0), im.cols, im.rows, static_cast<int32_t>(im.step()), im.channels()};
    }
    return frames;
}

// dd, the features per HOG cell of vl_hog_new(variant, num_bins): 3K + 4 for UoCTTI (variant 1), 4K for Dalal-Triggs
inline int hog_dimension(int variant, int num_bins) { return variant == 1 ? 3 * num_bins + 4 : 4 * num_bins; }

inline cv::Mat download(const float* d, int rows, int cols, int64_t ld)
{
    cv::Mat m(rows, cols, CV_32FC1);
    sd_ctx* ctx = context();
    if (ld == cols) {
        check(ctx, sd_memcpy_d2h(ctx, m.ptr<float>(0), d, static_cast<size_t>(rows) * cols * sizeof(float)), "download");
    } else {
        check(ctx, sd_memcpy2d_d2h(ctx, m.ptr<float>(0), m.step(), d, static_cast<size_t>(ld) * sizeof(float),
                                   static_cast<size_t>(cols) * sizeof(float), static_cast<size_t>(rows)), "download");
    }
    check(ctx, sd_sync(ctx), "download");
    return m;
}

}  // namespace sd_b200
