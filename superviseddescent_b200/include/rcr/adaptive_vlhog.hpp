// H100 drop-in for include/rcr/adaptive_vlhog.hpp: HoGParam (:41-60) and the projection functor
// HogTransform (:70-195).  The functor keeps the reference's constructor and call signature
//     cv::Mat operator()(cv::Mat parameters, size_t regressorLevel, int trainingIndex = 0)
// (one sample, used by predict(), superviseddescent.hpp:332) and exposes its device images, eyes and per-level
// HOG parameters, with which the optimiser projects ALL samples of a level on the device (sd_train_level, sd_apply_level).
// Each distinct image is held once: uploaded to HBM on first use, or kept in host memory when it does not fit; crop / resize /
// HOG run in sd_hog_batch (sm_90a).
#pragma once

#include <algorithm>
#include <array>
#include <cstring>
#include <map>
#include <memory>
#include <string>
#include <tuple>
#include <vector>

#include "rcr/helpers.hpp"
#include "rcr/hog.h"   // VlHogVariant, and VLFeat's VlHog API for callers that include this header only
#include "sd_b200/device.hpp"

namespace rcr {

struct HoGParam {
    VlHogVariant vlhog_variant;
    int num_cells;
    int cell_size;
    int num_bins;
    float relative_patch_size;
    sd_hog_param c() const { sd_hog_param p; p.variant = vlhog_variant; p.num_cells = num_cells; p.cell_size = cell_size; p.num_bins = num_bins; p.relative_patch_size = relative_patch_size; return p; }
};

namespace hog_batch {

// The results of one batched call, end to end in one device buffer: item i is a CV_32FC1 Mat of rows[i] x cols[i] floats at
// offset[i].  An item without rows or columns is empty: it holds nothing and downloads as an empty Mat.
struct Results {
    std::vector<int64_t> offset;
    std::vector<int> rows, cols;
    int64_t total = 0;
    sd_b200::DeviceBuffer d_out, d_offset;

    void add(int r, int c)
    {
        if (r <= 0 || c <= 0) r = c = 0;
        offset.push_back(total);
        rows.push_back(r);
        cols.push_back(c);
        total += static_cast<int64_t>(r) * c;
    }
    // the buffer, one float at least, so that a call whose items are all empty gets a valid pointer
    float* out()
    {
        d_out.allocate(static_cast<size_t>(std::max<int64_t>(total, 1)) * sizeof(float));
        return d_out.as<float>();
    }
    // the items' offsets, uploaded for the calls that take one int64 offset per item
    const int64_t* offsets(sd_ctx* ctx, const char* what)
    {
        d_offset.allocate(offset.size() * sizeof(int64_t));
        sd_b200::check(ctx, sd_memcpy_h2d(ctx, d_offset.as<int64_t>(), offset.data(), offset.size() * sizeof(int64_t)), what);
        return d_offset.as<int64_t>();
    }
    std::vector<cv::Mat> download() const
    {
        std::vector<cv::Mat> items;
        for (size_t i = 0; i < offset.size(); ++i)
            items.push_back(cols[i] ? sd_b200::download(d_out.as<float>() + offset[i], rows[i], cols[i], cols[i]) : cv::Mat());
        return items;
    }
};

// 8UC1 / 8UC3 (B,G,R) frames on the device as one grey batch (sd_upload_frames), in buf
inline sd_image_batch upload_grey(sd_ctx* ctx, const std::vector<sd_host_frame>& frames, sd_b200::DeviceBuffer& buf, const char* what)
{
    const int n = static_cast<int>(frames.size());
    size_t bytes = 0;
    sd_b200::check(ctx, sd_upload_frames(ctx, frames.data(), n, nullptr, &bytes, nullptr), what);
    buf.allocate(bytes);
    sd_image_batch batch{};
    sd_b200::check(ctx, sd_upload_frames(ctx, frames.data(), n, buf.as<void>(), &bytes, &batch), what);
    return batch;
}

// The output of one sd_hog_detections call on the host: the n frames' max(max_detections, 1) slots each into out; returns each
// frame's detection count.  Copies queued on the stream before the call are complete when it returns.
inline std::vector<int32_t> download_detections(sd_ctx* ctx, const sd_b200::DeviceBuffer& d_out, const sd_b200::DeviceBuffer& d_count,
                                                int n, int max_detections, std::vector<sd_hog_detection>& out, const char* what)
{
    out.resize(static_cast<size_t>(n) * static_cast<size_t>(std::max(max_detections, 1)));
    std::vector<int32_t> count(n);
    sd_b200::check(ctx, sd_memcpy_d2h(ctx, out.data(), d_out.as<void>(), out.size() * sizeof(sd_hog_detection)), what);
    sd_b200::check(ctx, sd_memcpy_d2h(ctx, count.data(), d_count.as<void>(), count.size() * sizeof(int32_t)), what);
    sd_b200::check(ctx, sd_sync(ctx), what);
    return count;
}

// CV_8UC1 or CV_32FC1 planes of elem_size bytes per element (row steps allowed) packed end to end into buf, in the order
// given; returns where each plane starts, in elements
inline std::vector<int64_t> pack_planes(sd_ctx* ctx, const std::vector<cv::Mat>& planes, size_t elem_size, sd_b200::DeviceBuffer& buf,
                                        const char* what)
{
    std::vector<int64_t> start(planes.size());
    int64_t elems = 0;
    for (size_t i = 0; i < planes.size(); ++i) {
        start[i] = elems;
        elems += static_cast<int64_t>(planes[i].rows) * planes[i].cols;
    }
    buf.allocate(static_cast<size_t>(elems) * elem_size);
    for (size_t i = 0; i < planes.size(); ++i) {
        const cv::Mat& p = planes[i];
        const size_t row_bytes = static_cast<size_t>(p.cols) * elem_size;
        sd_b200::check(ctx, sd_memcpy2d_h2d(ctx, buf.as<unsigned char>() + static_cast<size_t>(start[i]) * elem_size, row_bytes,
                                            p.ptr<unsigned char>(0), p.step(), row_bytes, static_cast<size_t>(p.rows)), what);
    }
    return start;
}

// Frames of one type with C channels of elem bytes each (checked by the caller) on the device, interleaved as OpenCV holds
// them: packed end to end into buf (row steps dropped), one descriptor per frame in table (and in *desc, if given)
inline sd_hog_images upload_interleaved(sd_ctx* ctx, const std::vector<cv::Mat>& images, size_t elem, int dtype,
                                        sd_b200::DeviceBuffer& buf, sd_b200::DeviceBuffer& table, const char* what,
                                        std::vector<sd_hog_image>* desc_out = nullptr)
{
    const int n = static_cast<int>(images.size()), C = images[0].channels();
    const std::vector<int64_t> start = pack_planes(ctx, images, elem * static_cast<size_t>(C), buf, what);
    std::vector<sd_hog_image> desc;
    for (int i = 0; i < n; ++i)
        desc.push_back(sd_hog_image{images[i].cols, images[i].rows, start[i] * C, static_cast<int64_t>(images[i].cols) * C, C, 1});
    table.allocate(desc.size() * sizeof(sd_hog_image));
    sd_b200::check(ctx, sd_memcpy_h2d(ctx, table.as<sd_hog_image>(), desc.data(), desc.size() * sizeof(sd_hog_image)), what);
    sd_hog_images batch{};
    batch.d_data = buf.as<void>();
    batch.dtype = dtype;
    batch.channels = C;
    batch.count = n;
    batch.d_frames = table.as<sd_hog_image>();
    if (desc_out) *desc_out = desc;
    return batch;
}

// The flags of a sliding-window call (vl_hog_pyramid, train_hog_filter, hog_box_scores, the tracking steps): bilinear_orientations
// and float_frames need multichannel.  Throws std::runtime_error naming what.
inline void check_window_flags(bool multichannel, bool bilinear_orientations, bool float_frames, const char* what)
{
    if (bilinear_orientations && !multichannel) throw std::runtime_error(std::string(what) + ": bilinear_orientations needs multichannel");
    if (float_frames && !multichannel) throw std::runtime_error(std::string(what) + ": float_frames needs multichannel");
}

// The frames of a sliding-window call on the device: grey or colour as the call's flags select.
struct WindowFrames {
    sd_image_batch grey{};              // without multichannel
    sd_hog_images colour{};             // with multichannel
    sd_b200::DeviceBuffer buf, table;
};

// Checks the flags (check_window_flags) and uploads.  Without multichannel the frames (8UC1 / 8UC3 B,G,R) become the grey batch
// (upload_grey).  With it they keep their channels (upload_interleaved, which fills *desc_out if given): all CV_8UC1 or all
// CV_8UC3, or with float_frames all CV_32FC1 or all CV_32FC3.  Throws std::runtime_error naming what where either refuses.
inline void upload_window_frames(sd_ctx* ctx, const std::vector<cv::Mat>& images, bool multichannel, bool bilinear_orientations,
                                 bool float_frames, WindowFrames& out, const char* what, std::vector<sd_hog_image>* desc_out = nullptr)
{
    check_window_flags(multichannel, bilinear_orientations, float_frames, what);
    if (!multichannel) {
        out.grey = upload_grey(ctx, sd_b200::host_frames(images), out.buf, what);
        return;
    }
    const int type1 = float_frames ? CV_32FC1 : CV_8UC1, type3 = float_frames ? CV_32FC3 : CV_8UC3;
    for (const cv::Mat& m : images)
        if (m.type() != images[0].type() || (m.type() != type1 && m.type() != type3))
            throw std::runtime_error(std::string(what) + (float_frames ? ": float frames must be all CV_32FC1 or all CV_32FC3"
                                                                       : ": frames must be all CV_8UC1 or all CV_8UC3"));
    out.colour = upload_interleaved(ctx, images, float_frames ? sizeof(float) : 1, float_frames ? SD_HOG_F32 : SD_HOG_U8, out.buf,
                                    out.table, what, desc_out);
}

// The frames of a tracking step: colour, the frames the filter reads, and grey, the cascade's grey batch.  Without multichannel
// grey is the window frames' grey batch.  With it the grey frames are *grey_images (8UC1 / 8UC3, the sizes of images) when
// given; else 8UC3 frames are converted on the device (sd_bgr2gray_images, so a colour frame is uploaded once) and 8UC1 frames
// are read in place; float frames need grey_images.
struct TrackFrames : WindowFrames {
    sd_b200::DeviceBuffer grey_buf;
};

// sd_bgr2gray_images' size for frames of these sizes, by the layout include/sd_b200.h states (sd_upload_frames'): no read-back
inline size_t bgr2gray_bytes(const std::vector<sd_hog_image>& desc)
{
    size_t bytes = 0;
    bool uniform = true;
    for (const sd_hog_image& d : desc) {
        bytes += static_cast<size_t>(d.height) * ((static_cast<size_t>(d.width) + 15) / 16 * 16);
        uniform = uniform && d.width == desc[0].width && d.height == desc[0].height;
    }
    return bytes + (uniform ? 0 : desc.size() * sizeof(sd_frame));
}

inline void upload_track_frames(sd_ctx* ctx, const std::vector<cv::Mat>& images, bool multichannel, bool bilinear_orientations,
                                bool float_frames, const std::vector<cv::Mat>* grey_images, TrackFrames& out, const char* what)
{
    const std::string w(what);
    check_window_flags(multichannel, bilinear_orientations, float_frames, what);
    if (grey_images && !multichannel) throw std::runtime_error(w + ": grey_images needs multichannel (grey frames are the cascade's)");
    std::vector<sd_hog_image> desc;
    upload_window_frames(ctx, images, multichannel, bilinear_orientations, float_frames, out, what, &desc);
    if (!multichannel) return;
    if (grey_images) {
        if (grey_images->size() != images.size()) throw std::runtime_error(w + ": grey_images needs one frame per frame");
        out.grey = upload_grey(ctx, sd_b200::host_frames(*grey_images), out.grey_buf, what);
    } else if (float_frames) {
        throw std::runtime_error(w + ": float frames need grey_images for the cascade");
    } else if (images[0].type() == CV_8UC3) {
        size_t bytes = bgr2gray_bytes(desc);
        out.grey_buf.allocate(bytes);
        sd_b200::check(ctx, sd_bgr2gray_images(ctx, &out.colour, out.grey_buf.as<void>(), &bytes, &out.grey), what);
    } else {                                  // 8UC1: the grey batch is the uploaded frames, with its own sd_frame table
        std::vector<sd_frame> grey;
        for (const sd_hog_image& d : desc) grey.push_back(sd_frame{d.width, d.height, static_cast<int32_t>(d.row_stride), 0, d.offset});
        out.grey_buf.allocate(grey.size() * sizeof(sd_frame));
        sd_b200::check(ctx, sd_memcpy_h2d(ctx, out.grey_buf.as<void>(), grey.data(), grey.size() * sizeof(sd_frame)), what);
        out.grey.d_data = static_cast<const uint8_t*>(out.colour.d_data);
        out.grey.count = out.colour.count;
        out.grey.d_frames = out.grey_buf.as<sd_frame>();
    }
}

}  // namespace hog_batch

class HogTransform {
public:
    // Do not call with `images` that are temporaries (the reference holds a const&, adaptive_vlhog.hpp:188).
    // mirrored (optional, one entry per image entry, i.e. per sample): entry i is a sample of the left-right mirror of its photo
    // (cv::flip(image, 1)), with its landmarks in the mirror's coordinates (rcr::mirror_landmarks).  The photo is still held once
    // -- a mirrored shallow copy shares its frame -- and read right to left (SD_SAMPLE_MIRRORED): rows, weights and predictions are
    // bit for bit those of a flipped deep copy.
    // warps (optional, one sd_sample_warp per image entry; not with mirrored): entry i is a sample of the virtual frame
    // V = cv::warpAffine(grey photo, warps[i].m, (width, height), INTER_LINEAR | WARP_INVERSE_MAP) (rcr::rotation_warp,
    // rcr::make_warp), with its landmarks in V's coordinates (rcr::warp_landmarks).  V is never built; rows, weights and predictions
    // are bit for bit those of V passed as an image of its own.
    HogTransform(const std::vector<cv::Mat>& images, std::vector<HoGParam> hog_params, std::vector<std::string> modelLandmarksList,
                 std::vector<std::string> rightEyeIdentifiers, std::vector<std::string> leftEyeIdentifiers,
                 std::vector<bool> mirrored = {}, std::vector<sd_sample_warp> warps = {})
        : images(images), hog_params(hog_params), modelLandmarksList(modelLandmarksList), rightEyeIdentifiers(rightEyeIdentifiers),
          leftEyeIdentifiers(leftEyeIdentifiers), mirrored(mirrored), warps(warps), dev(std::make_shared<DeviceImages>())
    {
        if (!this->mirrored.empty() && this->mirrored.size() != images.size())
            throw std::runtime_error("HogTransform: mirrored needs one entry per image");
        if (!this->warps.empty() && this->warps.size() != images.size())
            throw std::runtime_error("HogTransform: warps needs one entry per image");
        if (!this->warps.empty() && !this->mirrored.empty())
            throw std::runtime_error("HogTransform: mirrored and warps exclude each other (a mirror is the warp [-1, 0, W - 1; 0, 1, 0])");
    }

    int feature_length(size_t level) const
    {
        const sd_hog_param p = hog_params[level].c();
        return sd_hog_feature_length(static_cast<int>(modelLandmarksList.size()), &p);
    }

    // Features of ONE sample (adaptive_vlhog.hpp:109-185)
    cv::Mat operator()(cv::Mat parameters, size_t regressorLevel, int trainingIndex = 0)
    {
        sd_ctx* ctx = sd_b200::context();
        const sd_image_batch& batch = device_batch();
        const int D = feature_length(regressorLevel);
        sd_b200::DeviceBuffer dx, dA(static_cast<size_t>(D) * sizeof(float)), didx(sizeof(int32_t));
        sd_b200::upload(parameters, dx, parameters.cols);
        // an index outside images stays out of range, and the projection reports it
        const int32_t idx = trainingIndex >= 0 && trainingIndex < static_cast<int>(dev->frame_of.size()) ? sample_index(trainingIndex) : -1;
        sd_b200::check(ctx, sd_memcpy_h2d(ctx, didx.as<int32_t>(), &idx, sizeof(idx)), "HogTransform");
        const sd_normalisation nrm = eyes();
        const sd_hog_param p = hog_params[regressorLevel].c();
        const int L = static_cast<int>(modelLandmarksList.size());
        if (!warps.empty() && idx >= 0) {
            const sd_b200::DeviceBuffer dw(sizeof(sd_sample_warp));
            sd_b200::check(ctx, sd_memcpy_h2d(ctx, dw.as<sd_sample_warp>(), &warps[trainingIndex], sizeof(sd_sample_warp)), "HogTransform");
            sd_b200::check(ctx, sd_hog_batch_warped(ctx, &batch, didx.as<int32_t>(), dx.as<float>(), parameters.cols, 1, L, &nrm, &p,
                                                    dw.as<sd_sample_warp>(), dA.as<float>(), D), "sd_hog_batch_warped");
            return sd_b200::download(dA.as<float>(), 1, D, D);
        }
        sd_b200::check(ctx, sd_hog_batch(ctx, &batch, didx.as<int32_t>(), dx.as<float>(), parameters.cols, 1, L,
                                         &nrm, &p, dA.as<float>(), D), "sd_hog_batch");
        return sd_b200::download(dA.as<float>(), 1, D, D);
    }

    // The route, chosen once on first use: the distinct frames are uploaded when their grey bytes fit in device_frame_share() of
    // the free device memory; otherwise they stay in host memory and the optimiser's train() / test() read them level by level.
    // Uploaded frames are copied when the transform is first used; frames kept on the
    // host are read in place at every level when they are pinned and aligned (sd_host_frame_in_place), and copied once into one
    // pinned buffer otherwise.
    static double& device_frame_share()
    {
        static double share = 0.5;
        return share;
    }
    bool on_device()
    {
        ensure_ready();
        return !dev->host;
    }

    // The distinct images resident on the device (uploaded on first use), for the one-sample operator()
    const sd_image_batch& device_batch()
    {
        ensure_ready();
        if (dev->host) throw std::runtime_error("HogTransform: the frames stay in host memory (they do not fit on the device); only the optimiser's train() / test() / predict() read them");
        return dev->batch;
    }
    // What the optimiser hands to sd_train_level / sd_apply_level with the eye landmarks (eyes()) and a level's HOG parameters: the
    // distinct frames -- on the device, or in host memory -- and the index by which sample i reads the frame of images[i].  Entries
    // of `images` with equal data, size and step (rcr-train's shallow copies of one photo) are one frame, held once.
    sd_level_frames level_frames(int n)
    {
        ensure_ready();
        if (n > static_cast<int>(images.size())) throw std::runtime_error("HogTransform: more samples than images");
        sd_level_frames f{};
        if (dev->host) {
            f.host_frames = dev->frames.data();
            f.num_host_frames = static_cast<int32_t>(dev->frames.size());
        } else {
            f.images = &dev->batch;
        }
        f.d_sample_frame = dev->index.as<int32_t>();
        f.d_sample_warp = warps.empty() ? nullptr : dev->warp.as<sd_sample_warp>();
        return f;
    }
    // number of distinct frames
    int num_frames()
    {
        ensure_ready();
        return static_cast<int>(dev->frames.size());
    }
    sd_hog_param hog_param(size_t level) const { return hog_params[level].c(); }

    sd_normalisation eyes() const
    {
        sd_normalisation nrm{};
        nrm.kind = 1;
        const auto r = eye_indices(modelLandmarksList, rightEyeIdentifiers, "right");
        const auto l = eye_indices(modelLandmarksList, leftEyeIdentifiers, "left");
        if (r.empty() || l.empty() || r.size() > 4 || l.size() > 4) throw std::runtime_error("HogTransform: 1..4 eye identifiers per eye are supported");
        nrm.n_right = static_cast<int>(r.size());
        nrm.n_left = static_cast<int>(l.size());
        for (size_t i = 0; i < r.size(); ++i) nrm.right_idx[i] = r[i];
        for (size_t i = 0; i < l.size(); ++i) nrm.left_idx[i] = l[i];
        return nrm;
    }

private:
    // the frame image entry i reads, with SD_SAMPLE_MIRRORED when the entry is mirrored
    int32_t sample_index(size_t i) const
    {
        return dev->frame_of[i] | (!mirrored.empty() && mirrored[i] ? SD_SAMPLE_MIRRORED : 0);
    }

    struct DeviceImages {
        std::vector<sd_host_frame> frames;   // the distinct frames (on the host route: where the levels read them)
        std::vector<int32_t> frame_of;        // images[i] -> distinct frame
        sd_b200::DeviceBuffer index;          // frame_of on the device
        sd_b200::DeviceBuffer warp;           // the entries' warps on the device (when there are any)
        sd_b200::DeviceBuffer buf;            // device route: the grey frames
        sd_image_batch batch{};
        sd_b200::HostBuffer packed;           // host route: the frames that could not be read in place
        bool host = false;
        bool ready = false;
    };

    // frames of any sizes (the reference's std::vector<cv::Mat>), grey or colour: colour is converted once on the device, where the
    // reference converts it in every call (adaptive_vlhog.hpp:114-120).  Each distinct frame is held once.
    void ensure_ready()
    {
        if (dev->ready) return;
        if (images.empty()) throw std::runtime_error("HogTransform: no images");
        sd_ctx* ctx = sd_b200::context();
        const std::vector<sd_host_frame> all = sd_b200::host_frames(images);
        std::vector<sd_host_frame>& frames = dev->frames;
        std::map<std::tuple<const void*, int, int, int, int>, int32_t> seen;
        dev->frame_of.resize(all.size());
        size_t grey = 0;
        for (size_t i = 0; i < all.size(); ++i) {
            const sd_host_frame& f = all[i];
            const auto key = std::make_tuple(static_cast<const void*>(f.h_data), f.width, f.height, f.row_stride, f.channels);
            const auto it = seen.find(key);
            if (it != seen.end()) { dev->frame_of[i] = it->second; continue; }
            dev->frame_of[i] = seen[key] = static_cast<int32_t>(frames.size());
            frames.push_back(f);
            grey += static_cast<size_t>(f.height) * ((static_cast<size_t>(f.width) + 15) / 16 * 16);
        }
        std::vector<int32_t> index(all.size());
        for (size_t i = 0; i < all.size(); ++i) index[i] = sample_index(i);
        dev->index.allocate(all.size() * sizeof(int32_t));
        sd_b200::check(ctx, sd_memcpy_h2d(ctx, dev->index.as<int32_t>(), index.data(), all.size() * sizeof(int32_t)), "HogTransform upload");
        if (!warps.empty()) {
            dev->warp.allocate(warps.size() * sizeof(sd_sample_warp));
            sd_b200::check(ctx, sd_memcpy_h2d(ctx, dev->warp.as<sd_sample_warp>(), warps.data(), warps.size() * sizeof(sd_sample_warp)),
                           "HogTransform upload");
        }
        sd_b200::check(ctx, sd_sync(ctx), "HogTransform upload");
        size_t free_bytes = 0, total = 0;
        sd_b200::check(ctx, sd_device_memory(ctx, &free_bytes, &total), "sd_device_memory");
        if (static_cast<double>(grey) <= device_frame_share() * static_cast<double>(free_bytes)) {
            dev->batch = hog_batch::upload_grey(ctx, frames, dev->buf, "HogTransform upload");
        } else {
            // host route: frames the levels cannot read in place are packed once into one pinned buffer, rows at a pitch of
            // channels * (width rounded up to 16) bytes
            std::vector<char> pack(frames.size());
            size_t packed = 0;
            for (size_t f = 0; f < frames.size(); ++f) {
                int in_place = 0;
                sd_b200::check(ctx, sd_host_frame_in_place(ctx, &frames[f], &in_place), "HogTransform");
                pack[f] = !in_place;
                if (pack[f]) packed += static_cast<size_t>(frames[f].height) * frames[f].channels * ((static_cast<size_t>(frames[f].width) + 15) / 16 * 16);
            }
            if (packed) dev->packed.allocate(packed);
            unsigned char* dst = dev->packed.as<unsigned char>();
            for (size_t f = 0; f < frames.size(); ++f) {
                if (!pack[f]) continue;
                sd_host_frame& fr = frames[f];
                const size_t pitch = static_cast<size_t>(fr.channels) * ((static_cast<size_t>(fr.width) + 15) / 16 * 16);
                for (int y = 0; y < fr.height; ++y)
                    std::memcpy(dst + y * pitch, fr.h_data + static_cast<size_t>(y) * fr.row_stride, static_cast<size_t>(fr.width) * fr.channels);
                fr.h_data = dst;
                fr.row_stride = static_cast<int32_t>(pitch);
                dst += pitch * fr.height;
            }
            dev->host = true;
        }
        dev->ready = true;
    }

    const std::vector<cv::Mat>& images;
    std::vector<HoGParam> hog_params;
    std::vector<std::string> modelLandmarksList;
    std::vector<std::string> rightEyeIdentifiers;
    std::vector<std::string> leftEyeIdentifiers;
    std::vector<bool> mirrored;          // per image entry: a sample of the photo's mirror (empty: none)
    std::vector<sd_sample_warp> warps;   // per image entry: the warp of its photo it samples (empty: none)
    std::shared_ptr<DeviceImages> dev;   // shared between the copies the optimiser makes of this functor
};

// VLFeat HOG of whole frames (hog.h:104-139: vl_hog_new(variant, num_bins), vl_hog_put_image(frame, 1 channel, cell_size),
// vl_hog_extract), for frames of any sizes, 8UC1 or 8UC3 (B,G,R, converted to grey as HogTransform does), in one batched call
// on the device (sd_hog_dense).  Returns one CV_32FC1 Mat per frame with dd * hogH rows and hogW columns: VLFeat's planar
// [dd][hogH][hogW] order, so row d * hogH + y holds dimension d of cell row y.  Throws std::runtime_error for a frame or a
// configuration that sd_hog_dense_shape refuses.
inline std::vector<cv::Mat> hog_dense(const std::vector<cv::Mat>& images, VlHogVariant variant, int cell_size, int num_bins)
{
    if (images.empty()) return {};
    sd_ctx* ctx = sd_b200::context();
    const std::vector<sd_host_frame> frames = sd_b200::host_frames(images);
    hog_batch::Results res;
    for (size_t i = 0; i < frames.size(); ++i) {
        int w = 0, h = 0, dd = 0;
        if (sd_hog_dense_shape(frames[i].width, frames[i].height, cell_size, num_bins, variant, &w, &h, &dd) != SD_OK)
            throw std::runtime_error("hog_dense: frame " + std::to_string(i) + " (" + std::to_string(frames[i].width) + " x " +
                                     std::to_string(frames[i].height) + ") or the configuration is invalid: frames wider and taller "
                                     "than 3 px and at least half a cell, cell_size 1..32, num_bins 1..16");
        res.add(dd * h, w);
    }
    sd_b200::DeviceBuffer buf;
    const sd_image_batch batch = hog_batch::upload_grey(ctx, frames, buf, "hog_dense upload");
    sd_b200::check(ctx, sd_hog_dense(ctx, &batch, cell_size, num_bins, variant, res.out(), res.offsets(ctx, "hog_dense")), "sd_hog_dense");
    return res.download();
}

// Dense HOG of every frame at every scale, in one batched call on the device (sd_hog_pyramid): level s of a W x H frame is the
// frame resized by cv::resize INTER_LINEAR to floor(W * s + 0.5) x floor(H * s + 0.5), and its features are hog_dense's of that
// level.  Returns, per frame, one Mat per scale as hog_dense returns it (dd * hogH rows of hogW columns), or an empty Mat for
// an empty level (smaller than 4 px or than half a cell).  multichannel: frames keep their channels (8-bit, one channel count;
// 8UC3 is B,G,R as given) and go through sd_hog_pyramid_images, where the channel with the largest gradient votes at each
// pixel; bilinear_orientations (multichannel only): every pixel votes into its two nearest orientation bins.  float_frames
// (multichannel only): the frames are CV_32FC1 or CV_32FC3 and go through sd_hog_pyramid_float, each channel resized by
// cv::resize's float rule, values and range as given.  Throws std::runtime_error for no scales, a scale outside (0, 4], or a
// configuration that sd_hog_pyramid_shape refuses.
inline std::vector<std::vector<cv::Mat>> vl_hog_pyramid(const std::vector<cv::Mat>& images, const std::vector<double>& scales,
                                                        VlHogVariant variant, int cell_size, int num_bins, bool multichannel = false,
                                                        bool bilinear_orientations = false, bool float_frames = false)
{
    if (images.empty()) return {};
    if (scales.empty()) throw std::runtime_error("vl_hog_pyramid: no scales");
    hog_batch::check_window_flags(multichannel, bilinear_orientations, float_frames, "vl_hog_pyramid");
    sd_ctx* ctx = sd_b200::context();
    const int n = static_cast<int>(images.size()), S = static_cast<int>(scales.size());
    hog_batch::Results res;
    for (int i = 0; i < n; ++i)
        for (int s = 0; s < S; ++s) {
            int lw = 0, lh = 0, w = 0, h = 0, dd = 0;
            if (sd_hog_pyramid_shape(images[i].cols, images[i].rows, scales[s], cell_size, num_bins, variant, &lw, &lh, &w, &h, &dd) != SD_OK)
                throw std::runtime_error("vl_hog_pyramid: frame " + std::to_string(i) + " at scale " + std::to_string(scales[s]) +
                                         " or the configuration is invalid: scales in (0, 4], cell_size 1..32, num_bins 1..16");
            res.add(dd * h, w);
        }
    hog_batch::WindowFrames fr;
    hog_batch::upload_window_frames(ctx, images, multichannel, bilinear_orientations, float_frames, fr, "vl_hog_pyramid upload");
    if (multichannel)
        sd_b200::check(ctx, (float_frames ? sd_hog_pyramid_float : sd_hog_pyramid_images)(
                                ctx, &fr.colour, scales.data(), S, cell_size, num_bins, variant, bilinear_orientations ? 1 : 0, res.out(),
                                res.offsets(ctx, "vl_hog_pyramid")),
                       float_frames ? "sd_hog_pyramid_float" : "sd_hog_pyramid_images");
    else
        sd_b200::check(ctx, sd_hog_pyramid(ctx, &fr.grey, scales.data(), S, cell_size, num_bins, variant, res.out(),
                                           res.offsets(ctx, "vl_hog_pyramid")), "sd_hog_pyramid");
    const std::vector<cv::Mat> levels = res.download();
    std::vector<std::vector<cv::Mat>> out;
    for (int i = 0; i < n; ++i) out.emplace_back(levels.begin() + static_cast<size_t>(i) * S, levels.begin() + static_cast<size_t>(i + 1) * S);
    return out;
}

// Scores of a bank of HOG filters over HOG grids, in one batched call on the device (sd_hog_correlate).  maps: grids as
// hog_dense returns them (CV_32FC1, dd * h rows of w columns); filters: Q filters in the same layout, dd * fh rows of fw
// columns each (hog_dense of a template image is one); bias: Q values, or empty for none.  Returns one CV_32FC1 Mat per map of
// Q * oh rows and ow columns, filter q's score map in rows q * oh .. q * oh + oh - 1, with oh = h + 2 pad_y - fh + 1 and
// ow = w + 2 pad_x - fw + 1 (an empty Mat when either is <= 0).  Throws std::runtime_error for maps or filters of the wrong
// shape, and for a configuration that sd_hog_correlate refuses.
inline std::vector<cv::Mat> vl_hog_correlate(const std::vector<cv::Mat>& maps, const std::vector<cv::Mat>& filters, VlHogVariant variant,
                                             int num_bins, const std::vector<float>& bias, int pad_x, int pad_y)
{
    if (maps.empty()) return {};
    sd_ctx* ctx = sd_b200::context();
    const int dd = sd_b200::hog_dimension(variant, num_bins);
    const int Q = static_cast<int>(filters.size());
    if (Q < 1 || dd < 1 || filters[0].rows % dd) throw std::runtime_error("vl_hog_correlate: no filters, or filters not dd * fh rows");
    const int fh = filters[0].rows / dd, fw = filters[0].cols;
    if (!bias.empty() && static_cast<int>(bias.size()) != Q) throw std::runtime_error("vl_hog_correlate: one bias per filter");
    // filters and maps packed on the host, then one upload each
    std::vector<float> hf;
    for (const cv::Mat& f : filters) {
        if (f.type() != CV_32FC1 || f.rows != dd * fh || f.cols != fw) throw std::runtime_error("vl_hog_correlate: filters differ in shape");
        for (int r = 0; r < f.rows; ++r) hf.insert(hf.end(), f.ptr<float>(r), f.ptr<float>(r) + f.cols);
    }
    std::vector<float> hm;
    std::vector<sd_hog_grid> grids;
    hog_batch::Results res;
    for (size_t i = 0; i < maps.size(); ++i) {
        const cv::Mat& m = maps[i];
        if (m.type() != CV_32FC1 || m.rows < dd || m.rows % dd || m.cols < 1)
            throw std::runtime_error("vl_hog_correlate: map " + std::to_string(i) + " is not dd * h rows of w columns");
        const int h = m.rows / dd, w = m.cols;
        const int oh = h + 2 * pad_y - fh + 1, ow = w + 2 * pad_x - fw + 1;
        res.add(Q * oh, ow);
        grids.push_back(sd_hog_grid{w, h, static_cast<int64_t>(hm.size()), res.offset[i]});
        for (int r = 0; r < m.rows; ++r) hm.insert(hm.end(), m.ptr<float>(r), m.ptr<float>(r) + m.cols);
    }
    sd_b200::DeviceBuffer d_maps(hm.size() * sizeof(float)), d_filters(hf.size() * sizeof(float)),
        d_bias(std::max<size_t>(bias.size(), 1) * sizeof(float)), d_grids(grids.size() * sizeof(sd_hog_grid));
    sd_b200::check(ctx, sd_memcpy_h2d(ctx, d_maps.as<float>(), hm.data(), hm.size() * sizeof(float)), "vl_hog_correlate");
    sd_b200::check(ctx, sd_memcpy_h2d(ctx, d_filters.as<float>(), hf.data(), hf.size() * sizeof(float)), "vl_hog_correlate");
    sd_b200::check(ctx, sd_memcpy_h2d(ctx, d_grids.as<sd_hog_grid>(), grids.data(), grids.size() * sizeof(sd_hog_grid)), "vl_hog_correlate");
    if (!bias.empty()) sd_b200::check(ctx, sd_memcpy_h2d(ctx, d_bias.as<float>(), bias.data(), bias.size() * sizeof(float)), "vl_hog_correlate");
    sd_hog_grids g{};
    g.d_features = d_maps.as<float>();
    g.count = static_cast<int32_t>(maps.size());
    g.d_grids = d_grids.as<sd_hog_grid>();
    sd_b200::check(ctx, sd_hog_correlate(ctx, &g, num_bins, variant, d_filters.as<float>(), Q, fw, fh, bias.empty() ? nullptr : d_bias.as<float>(),
                                         pad_x, pad_y, res.out()), "sd_hog_correlate");
    return res.download();
}

// One detection of vl_hog_detect: the box in frame pixels (not clipped to the frame), the score, the filter index q, the level
// (the scale's index) and the score position in that level.
struct hog_detection {
    cv::Rect box;
    float score;
    int filter, level;
    int cell_x, cell_y;
};

inline hog_detection to_hog_detection(const sd_hog_detection& r) { return {cv::Rect(r.x, r.y, r.w, r.h), r.score, r.filter, r.level, r.cell_x, r.cell_y}; }

// A sliding-window detector over image pyramids: vl_hog_pyramid of every frame, vl_hog_correlate of the filter bank on every
// level, then sd_hog_detections over all score maps (the scores above threshold, their boxes in frame pixels, the first
// max_candidates of each frame by score, and greedy non-maximum suppression at IoU overlap over all filters as one class).
// Arguments as vl_hog_pyramid and vl_hog_correlate take them; filters trained with multichannel, bilinear_orientations or
// float_frames are scored with the same.  Returns one list per frame, in the rule's order (include/sd_b200.h); each box is what detect_faces
// takes.  Throws std::runtime_error where those calls or sd_hog_detections refuse.
inline std::vector<std::vector<hog_detection>> vl_hog_detect(const std::vector<cv::Mat>& images, const std::vector<double>& scales,
                                                             const std::vector<cv::Mat>& filters, VlHogVariant variant, int cell_size,
                                                             int num_bins, const std::vector<float>& bias, int pad_x, int pad_y,
                                                             float threshold, double overlap, int max_candidates, int max_detections,
                                                             bool multichannel = false, bool bilinear_orientations = false,
                                                             bool float_frames = false)
{
    if (images.empty()) return {};
    const std::vector<std::vector<cv::Mat>> pyr = vl_hog_pyramid(images, scales, variant, cell_size, num_bins, multichannel, bilinear_orientations,
                                                                 float_frames);
    const int dd = sd_b200::hog_dimension(variant, num_bins);
    const int Q = static_cast<int>(filters.size());
    if (Q < 1 || filters[0].rows % dd) throw std::runtime_error("vl_hog_detect: no filters, or filters not dd * fh rows");
    const int fh = filters[0].rows / dd, fw = filters[0].cols;
    const int n = static_cast<int>(images.size());
    std::vector<cv::Mat> maps;
    std::vector<sd_hog_score_map> descs;
    for (int i = 0; i < n; ++i)
        for (size_t s = 0; s < scales.size(); ++s) {
            if (pyr[i][s].empty()) continue;
            int lw = 0, lh = 0, w = 0, h = 0, d = 0;
            sd_hog_pyramid_shape(images[i].cols, images[i].rows, scales[s], cell_size, num_bins, variant, &lw, &lh, &w, &h, &d);
            maps.push_back(pyr[i][s]);
            descs.push_back(sd_hog_score_map{i, static_cast<int32_t>(s), images[i].cols, images[i].rows, lw, lh, 0, 0, 0});
        }
    // the score maps with scores, packed end to end: a map smaller than the filter has no candidates
    const std::vector<cv::Mat> scores = vl_hog_correlate(maps, filters, variant, num_bins, bias, pad_x, pad_y);
    std::vector<cv::Mat> planes;
    std::vector<sd_hog_score_map> table;
    for (size_t k = 0; k < scores.size(); ++k)
        if (!scores[k].empty()) {
            planes.push_back(scores[k]);
            table.push_back(descs[k]);
            table.back().width = scores[k].cols;
            table.back().height = scores[k].rows / Q;
        }
    sd_ctx* ctx = sd_b200::context();
    sd_b200::DeviceBuffer d_scores, d_table(table.size() * sizeof(sd_hog_score_map));
    const std::vector<int64_t> start = hog_batch::pack_planes(ctx, planes, sizeof(float), d_scores, "vl_hog_detect upload");
    for (size_t k = 0; k < table.size(); ++k) table[k].offset = start[k];
    if (!table.empty())
        sd_b200::check(ctx, sd_memcpy_h2d(ctx, d_table.as<sd_hog_score_map>(), table.data(), table.size() * sizeof(sd_hog_score_map)),
                       "vl_hog_detect upload");
    const size_t slots = static_cast<size_t>(n) * static_cast<size_t>(std::max(max_detections, 1));
    sd_b200::DeviceBuffer d_out(slots * sizeof(sd_hog_detection)), d_count(static_cast<size_t>(n) * sizeof(int32_t));
    sd_b200::check(ctx, sd_hog_detections(ctx, d_scores.as<float>(), d_table.as<sd_hog_score_map>(), static_cast<int>(table.size()), n, Q,
                                          cell_size, fw, fh, pad_x, pad_y, threshold, overlap, max_candidates, max_detections,
                                          d_out.as<sd_hog_detection>(), d_count.as<int32_t>(), nullptr), "sd_hog_detections");
    std::vector<sd_hog_detection> out;
    const std::vector<int32_t> count = hog_batch::download_detections(ctx, d_out, d_count, n, max_detections, out, "vl_hog_detect download");
    std::vector<std::vector<hog_detection>> result(n);
    for (int i = 0; i < n; ++i)
        for (int k = 0; k < count[i]; ++k) result[i].push_back(to_hog_detection(out[static_cast<size_t>(i) * max_detections + k]));
    return result;
}

// A star model for vl_hog_part_detect (include/sd_b200.h, sd_hog_part_model): Q root filters with their bias, and per component
// P part filters scored at twice the root's resolution, in the shell's filter layout (dd * fh rows of fw floats); anchors[q][p]
// = (ax, ay) in part-level cells relative to twice the root window's top-left cell; deformation[q][p] = (w0, w1, w2, w3), a
// displacement (dx, dy) costing w0 dx^2 + w1 dx + w2 dy^2 + w3 dy; the root and part pads; R = max_displacement bounding |dx|
// and |dy|, or, with unbounded, the exact transform of DPM (sd_hog_distance_transform_exact: no bound, w0 > 0 and w2 > 0;
// max_displacement is then ignored).
struct hog_part_model {
    std::vector<cv::Mat> root;
    std::vector<float> bias;
    std::vector<std::vector<cv::Mat>> parts;
    std::vector<std::vector<std::array<int, 2>>> anchors;
    std::vector<std::vector<std::array<float, 4>>> deformation;
    int pad_x = 0, pad_y = 0, part_pad_x = 0, part_pad_y = 0;
    int max_displacement = 4;
    bool unbounded = false;
};

// One part of a detection: its box in frame pixels (empty where it has no placement), its placement (u, v) in part score
// positions ((-1, -1) for none) and its transformed score D at the anchor.
struct hog_part {
    cv::Rect box;
    int u, v;
    float score;
};
struct hog_part_detection {
    hog_detection detection;      // the root box, the star model's score, the component as the filter
    std::vector<hog_part> parts;
};

// A star-model detector over image pyramids: vl_hog_pyramid over the root scales and their doubles (a scale present in both is
// computed once; root scales must be in (0, 2]), vl_hog_correlate of the roots and of all Q * P parts, then on the device
// sd_hog_distance_transform, sd_hog_part_scores, sd_hog_detections (the root's filter size and pad, all components as one
// class) and sd_hog_part_placements; an unbounded model takes sd_hog_distance_transform_exact and sd_hog_part_placements_mapped.  multichannel, bilinear_orientations and float_frames as vl_hog_pyramid takes them: a model of colour
// HOG is scored with the values it was built for.  Returns one list per frame, in the rule's order; each detection's box is
// what detect_faces takes.  Throws std::runtime_error for a model of inconsistent shapes and where those calls refuse.
inline std::vector<std::vector<hog_part_detection>> vl_hog_part_detect(const std::vector<cv::Mat>& images, const std::vector<double>& scales,
                                                                       const hog_part_model& model, VlHogVariant variant, int cell_size,
                                                                       int num_bins, float threshold, double overlap, int max_candidates,
                                                                       int max_detections, bool multichannel = false,
                                                                       bool bilinear_orientations = false, bool float_frames = false)
{
    if (images.empty()) return {};
    const int dd = sd_b200::hog_dimension(variant, num_bins);
    const int Q = static_cast<int>(model.root.size());
    if (Q < 1 || model.parts.size() != model.root.size() || model.parts[0].empty() || model.anchors.size() != model.root.size() ||
        model.deformation.size() != model.root.size() || model.root[0].rows % dd || model.parts[0][0].rows % dd)
        throw std::runtime_error("vl_hog_part_detect: the model needs Q roots, parts, anchors and deformations of dd * side rows");
    const int P = static_cast<int>(model.parts[0].size());
    std::vector<cv::Mat> part_filters;
    std::vector<int32_t> anchors;
    std::vector<float> deformation;
    for (int q = 0; q < Q; ++q) {
        if (static_cast<int>(model.parts[q].size()) != P || static_cast<int>(model.anchors[q].size()) != P ||
            static_cast<int>(model.deformation[q].size()) != P)
            throw std::runtime_error("vl_hog_part_detect: every component needs P parts, anchors and deformations");
        for (int p = 0; p < P; ++p) {
            part_filters.push_back(model.parts[q][p]);
            anchors.insert(anchors.end(), model.anchors[q][p].begin(), model.anchors[q][p].end());
            deformation.insert(deformation.end(), model.deformation[q][p].begin(), model.deformation[q][p].end());
        }
    }
    std::vector<double> every;
    for (double s : scales) {
        if (!(s > 0 && s <= 2)) throw std::runtime_error("vl_hog_part_detect: root scales must be in (0, 2]");
        if (std::find(every.begin(), every.end(), s) == every.end()) every.push_back(s);
    }
    for (double s : scales)
        if (std::find(every.begin(), every.end(), 2 * s) == every.end()) every.push_back(2 * s);
    auto index = [&every](double s) { return static_cast<int>(std::find(every.begin(), every.end(), s) - every.begin()); };
    const std::vector<std::vector<cv::Mat>> pyr = vl_hog_pyramid(images, every, variant, cell_size, num_bins, multichannel, bilinear_orientations,
                                                                 float_frames);
    const int n = static_cast<int>(images.size());
    std::vector<cv::Mat> root_maps;
    std::vector<std::array<int, 2>> root_of;   // (frame, scale index)
    for (int i = 0; i < n; ++i)
        for (size_t s = 0; s < scales.size(); ++s)
            if (!pyr[i][index(scales[s])].empty()) {
                root_maps.push_back(pyr[i][index(scales[s])]);
                root_of.push_back({{i, static_cast<int>(s)}});
            }
    const std::vector<cv::Mat> roots = vl_hog_correlate(root_maps, model.root, variant, num_bins, model.bias, model.pad_x, model.pad_y);
    // the part levels of the root maps with scores, each once
    std::vector<std::array<int, 2>> plevels;
    std::vector<cv::Mat> part_maps;
    std::vector<int> part_of(roots.size(), -1);
    for (size_t k = 0; k < roots.size(); ++k) {
        if (roots[k].empty()) continue;
        const std::array<int, 2> key{{root_of[k][0], index(2 * scales[root_of[k][1]])}};
        if (pyr[key[0]][key[1]].empty()) continue;
        auto it = std::find(plevels.begin(), plevels.end(), key);
        if (it == plevels.end()) {
            plevels.push_back(key);
            part_maps.push_back(pyr[key[0]][key[1]]);
            it = plevels.end() - 1;
        }
        part_of[k] = static_cast<int>(it - plevels.begin());
    }
    const std::vector<cv::Mat> part_scores =
        part_maps.empty() ? std::vector<cv::Mat>() : vl_hog_correlate(part_maps, part_filters, variant, num_bins, {}, model.part_pad_x, model.part_pad_y);
    sd_ctx* ctx = sd_b200::context();
    // the part score maps on the device, their transform at the same offsets
    sd_b200::DeviceBuffer d_raw, d_values, d_place, d_grids;
    std::vector<cv::Mat> pplanes;
    std::vector<int> pslot(part_scores.size(), -1);   // each part level's place among the maps with scores
    for (size_t k = 0; k < part_scores.size(); ++k)
        if (!part_scores[k].empty()) {
            pslot[k] = static_cast<int>(pplanes.size());
            pplanes.push_back(part_scores[k]);
        }
    const std::vector<int64_t> pstart = hog_batch::pack_planes(ctx, pplanes, sizeof(float), d_raw, "vl_hog_part_detect upload");
    std::vector<sd_hog_grid> grids;
    int64_t raw_floats = 0;
    for (size_t j = 0; j < pplanes.size(); ++j) {
        grids.push_back(sd_hog_grid{pplanes[j].cols, pplanes[j].rows / (Q * P), pstart[j], pstart[j]});
        raw_floats += static_cast<int64_t>(pplanes[j].rows) * pplanes[j].cols;
    }
    d_raw.allocate(static_cast<size_t>(std::max<int64_t>(raw_floats, 1)) * sizeof(float));
    d_values.allocate(static_cast<size_t>(std::max<int64_t>(raw_floats, 1)) * sizeof(float));
    if (model.unbounded) d_place.allocate(static_cast<size_t>(std::max<int64_t>(raw_floats, 1)) * 2 * sizeof(int32_t));
    if (!grids.empty()) {
        d_grids.allocate(grids.size() * sizeof(sd_hog_grid));
        sd_b200::check(ctx, sd_memcpy_h2d(ctx, d_grids.as<sd_hog_grid>(), grids.data(), grids.size() * sizeof(sd_hog_grid)), "vl_hog_part_detect upload");
        sd_hog_grids g{};
        g.d_features = d_raw.as<float>();
        g.count = static_cast<int32_t>(grids.size());
        g.d_grids = d_grids.as<sd_hog_grid>();
        if (model.unbounded)
            sd_b200::check(ctx, sd_hog_distance_transform_exact(ctx, &g, Q * P, deformation.data(), d_values.as<float>(), d_place.as<int32_t>()),
                           "sd_hog_distance_transform_exact");
        else
            sd_b200::check(ctx, sd_hog_distance_transform(ctx, &g, Q * P, deformation.data(), model.max_displacement, d_values.as<float>(), nullptr),
                           "sd_hog_distance_transform");
    }
    // the root scores and the star model's scores at the same offsets
    std::vector<cv::Mat> planes;
    std::vector<size_t> kept;
    for (size_t k = 0; k < roots.size(); ++k)
        if (!roots[k].empty()) {
            planes.push_back(roots[k]);
            kept.push_back(k);
        }
    sd_b200::DeviceBuffer d_root, d_total, d_table, d_maps, d_anchors(anchors.size() * sizeof(int32_t));
    const std::vector<int64_t> rstart = hog_batch::pack_planes(ctx, planes, sizeof(float), d_root, "vl_hog_part_detect upload");
    int64_t root_floats = 1;
    for (const cv::Mat& m : planes) root_floats += static_cast<int64_t>(m.rows) * m.cols;
    d_total.allocate(static_cast<size_t>(root_floats) * sizeof(float));
    sd_b200::check(ctx, sd_memcpy_h2d(ctx, d_anchors.as<int32_t>(), anchors.data(), anchors.size() * sizeof(int32_t)), "vl_hog_part_detect upload");
    std::vector<sd_hog_part_map> table;
    std::vector<sd_hog_score_map> maps;
    for (size_t j = 0; j < kept.size(); ++j) {
        const size_t k = kept[j];
        const int i = root_of[k][0], s = root_of[k][1];
        int lw = 0, lh = 0, w = 0, h = 0, d = 0, plw = 0, plh = 0;
        sd_hog_pyramid_shape(images[i].cols, images[i].rows, scales[s], cell_size, num_bins, variant, &lw, &lh, &w, &h, &d);
        sd_hog_pyramid_shape(images[i].cols, images[i].rows, 2 * scales[s], cell_size, num_bins, variant, &plw, &plh, &w, &h, &d);
        const int oh = roots[k].rows / Q, ow = roots[k].cols;
        int pw = 0, ph = 0;
        int64_t po = 0;
        if (part_of[k] >= 0 && pslot[part_of[k]] >= 0) {
            const int j = pslot[part_of[k]];
            pw = pplanes[j].cols;
            ph = pplanes[j].rows / (Q * P);
            po = pstart[j];
        }
        table.push_back(sd_hog_part_map{i, s, images[i].cols, images[i].rows, plw, plh, ow, oh, pw, ph, rstart[j], po, rstart[j]});
        maps.push_back(sd_hog_score_map{i, s, images[i].cols, images[i].rows, lw, lh, ow, oh, rstart[j]});
    }
    sd_hog_part_model m{};
    m.num_components = Q;
    m.num_parts = P;
    m.filter_w = model.root[0].cols;
    m.filter_h = model.root[0].rows / dd;
    m.part_w = model.parts[0][0].cols;
    m.part_h = model.parts[0][0].rows / dd;
    m.pad_x = model.pad_x; m.pad_y = model.pad_y;
    m.part_pad_x = model.part_pad_x; m.part_pad_y = model.part_pad_y;
    m.d_anchors = d_anchors.as<int32_t>();
    const int nm = static_cast<int>(table.size());
    if (nm > 0) {
        d_table.allocate(table.size() * sizeof(sd_hog_part_map));
        d_maps.allocate(maps.size() * sizeof(sd_hog_score_map));
        sd_b200::check(ctx, sd_memcpy_h2d(ctx, d_table.as<sd_hog_part_map>(), table.data(), table.size() * sizeof(sd_hog_part_map)), "vl_hog_part_detect upload");
        sd_b200::check(ctx, sd_memcpy_h2d(ctx, d_maps.as<sd_hog_score_map>(), maps.data(), maps.size() * sizeof(sd_hog_score_map)), "vl_hog_part_detect upload");
        sd_b200::check(ctx, sd_hog_part_scores(ctx, d_root.as<float>(), d_values.as<float>(), d_table.as<sd_hog_part_map>(), nm, &m, d_total.as<float>()),
                       "sd_hog_part_scores");
    }
    const size_t slots = static_cast<size_t>(n) * static_cast<size_t>(std::max(max_detections, 1));
    sd_b200::DeviceBuffer d_out(slots * sizeof(sd_hog_detection)), d_count(static_cast<size_t>(n) * sizeof(int32_t)),
        d_parts(slots * P * sizeof(sd_hog_part_placement));
    sd_b200::check(ctx, sd_hog_detections(ctx, d_total.as<float>(), d_maps.as<sd_hog_score_map>(), nm, n, Q, cell_size, m.filter_w, m.filter_h,
                                          m.pad_x, m.pad_y, threshold, overlap, max_candidates, max_detections, d_out.as<sd_hog_detection>(),
                                          d_count.as<int32_t>(), nullptr), "sd_hog_detections");
    if (model.unbounded)
        sd_b200::check(ctx, sd_hog_part_placements_mapped(ctx, d_values.as<float>(), d_place.as<int32_t>(), d_table.as<sd_hog_part_map>(), nm, &m,
                                                          cell_size, d_out.as<sd_hog_detection>(), d_count.as<int32_t>(), n, max_detections,
                                                          d_parts.as<sd_hog_part_placement>()), "sd_hog_part_placements_mapped");
    else
        sd_b200::check(ctx, sd_hog_part_placements(ctx, d_raw.as<float>(), d_table.as<sd_hog_part_map>(), nm, &m, deformation.data(),
                                                   model.max_displacement, cell_size, d_out.as<sd_hog_detection>(), d_count.as<int32_t>(), n,
                                                   max_detections, d_parts.as<sd_hog_part_placement>()), "sd_hog_part_placements");
    std::vector<sd_hog_part_placement> parts(slots * P);
    sd_b200::check(ctx, sd_memcpy_d2h(ctx, parts.data(), d_parts.as<void>(), parts.size() * sizeof(sd_hog_part_placement)), "vl_hog_part_detect download");
    std::vector<sd_hog_detection> out;
    const std::vector<int32_t> count = hog_batch::download_detections(ctx, d_out, d_count, n, max_detections, out, "vl_hog_part_detect download");
    std::vector<std::vector<hog_part_detection>> result(n);
    for (int i = 0; i < n; ++i)
        for (int k = 0; k < count[i]; ++k) {
            const size_t slot = static_cast<size_t>(i) * max_detections + k;
            hog_part_detection det{to_hog_detection(out[slot]), {}};
            for (int p = 0; p < P; ++p) {
                const sd_hog_part_placement& pp = parts[slot * P + p];
                det.parts.push_back(hog_part{cv::Rect(pp.x, pp.y, pp.w, pp.h), pp.u, pp.v, pp.term});
            }
            result[i].push_back(det);
        }
    return result;
}

// A HOG filter trained by train_hog_filter: the filter in the shell's filter layout (dd * fh rows of fw floats, as vl_hog_correlate
// and vl_hog_detect take filters), its bias, one report per round (sd_hog_train_report; rounds after an early stop are zero) and
// the negative cache in slot order (grid = frame * scales.size() + level).
struct hog_filter {
    cv::Mat filter;
    float bias;
    std::vector<sd_hog_train_report> rounds;
    std::vector<sd_hog_window> negatives;
};

// Trains a HOG filter for vl_hog_detect with a squared-hinge SVM and hard-negative mining (sd_hog_train_filter; the rule is in
// include/sd_b200.h).  images: 8UC1 or 8UC3 (B,G,R) frames of any sizes; box k, boxes[k] in frame pixels, belongs to frame
// box_frame[k]; frames without a box are pure negative frames.  multichannel, bilinear_orientations and float_frames as
// vl_hog_pyramid takes them (sd_hog_train_filter_images, with float_frames sd_hog_train_filter_float on CV_32FC1 or CV_32FC3
// frames); vl_hog_detect scores the filter with the same values.  Throws std::runtime_error where sd_hog_train_filter refuses.
inline hog_filter train_hog_filter(const std::vector<cv::Mat>& images, const std::vector<int>& box_frame, const std::vector<cv::Rect>& boxes,
                                   const std::vector<double>& scales, VlHogVariant variant, int cell_size, int num_bins, int filter_w,
                                   int filter_h, int pad_x, int pad_y, const sd_hog_train_param& params, bool multichannel = false,
                                   bool bilinear_orientations = false, bool float_frames = false)
{
    if (images.empty()) throw std::runtime_error("train_hog_filter: no frames");
    if (box_frame.size() != boxes.size()) throw std::runtime_error("train_hog_filter: box_frame and boxes differ in length");
    if (params.rounds < 0 || params.max_negatives < 1) throw std::runtime_error("train_hog_filter: rounds < 0 or max_negatives < 1");
    hog_batch::check_window_flags(multichannel, bilinear_orientations, float_frames, "train_hog_filter");
    sd_ctx* ctx = sd_b200::context();
    hog_batch::WindowFrames fr;
    hog_batch::upload_window_frames(ctx, images, multichannel, bilinear_orientations, float_frames, fr, "train_hog_filter upload");
    std::vector<sd_hog_box> hb;
    for (size_t k = 0; k < boxes.size(); ++k)
        hb.push_back(sd_hog_box{box_frame[k], boxes[k].x, boxes[k].y, boxes[k].width, boxes[k].height});
    const int dd = sd_b200::hog_dimension(variant, num_bins);
    sd_b200::DeviceBuffer d_filter(static_cast<size_t>(dd) * filter_h * filter_w * sizeof(float));
    hog_filter out;
    out.rounds.resize(static_cast<size_t>(params.rounds) + 1);
    out.negatives.resize(static_cast<size_t>(params.max_negatives));
    int num_negatives = 0;
    const int nb = static_cast<int>(hb.size()), S = static_cast<int>(scales.size());
    if (multichannel)
        sd_b200::check(ctx, (float_frames ? sd_hog_train_filter_float : sd_hog_train_filter_images)(
                                ctx, &fr.colour, bilinear_orientations ? 1 : 0, hb.data(), nb, scales.data(), S, cell_size, num_bins, variant,
                                filter_w, filter_h, pad_x, pad_y, &params, d_filter.as<float>(), &out.bias, out.rounds.data(),
                                out.negatives.data(), &num_negatives),
                       float_frames ? "sd_hog_train_filter_float" : "sd_hog_train_filter_images");
    else
        sd_b200::check(ctx, sd_hog_train_filter(ctx, &fr.grey, hb.data(), nb, scales.data(), S, cell_size, num_bins, variant, filter_w, filter_h,
                                                pad_x, pad_y, &params, d_filter.as<float>(), &out.bias, out.rounds.data(),
                                                out.negatives.data(), &num_negatives), "sd_hog_train_filter");
    out.negatives.resize(static_cast<size_t>(num_negatives));
    out.filter = sd_b200::download(d_filter.as<float>(), dd * filter_h, filter_w, filter_w);
    return out;
}

// A HOG filter's score at each box (sd_hog_box_scores; the rule is in include/sd_b200.h): box k, boxes[k] in pixels of frame
// box_frame[k], with one cell of context on every side, zero outside the frame, is resized to (fw + 2) x (fh + 2) cells of
// cell_size px and scored by the filter (dd * fh x fw CV_32FC1, hog_filter::filter's layout) and bias at each of the 3 x 3
// positions; the box's score is the largest (a NaN never is).  images: 8UC1 or 8UC3 (B,G,R) frames of any sizes, uploaded as
// grey.  multichannel, bilinear_orientations and float_frames as vl_hog_pyramid takes them (sd_hog_box_scores_images): a filter
// trained on colour or float frames scores the boxes on the frames as given (8UC1 / 8UC3, or CV_32FC1 / CV_32FC3 with
// float_frames).  Throws std::runtime_error where sd_hog_box_scores or sd_hog_box_scores_images refuses.
inline std::vector<float> hog_box_scores(const std::vector<cv::Mat>& images, const std::vector<int>& box_frame, const std::vector<cv::Rect>& boxes,
                                         const cv::Mat& filter, float bias, VlHogVariant variant, int cell_size, int num_bins,
                                         bool multichannel = false, bool bilinear_orientations = false, bool float_frames = false)
{
    hog_batch::check_window_flags(multichannel, bilinear_orientations, float_frames, "hog_box_scores");
    if (images.empty()) throw std::runtime_error("hog_box_scores: no frames");
    if (box_frame.size() != boxes.size()) throw std::runtime_error("hog_box_scores: box_frame and boxes differ in length");
    const int dd = sd_b200::hog_dimension(variant, num_bins);
    if (filter.type() != CV_32FC1 || filter.empty() || filter.rows % dd != 0)
        throw std::runtime_error("hog_box_scores: the filter must be a CV_32FC1 Mat of dd * fh rows and fw columns");
    const int n = static_cast<int>(boxes.size());
    std::vector<float> out(n);
    if (n == 0) return out;
    sd_ctx* ctx = sd_b200::context();
    sd_b200::DeviceBuffer d_filter, d_boxes(static_cast<size_t>(n) * 5 * sizeof(int32_t)), d_scores(static_cast<size_t>(n) * sizeof(float));
    hog_batch::WindowFrames fr;
    hog_batch::upload_window_frames(ctx, images, multichannel, bilinear_orientations, float_frames, fr, "hog_box_scores upload");
    sd_b200::upload(filter, d_filter, filter.cols);
    std::vector<int32_t> table(static_cast<size_t>(n) * 5);   // [frame indices | boxes]
    for (int k = 0; k < n; ++k) {
        table[k] = box_frame[k];
        const int32_t b[4] = {boxes[k].x, boxes[k].y, boxes[k].width, boxes[k].height};
        std::memcpy(&table[n + 4 * k], b, sizeof(b));
    }
    sd_b200::check(ctx, sd_memcpy_h2d(ctx, d_boxes.as<int32_t>(), table.data(), table.size() * sizeof(int32_t)), "hog_box_scores");
    if (multichannel)
        sd_b200::check(ctx, sd_hog_box_scores_images(ctx, &fr.colour, bilinear_orientations ? 1 : 0, d_boxes.as<int32_t>(), d_boxes.as<int32_t>() + n,
                                                     n, d_filter.as<float>(), filter.cols, filter.rows / dd, bias, cell_size, num_bins, variant,
                                                     d_scores.as<float>()), "sd_hog_box_scores_images");
    else
        sd_b200::check(ctx, sd_hog_box_scores(ctx, &fr.grey, d_boxes.as<int32_t>(), d_boxes.as<int32_t>() + n, n, d_filter.as<float>(), filter.cols,
                                              filter.rows / dd, bias, cell_size, num_bins, variant, d_scores.as<float>()), "sd_hog_box_scores");
    sd_b200::check(ctx, sd_memcpy_d2h(ctx, out.data(), d_scores.as<float>(), out.size() * sizeof(float)), "hog_box_scores");
    sd_b200::check(ctx, sd_sync(ctx), "hog_box_scores");
    return out;
}

// VLFeat HOG of whole frames of one or more channels, 8-bit or float (vl_hog_new(variant, num_bins),
// vl_hog_set_use_bilinear_orientation_assignments(bilinear_orientations), vl_hog_put_image(frame, channels, cell_size),
// vl_hog_extract), in one batched call on the device (sd_hog_dense_images).  Each frame is the list of its channel planes --
// what cv::split gives, VLFeat's planar layout -- all CV_8UC1 or all CV_32FC1, of one size per frame; every frame has the same
// number of planes and the same type.  Channels are used as given: at each pixel the one with the largest gradient wins.
// Returns what rcr::hog_dense returns: one CV_32FC1 Mat per frame with dd * hogH rows and hogW columns.  Throws
// std::runtime_error for frames or a configuration that sd_hog_dense_images refuses.
inline std::vector<cv::Mat> vl_hog(const std::vector<std::vector<cv::Mat>>& frames, VlHogVariant variant, int cell_size, int num_bins,
                                   bool bilinear_orientations = false)
{
    if (frames.empty()) return {};
    const int n = static_cast<int>(frames.size());
    const int channels = static_cast<int>(frames[0].size());
    if (channels < 1 || channels > 16) throw std::runtime_error("vl_hog: frames must have 1..16 channel planes");
    const int type = frames[0][0].type();
    if (type != CV_8UC1 && type != CV_32FC1) throw std::runtime_error("vl_hog: channel planes must be CV_8UC1 or CV_32FC1");
    std::vector<sd_hog_image> desc(n);
    std::vector<cv::Mat> planes;
    hog_batch::Results res;
    for (int i = 0; i < n; ++i) {
        const std::vector<cv::Mat>& f = frames[i];
        if (static_cast<int>(f.size()) != channels) throw std::runtime_error("vl_hog: frame " + std::to_string(i) + " has a different number of planes");
        for (const cv::Mat& p : f)
            if (p.type() != type || p.cols != f[0].cols || p.rows != f[0].rows)
                throw std::runtime_error("vl_hog: the planes of frame " + std::to_string(i) + " differ in type or size from the first frame's");
        const int W = f[0].cols, H = f[0].rows;
        int w = 0, h = 0, dd = 0;
        if (sd_hog_dense_shape(W, H, cell_size, num_bins, variant, &w, &h, &dd) != SD_OK)
            throw std::runtime_error("vl_hog: frame " + std::to_string(i) + " (" + std::to_string(W) + " x " + std::to_string(H) +
                                     ") or the configuration is invalid: frames wider and taller than 3 px and at least half a cell, "
                                     "cell_size 1..32, num_bins 1..16");
        desc[i] = sd_hog_image{W, H, 0, W, 1, static_cast<int64_t>(W) * H};   // offset: where the planes are packed
        planes.insert(planes.end(), f.begin(), f.end());
        res.add(dd * h, w);
    }
    sd_ctx* ctx = sd_b200::context();
    sd_b200::DeviceBuffer buf, d_desc(static_cast<size_t>(n) * sizeof(sd_hog_image));
    const std::vector<int64_t> start = hog_batch::pack_planes(ctx, planes, type == CV_8UC1 ? 1 : 4, buf, "vl_hog upload");
    for (int i = 0; i < n; ++i) desc[i].offset = start[static_cast<size_t>(i) * channels];
    sd_b200::check(ctx, sd_memcpy_h2d(ctx, d_desc.as<sd_hog_image>(), desc.data(), static_cast<size_t>(n) * sizeof(sd_hog_image)), "vl_hog upload");
    sd_hog_images images{};
    images.d_data = buf.as<void>();
    images.dtype = type == CV_8UC1 ? SD_HOG_U8 : SD_HOG_F32;
    images.channels = channels;
    images.count = n;
    images.d_frames = d_desc.as<sd_hog_image>();
    sd_b200::check(ctx, sd_hog_dense_images(ctx, &images, cell_size, num_bins, variant, bilinear_orientations ? 1 : 0, res.out(),
                                            res.offsets(ctx, "vl_hog")), "sd_hog_dense_images");
    return res.download();
}

// VLFeat HOG of gradient fields the caller computed (vl_hog_new(variant, num_bins),
// vl_hog_set_use_bilinear_orientation_assignments(bilinear_orientations), vl_hog_put_polar_field(modulus, angle, directed,
// cell_size), vl_hog_extract), in one batched call on the device (sd_hog_dense_polar): e.g. the gradient of another operator, or
// the magnitude and direction of an optical flow.  modulus[i] and angle[i] are CV_32FC1 planes of one size (row steps allowed);
// fields may differ in size.  Angles in radians, taken modulo 2 pi (directed) or pi; every pixel votes, the border included,
// except where the modulus is <= 0 or the angle is not finite.  Returns what rcr::vl_hog returns: one CV_32FC1 Mat per field with
// dd * hogH rows and hogW columns.  Throws std::runtime_error for pairs of different sizes, other types, or fields or a
// configuration that sd_hog_dense_polar refuses.
inline std::vector<cv::Mat> vl_hog_polar(const std::vector<cv::Mat>& modulus, const std::vector<cv::Mat>& angle, VlHogVariant variant,
                                         int cell_size, int num_bins, bool directed = true, bool bilinear_orientations = false)
{
    if (modulus.size() != angle.size()) throw std::runtime_error("vl_hog_polar: modulus and angle must hold the same number of fields");
    if (modulus.empty()) return {};
    const int n = static_cast<int>(modulus.size());
    std::vector<sd_hog_image> desc(n);
    hog_batch::Results res;
    for (int i = 0; i < n; ++i) {
        const cv::Mat& m = modulus[i];
        const cv::Mat& a = angle[i];
        if (m.type() != CV_32FC1 || a.type() != CV_32FC1) throw std::runtime_error("vl_hog_polar: fields must be CV_32FC1");
        if (m.cols != a.cols || m.rows != a.rows)
            throw std::runtime_error("vl_hog_polar: the modulus and angle of field " + std::to_string(i) + " differ in size");
        const int W = m.cols, H = m.rows;
        int w = 0, h = 0, dd = 0;
        if (sd_hog_dense_shape(W, H, cell_size, num_bins, variant, &w, &h, &dd) != SD_OK)
            throw std::runtime_error("vl_hog_polar: field " + std::to_string(i) + " (" + std::to_string(W) + " x " + std::to_string(H) +
                                     ") or the configuration is invalid: fields wider and taller than 3 px and at least half a cell, "
                                     "cell_size 1..32, num_bins 1..16");
        desc[i] = sd_hog_image{W, H, 0, W, 1, 0};   // offset: where the field is packed
        res.add(dd * h, w);
    }
    sd_ctx* ctx = sd_b200::context();
    sd_b200::DeviceBuffer d_mod, d_ang, d_desc(static_cast<size_t>(n) * sizeof(sd_hog_image));
    const std::vector<int64_t> start = hog_batch::pack_planes(ctx, modulus, sizeof(float), d_mod, "vl_hog_polar upload");
    hog_batch::pack_planes(ctx, angle, sizeof(float), d_ang, "vl_hog_polar upload");   // the same starts: each pair is one size
    for (int i = 0; i < n; ++i) desc[i].offset = start[i];
    sd_b200::check(ctx, sd_memcpy_h2d(ctx, d_desc.as<sd_hog_image>(), desc.data(), static_cast<size_t>(n) * sizeof(sd_hog_image)), "vl_hog_polar upload");
    sd_hog_polar_fields fields{};
    fields.d_modulus = d_mod.as<float>();
    fields.d_angle = d_ang.as<float>();
    fields.count = n;
    fields.d_frames = d_desc.as<sd_hog_image>();
    sd_b200::check(ctx, sd_hog_dense_polar(ctx, &fields, cell_size, num_bins, variant, directed ? 1 : 0, bilinear_orientations ? 1 : 0,
                                           res.out(), res.offsets(ctx, "vl_hog_polar")), "sd_hog_dense_polar");
    return res.download();
}

}  // namespace rcr
