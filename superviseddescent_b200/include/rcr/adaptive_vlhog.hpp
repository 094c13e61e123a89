// H100 drop-in for include/rcr/adaptive_vlhog.hpp: HoGParam (:41-60) and the projection functor
// HogTransform (:70-195).  The functor keeps the reference's constructor and call signature
//     cv::Mat operator()(cv::Mat parameters, size_t regressorLevel, int trainingIndex = 0)
// (one sample, used by predict(), superviseddescent.hpp:332) and exposes its device images, eyes and per-level
// HOG parameters, with which the optimiser projects ALL samples of a level on the device (sd_train_level, sd_apply_level).
// Each distinct image is held once: uploaded to HBM on first use, or kept in host memory when it does not fit; crop / resize /
// HOG run in sd_hog_batch (sm_90a).
#pragma once

#include <cstring>
#include <map>
#include <memory>
#include <string>
#include <tuple>
#include <vector>

#include "rcr/helpers.hpp"
#include "sd_b200/device.hpp"

typedef enum { VlHogVariantDalalTriggs = 0, VlHogVariantUoctti = 1 } VlHogVariant;   // hog.h:70-72

namespace rcr {

struct HoGParam {
    VlHogVariant vlhog_variant;
    int num_cells;
    int cell_size;
    int num_bins;
    float relative_patch_size;
    sd_hog_param c() const { sd_hog_param p; p.variant = vlhog_variant; p.num_cells = num_cells; p.cell_size = cell_size; p.num_bins = num_bins; p.relative_patch_size = relative_patch_size; return p; }
};

class HogTransform {
public:
    // Do not call with `images` that are temporaries (the reference holds a const&, adaptive_vlhog.hpp:188).
    HogTransform(const std::vector<cv::Mat>& images, std::vector<HoGParam> hog_params, std::vector<std::string> modelLandmarksList,
                 std::vector<std::string> rightEyeIdentifiers, std::vector<std::string> leftEyeIdentifiers)
        : images(images), hog_params(hog_params), modelLandmarksList(modelLandmarksList), rightEyeIdentifiers(rightEyeIdentifiers),
          leftEyeIdentifiers(leftEyeIdentifiers), dev(std::make_shared<DeviceImages>()) {}

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
        const int32_t idx = trainingIndex >= 0 && trainingIndex < static_cast<int>(dev->frame_of.size()) ? dev->frame_of[trainingIndex] : -1;
        sd_b200::check(ctx, sd_memcpy_h2d(ctx, didx.as<int32_t>(), &idx, sizeof(idx)), "HogTransform");
        const sd_normalisation nrm = eyes();
        const sd_hog_param p = hog_params[regressorLevel].c();
        sd_b200::check(ctx, sd_hog_batch(ctx, &batch, didx.as<int32_t>(), dx.as<float>(), parameters.cols, 1, static_cast<int>(modelLandmarksList.size()),
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
    struct DeviceImages {
        std::vector<sd_host_frame> frames;   // the distinct frames (on the host route: where the levels read them)
        std::vector<int32_t> frame_of;        // images[i] -> distinct frame
        sd_b200::DeviceBuffer index;          // frame_of on the device
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
        dev->index.allocate(all.size() * sizeof(int32_t));
        sd_b200::check(ctx, sd_memcpy_h2d(ctx, dev->index.as<int32_t>(), dev->frame_of.data(), all.size() * sizeof(int32_t)), "HogTransform upload");
        sd_b200::check(ctx, sd_sync(ctx), "HogTransform upload");
        size_t free_bytes = 0, total = 0;
        sd_b200::check(ctx, sd_device_memory(ctx, &free_bytes, &total), "sd_device_memory");
        const int n = static_cast<int>(frames.size());
        if (static_cast<double>(grey) <= device_frame_share() * static_cast<double>(free_bytes)) {
            size_t bytes = 0;
            sd_b200::check(ctx, sd_upload_frames(ctx, frames.data(), n, nullptr, &bytes, nullptr), "HogTransform upload");
            dev->buf.allocate(bytes);
            sd_b200::check(ctx, sd_upload_frames(ctx, frames.data(), n, dev->buf.as<void>(), &bytes, &dev->batch), "HogTransform upload");
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
    std::shared_ptr<DeviceImages> dev;   // shared between the copies the optimiser makes of this functor
};

}  // namespace rcr
