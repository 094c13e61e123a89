// H100 drop-in for include/rcr/adaptive_vlhog.hpp: HoGParam (:41-60) and the projection functor
// HogTransform (:70-195).  The functor keeps the reference's constructor and call signature
//     cv::Mat operator()(cv::Mat parameters, size_t regressorLevel, int trainingIndex = 0)
// (one sample, used by predict(), superviseddescent.hpp:332) and exposes its device images, eyes and per-level
// HOG parameters, with which the optimiser projects ALL samples of a level on the device (sd_train_level,
// sd_apply_level).  The images are uploaded to HBM once, on first use; crop / resize / HOG run in sd_hog_batch (sm_90a).
#pragma once

#include <memory>
#include <string>
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
        ensure_uploaded();
        const int D = feature_length(regressorLevel);
        sd_b200::DeviceBuffer dx, dA(static_cast<size_t>(D) * sizeof(float)), didx(sizeof(int32_t));
        sd_b200::upload(parameters, dx, parameters.cols);
        const int32_t idx = trainingIndex;
        sd_b200::check(ctx, sd_memcpy_h2d(ctx, didx.as<int32_t>(), &idx, sizeof(idx)), "HogTransform");
        launch(dx.as<float>(), parameters.cols, 1, regressorLevel, dA.as<float>(), D, didx.as<int32_t>());
        return sd_b200::download(dA.as<float>(), 1, D, D);
    }

    // What the optimiser's device route hands to sd_train_level / sd_apply_level: the images resident on the device (uploaded
    // on first use; sample i reads image i), the eye landmarks (eyes()) and the HOG parameters of a level.
    const sd_image_batch& device_batch()
    {
        ensure_uploaded();
        return dev->batch;
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
        sd_b200::DeviceBuffer buf;
        sd_image_batch batch{};
        bool ready = false;
    };

    // frames of any sizes (the reference's std::vector<cv::Mat>), grey or colour: colour is converted once here, where the
    // reference converts it in every call (adaptive_vlhog.hpp:114-120)
    void ensure_uploaded()
    {
        if (dev->ready) return;
        if (images.empty()) throw std::runtime_error("HogTransform: no images");
        sd_ctx* ctx = sd_b200::context();
        const std::vector<sd_host_frame> frames = sd_b200::host_frames(images);
        const int n = static_cast<int>(frames.size());
        size_t bytes = 0;
        sd_b200::check(ctx, sd_upload_frames(ctx, frames.data(), n, nullptr, &bytes, nullptr), "HogTransform upload");
        dev->buf.allocate(bytes);
        sd_b200::check(ctx, sd_upload_frames(ctx, frames.data(), n, dev->buf.as<void>(), &bytes, &dev->batch), "HogTransform upload");
        dev->ready = true;
    }

    void launch(const float* d_x, int64_t ldx, int n, size_t level, float* d_A, int64_t ld, const int32_t* d_index)
    {
        sd_ctx* ctx = sd_b200::context();
        const sd_normalisation nrm = eyes();
        const sd_hog_param p = hog_params[level].c();
        sd_b200::check(ctx, sd_hog_batch(ctx, &dev->batch, d_index, d_x, ldx, n, static_cast<int>(modelLandmarksList.size()), &nrm, &p, d_A, ld), "sd_hog_batch");
    }

    const std::vector<cv::Mat>& images;
    std::vector<HoGParam> hog_params;
    std::vector<std::string> modelLandmarksList;
    std::vector<std::string> rightEyeIdentifiers;
    std::vector<std::string> leftEyeIdentifiers;
    std::shared_ptr<DeviceImages> dev;   // shared between the copies the optimiser makes of this functor
};

}  // namespace rcr
