// A device batch projection (feature_length / project_device) through SupervisedDescentOptimiser::train / test on the device
// route (sd_train_level_projected / sd_apply_level_projected).  Needs a GPU to run; compiling it (g++ -std=c++14) is part of the
// CPU test-suite.
//
//   test_projection MODEL
//     HogRows writes the HOG rows of a HogTransform's device frames with sd_hog_batch: trained and tested through the callback
//     it must give the HogTransform cascade bit for bit ("IDENTICAL <case>"), in one chunk and with set_rows_per_chunk, with a
//     training callback.  An exception thrown by project_device must come out of train() ("RETHROWN").
#include <cmath>
#include <cstdio>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include "rcr/model.hpp"

using namespace superviseddescent;
using cv::Mat;

// HOG rows of a HogTransform's frames, computed by the projection itself
struct HogRows {
    rcr::HogTransform* hog;
    int n, L;
    int* calls;
    bool fail;
    int feature_length(size_t level) const { return hog->feature_length(level); }
    int project_device(sd_ctx* ctx, size_t level, const float* d_x, int64_t ldx, int64_t first_row, int rows, float* d_out, int64_t ld)
    {
        ++*calls;
        if (fail) throw std::runtime_error("projection failed on purpose");
        const sd_level_frames f = hog->level_frames(n);
        const sd_normalisation eyes = hog->eyes();
        const sd_hog_param p = hog->hog_param(level);
        return sd_hog_batch(ctx, f.images, f.d_sample_frame + first_row, d_x, ldx, rows, L, &eyes, &p, d_out, ld);
    }
};

static bool same(const Mat& a, const Mat& b)
{
    return a.rows == b.rows && a.cols == b.cols && std::memcmp(a.ptr<float>(0), b.ptr<float>(0), static_cast<size_t>(a.rows) * a.cols * sizeof(float)) == 0;
}

int main(int argc, char** argv)
{
    if (argc < 2) {
        std::printf("usage: test_projection MODEL\n");
        return 2;
    }
    int failures = 0;
    try {
        using namespace rcr;
        detection_model pre = load_detection_model(argv[1]);
        const Mat mean = pre.get_mean();
        const int L = mean.cols / 2;
        std::vector<std::string> ids;
        for (int i = 0; i < L; ++i) ids.emplace_back(sd_model_landmark_id(pre.native(), i));
        const std::vector<std::string> reye{"37", "40"}, leye{"43", "46"};
        const int n = 600, w = 112, hgt = 112;
        std::vector<Mat> images;
        unsigned s = 4242;
        for (int i = 0; i < n; ++i) {
            Mat im(hgt, w, CV_8UC1);
            for (int yy = 0; yy < hgt; ++yy)
                for (int xx = 0; xx < w; ++xx) {
                    s = s * 1664525u + 1013904223u;
                    im.at<unsigned char>(yy, xx) = static_cast<unsigned char>(128 + 60 * std::sin(0.13 * xx + 0.02 * i) * std::cos(0.05 * yy + 0.01 * i) + ((s >> 24) & 31));
                }
            images.push_back(im);
        }
        Mat x_gt, x0;
        for (int i = 0; i < n; ++i) {
            const cv::Rect box(8 + (i % 5), 7 + (i % 7), 96, 96);
            x_gt.push_back(align_mean(mean, box, 1.0f + 0.01f * (i % 3), 1.0f, 0.01f * (i % 4 - 2), 0.01f * (i % 5 - 2)));
            x0.push_back(align_mean(mean, box));
        }
        const std::vector<HoGParam> hp{{VlHogVariantUoctti, 3, 8, 4, 0.8f}, {VlHogVariantUoctti, 3, 6, 4, 0.5f}};
        HogTransform hog(images, hp, ids, reye, leye);
        int calls = 0;
        HogRows rows{&hog, n, L, &calls, false};
        static_assert(detail::is_device_batch_projection<HogRows>::value && !detail::is_device_projection<HogRows>::value,
                      "HogRows takes the batch projection route");
        const Regulariser reg(Regulariser::RegularisationType::MatrixNorm, 1.5f, false);
        using Opt = SupervisedDescentOptimiser<LinearRegressor<>, InterEyeDistanceNormalisation>;
        for (int chunk : {0, 250}) {
            Opt a({LinearRegressor<>(reg), LinearRegressor<>(reg)}, InterEyeDistanceNormalisation(ids, reye, leye));
            Opt b({LinearRegressor<>(reg), LinearRegressor<>(reg)}, InterEyeDistanceNormalisation(ids, reye, leye));
            a.set_rows_per_chunk(chunk);
            b.set_rows_per_chunk(chunk);
            std::vector<Mat> seen_a, seen_b;
            a.train(x_gt, x0, Mat(), hog, [&](const Mat& x) { seen_a.push_back(x.clone()); });
            calls = 0;
            b.train(x_gt, x0, Mat(), rows, [&](const Mat& x) { seen_b.push_back(x.clone()); });
            const int want_calls = chunk ? 2 * (2 * ((n + chunk - 1) / chunk) - 1) : 2;     // twice per chunk but the last, per level
            bool ok = calls == want_calls && seen_a.size() == 2 && seen_b.size() == 2;
            for (size_t level = 0; level < 2 && ok; ++level)
                ok = same(a.get_regressors()[level].x, b.get_regressors()[level].x) && same(seen_a[level], seen_b[level]);
            ok = ok && same(a.test(x0, Mat(), hog), b.test(x0, Mat(), rows));
            std::printf("%s chunk %d (%d projection calls)\n", ok ? "IDENTICAL" : "DIFFERENT", chunk, calls);
            if (!ok) { std::printf("FAIL chunk %d: the batch projection is not the HogTransform level\n", chunk); ++failures; }
        }
        HogRows failing{&hog, n, L, &calls, true};
        Opt c({LinearRegressor<>(reg)}, InterEyeDistanceNormalisation(ids, reye, leye));
        try {
            c.train(x_gt, x0, Mat(), failing);
            std::printf("FAIL train() returned although project_device threw\n");
            ++failures;
        } catch (const std::runtime_error& e) {
            const bool ok = std::string(e.what()) == "projection failed on purpose";
            std::printf(ok ? "RETHROWN\n" : "FAIL wrong exception: %s\n", e.what());
            failures += ok ? 0 : 1;
        }
    } catch (const std::exception& e) {
        std::printf("EXCEPTION %s\n", e.what());
        return 2;
    }
    std::printf(failures ? "FAILED %d\n" : "ALL OK %d\n", failures);
    return failures ? 1 : 0;
}
