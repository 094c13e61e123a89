// Several samples per photo on the optimiser's device route, written as apps/rcr/rcr-train.cpp builds its training set: one
// shallow cv::Mat copy of the photo per sample (the detected box and its perturbations).  Needs a GPU to run; compiling it
// (g++ -std=c++14) is part of the CPU test-suite.
//
//   test_train_host_frames MODEL
//     trains a two-level HogTransform cascade on the shallow copies and on deep copies of the same photos, prints
//     "FRAMES shallow S deep D" (frames each HogTransform holds on the device), "WEIGHTS level L: d" and "TEST: d" (largest
//     differences between the two runs, which must be 0); then trains on the shallow copies kept in host memory
//     (HogTransform::device_frame_share() lowered to 0) and prints "HOST WEIGHTS level L: d" and "HOST TEST: d" against the
//     device route (also 0).
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <string>
#include <vector>

#include "rcr/model.hpp"

using namespace superviseddescent;
using cv::Mat;

static double max_abs_diff(const Mat& a, const Mat& b)
{
    double v = 0.0;
    for (int r = 0; r < a.rows; ++r)
        for (int c = 0; c < a.cols; ++c) v = std::max(v, std::fabs(static_cast<double>(a.at<float>(r, c)) - b.at<float>(r, c)));
    return v;
}

int main(int argc, char** argv)
{
    if (argc < 2) {
        std::printf("usage: test_train_host_frames MODEL\n");
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
        // the loaded photos: grey and colour, two sizes
        const int photos = 40;
        std::vector<Mat> loaded_images;
        std::vector<cv::Rect> boxes;
        unsigned s = 4242;
        for (int i = 0; i < photos; ++i) {
            const int w = i % 2 ? 150 : 131, h = i % 2 ? 140 : 127;
            Mat im(h, w, i % 3 == 0 ? CV_8UC3 : CV_8UC1);
            const int ch = im.channels();
            for (int yy = 0; yy < h; ++yy)
                for (int xx = 0; xx < w * ch; ++xx) {
                    s = s * 1664525u + 1013904223u;
                    im.ptr<unsigned char>(yy)[xx] = static_cast<unsigned char>(128 + 60 * std::sin(0.11 * xx + 0.03 * i) * std::cos(0.07 * yy) + ((s >> 24) & 31));
                }
            loaded_images.push_back(im);
            boxes.emplace_back(10 + i % 7, 9 + i % 5, 100, 100);
        }
        // apps/rcr/rcr-train.cpp:396-430: the box itself and 10 perturbations of it, each with its own entry in training_images
        Mat x_gt, x0;
        std::vector<Mat> training_images, deep_images;
        for (int i = 0; i < photos; ++i) {
            for (int k = 0; k < 11; ++k) {
                const float tx = k == 0 ? 0.f : 0.02f * ((k * 7) % 5 - 2), ty = k == 0 ? 0.f : 0.02f * ((k * 3) % 5 - 2);
                const float sc = k == 0 ? 1.f : 1.f + 0.015f * ((k * 5) % 3 - 1);
                x0.push_back(align_mean(mean, boxes[i], sc, sc, tx, ty));
                x_gt.push_back(align_mean(mean, boxes[i]));
                training_images.emplace_back(loaded_images[i]);
                deep_images.emplace_back(loaded_images[i].clone());
            }
        }
        const std::vector<HoGParam> hp{{VlHogVariantUoctti, 3, 8, 4, 0.8f}, {VlHogVariantUoctti, 3, 6, 4, 0.5f}};
        HogTransform shallow(training_images, hp, ids, reye, leye), deep(deep_images, hp, ids, reye, leye);
        const Regulariser reg(Regulariser::RegularisationType::MatrixNorm, 1.5f, false);
        using Opt = SupervisedDescentOptimiser<LinearRegressor<>, InterEyeDistanceNormalisation>;
        Opt a({LinearRegressor<>(reg), LinearRegressor<>(reg)}, InterEyeDistanceNormalisation(ids, reye, leye));
        Opt b({LinearRegressor<>(reg), LinearRegressor<>(reg)}, InterEyeDistanceNormalisation(ids, reye, leye));
        a.train(x_gt, x0, Mat(), shallow);
        b.train(x_gt, x0, Mat(), deep);
        std::printf("FRAMES shallow %d deep %d\n", shallow.num_frames(), deep.num_frames());
        if (shallow.num_frames() != photos || deep.num_frames() != 11 * photos || !shallow.on_device() || !deep.on_device()) {
            std::printf("FAIL frame counts or route\n");
            ++failures;
        }
        for (size_t level = 0; level < 2; ++level) {
            const double e = max_abs_diff(a.get_regressors()[level].x, b.get_regressors()[level].x);
            std::printf("WEIGHTS level %zu: %.3e\n", level, e);
            if (e != 0.0) { std::printf("FAIL level %zu: weights differ\n", level); ++failures; }
        }
        const double d = max_abs_diff(a.test(x0, Mat(), shallow), b.test(x0, Mat(), deep));
        std::printf("TEST: %.3e\n", d);
        if (d != 0.0) { std::printf("FAIL test() differs\n"); ++failures; }
        // the same training set kept in host memory (the route threshold lowered): bit for bit the device route
        HogTransform::device_frame_share() = 0.0;
        HogTransform on_host(training_images, hp, ids, reye, leye);
        Opt h({LinearRegressor<>(reg), LinearRegressor<>(reg)}, InterEyeDistanceNormalisation(ids, reye, leye));
        h.train(x_gt, x0, Mat(), on_host);
        HogTransform::device_frame_share() = 0.5;
        std::printf("HOST ROUTE on_device %d frames %d\n", on_host.on_device() ? 1 : 0, on_host.num_frames());
        if (on_host.on_device() || on_host.num_frames() != photos) { std::printf("FAIL host route not taken\n"); ++failures; }
        for (size_t level = 0; level < 2; ++level) {
            const double e = max_abs_diff(a.get_regressors()[level].x, h.get_regressors()[level].x);
            std::printf("HOST WEIGHTS level %zu: %.3e\n", level, e);
            if (e != 0.0) { std::printf("FAIL level %zu: host-route weights differ\n", level); ++failures; }
        }
        const double dh = max_abs_diff(a.test(x0, Mat(), shallow), h.test(x0, Mat(), on_host));
        std::printf("HOST TEST: %.3e\n", dh);
        if (dh != 0.0) { std::printf("FAIL host-route test() differs\n"); ++failures; }
        // one sample through the functor (predict()'s call shape): entry 11 * 5 is photo 5
        const double f = max_abs_diff(shallow(x0.row(55), 0, 55), deep(x0.row(55), 0, 55));
        if (f != 0.0) { std::printf("FAIL functor differs\n"); ++failures; }
    } catch (const std::exception& e) {
        std::printf("EXCEPTION %s\n", e.what());
        return 2;
    }
    std::printf(failures ? "FAILED %d\n" : "ALL OK %d\n", failures);
    return failures ? 1 : 0;
}
