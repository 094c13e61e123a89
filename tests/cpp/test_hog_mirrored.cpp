// Mirrored samples in the C++14 shells, written as apps/rcr/rcr-train.cpp would build a mirrored training set: for every photo,
// shallow copies for the box and its perturbations, and as many shallow copies marked mirrored in HogTransform's `mirrored`, with
// ground truth and initialisations from rcr::mirror_box / rcr::mirror_landmarks.  Needs a GPU to run; compiling it
// (g++ -std=c++14) is part of the CPU test-suite.
//
//   test_hog_mirrored MODEL
//     trains a two-level cascade on that set and on the same set with hand-flipped deep copies in place of the mirrored entries,
//     prints "PERM ..." (rcr::mirror_permutation of the model's list), "FRAMES mirrored S copies D" (frames each transform
//     holds), "WEIGHTS level L: d" and "TEST: d" (largest differences, which must be 0); then the same on the host route
//     ("HOST WEIGHTS level L: d", "HOST TEST: d") and one mirrored entry through the functor ("FUNCTOR: d").
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

// cv::flip(m, 1) by hand: a deep copy with every row reversed, pixel by pixel
static Mat flipped(const Mat& m)
{
    Mat out(m.rows, m.cols, m.type());
    const int ch = m.channels();
    for (int y = 0; y < m.rows; ++y)
        for (int x = 0; x < m.cols; ++x)
            for (int c = 0; c < ch; ++c) out.ptr<unsigned char>(y)[x * ch + c] = m.ptr<unsigned char>(y)[(m.cols - 1 - x) * ch + c];
    return out;
}

int main(int argc, char** argv)
{
    if (argc < 2) {
        std::printf("usage: test_hog_mirrored MODEL\n");
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
        const std::vector<int> perm = mirror_permutation(ids);
        std::printf("PERM");
        for (int p : perm) std::printf(" %d", p);
        std::printf("\n");
        const std::vector<std::string> reye{"37", "40"}, leye{"43", "46"};
        const int photos = 12, per = 5;
        std::vector<Mat> loaded_images;
        std::vector<cv::Rect> boxes;
        unsigned s = 777;
        for (int i = 0; i < photos; ++i) {
            const int w = i % 2 ? 151 : 130, h = i % 2 ? 140 : 127;         // odd and even widths
            Mat im(h, w, i % 3 == 0 ? CV_8UC3 : CV_8UC1);
            const int ch = im.channels();
            for (int yy = 0; yy < h; ++yy)
                for (int xx = 0; xx < w * ch; ++xx) {
                    s = s * 1664525u + 1013904223u;
                    im.ptr<unsigned char>(yy)[xx] = static_cast<unsigned char>(128 + 60 * std::sin(0.13 * xx + 0.05 * i) * std::cos(0.06 * yy) + ((s >> 24) & 31));
                }
            loaded_images.push_back(im);
            boxes.emplace_back(8 + i % 7, 9 + i % 5, 100, 100);
        }
        Mat x_gt, x0;
        std::vector<Mat> in_place, copies, flips;
        std::vector<bool> mirrored;
        for (int i = 0; i < photos; ++i) flips.push_back(flipped(loaded_images[i]));
        for (int m = 0; m < 2; ++m)
            for (int i = 0; i < photos; ++i) {
                const int W = loaded_images[i].cols;
                const cv::Rect box = m ? mirror_box(boxes[i], W) : boxes[i];
                for (int k = 0; k < per; ++k) {
                    const float tx = k == 0 ? 0.f : 0.02f * ((k * 7) % 5 - 2), ty = k == 0 ? 0.f : 0.02f * ((k * 3) % 5 - 2);
                    const float sc = k == 0 ? 1.f : 1.f + 0.015f * ((k * 5) % 3 - 1);
                    Mat gt = align_mean(mean, boxes[i]), init = align_mean(mean, boxes[i], sc, sc, tx, ty);
                    if (m) {                                                    // the mirrored photo's ground truth and start
                        gt = mirror_landmarks(gt, {W}, perm);
                        init = align_mean(mean, box, sc, sc, tx, ty);
                    }
                    x_gt.push_back(gt);
                    x0.push_back(init);
                    in_place.emplace_back(loaded_images[i]);
                    mirrored.push_back(m == 1);
                    copies.emplace_back(m ? flips[i] : loaded_images[i]);
                }
            }
        const std::vector<HoGParam> hp{{VlHogVariantUoctti, 3, 8, 4, 0.8f}, {VlHogVariantUoctti, 3, 6, 4, 0.5f}};
        HogTransform a_h(in_place, hp, ids, reye, leye, mirrored), b_h(copies, hp, ids, reye, leye);
        const Regulariser reg(Regulariser::RegularisationType::MatrixNorm, 1.5f, false);
        using Opt = SupervisedDescentOptimiser<LinearRegressor<>, InterEyeDistanceNormalisation>;
        Opt a({LinearRegressor<>(reg), LinearRegressor<>(reg)}, InterEyeDistanceNormalisation(ids, reye, leye));
        Opt b({LinearRegressor<>(reg), LinearRegressor<>(reg)}, InterEyeDistanceNormalisation(ids, reye, leye));
        a.train(x_gt, x0, Mat(), a_h);
        b.train(x_gt, x0, Mat(), b_h);
        std::printf("FRAMES mirrored %d copies %d\n", a_h.num_frames(), b_h.num_frames());
        if (a_h.num_frames() != photos || b_h.num_frames() != 2 * photos || !a_h.on_device() || !b_h.on_device()) {
            std::printf("FAIL frame counts or route\n");
            ++failures;
        }
        for (size_t level = 0; level < 2; ++level) {
            const double e = max_abs_diff(a.get_regressors()[level].x, b.get_regressors()[level].x);
            std::printf("WEIGHTS level %zu: %.3e\n", level, e);
            if (e != 0.0) { std::printf("FAIL level %zu: weights differ\n", level); ++failures; }
        }
        const double d = max_abs_diff(a.test(x0, Mat(), a_h), b.test(x0, Mat(), b_h));
        std::printf("TEST: %.3e\n", d);
        if (d != 0.0) { std::printf("FAIL test() differs\n"); ++failures; }
        // the same set kept in host memory: bit for bit the device route
        HogTransform::device_frame_share() = 0.0;
        HogTransform on_host(in_place, hp, ids, reye, leye, mirrored);
        Opt h({LinearRegressor<>(reg), LinearRegressor<>(reg)}, InterEyeDistanceNormalisation(ids, reye, leye));
        h.train(x_gt, x0, Mat(), on_host);
        HogTransform::device_frame_share() = 0.5;
        if (on_host.on_device() || on_host.num_frames() != photos) { std::printf("FAIL host route not taken\n"); ++failures; }
        for (size_t level = 0; level < 2; ++level) {
            const double e = max_abs_diff(b.get_regressors()[level].x, h.get_regressors()[level].x);
            std::printf("HOST WEIGHTS level %zu: %.3e\n", level, e);
            if (e != 0.0) { std::printf("FAIL level %zu: host-route weights differ\n", level); ++failures; }
        }
        const double dh = max_abs_diff(b.test(x0, Mat(), b_h), h.test(x0, Mat(), on_host));
        std::printf("HOST TEST: %.3e\n", dh);
        if (dh != 0.0) { std::printf("FAIL host-route test() differs\n"); ++failures; }
        // one mirrored entry through the functor (predict()'s call shape)
        const int e = photos * per + 3;
        const double f = max_abs_diff(a_h(x0.row(e), 0, e), b_h(x0.row(e), 0, e));
        std::printf("FUNCTOR: %.3e\n", f);
        if (f != 0.0) { std::printf("FAIL functor differs\n"); ++failures; }
    } catch (const std::exception& ex) {
        std::printf("EXCEPTION %s\n", ex.what());
        return 2;
    }
    std::printf(failures ? "FAILED %d\n" : "ALL OK %d\n", failures);
    return failures ? 1 : 0;
}
