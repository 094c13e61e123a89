// Training and testing in chunks of rows on the optimiser's device route (SupervisedDescentOptimiser::set_rows_per_chunk).
// Needs a GPU to run; compiling it (g++ -std=c++14) is part of the CPU test-suite.
//
//   test_train_chunks MODEL
//     trains a two-level HogTransform cascade in one chunk and in chunks of 300 rows, prints "WEIGHTS level L: e" (largest
//     weight difference relative to the largest weight) and "TEST: d" (largest difference of the chunked test() from the
//     unchunked one).
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <string>
#include <vector>

#include "rcr/model.hpp"

using namespace superviseddescent;
using cv::Mat;

static double max_abs(const Mat& m)
{
    double v = 0.0;
    for (int r = 0; r < m.rows; ++r)
        for (int c = 0; c < m.cols; ++c) v = std::max(v, std::fabs(static_cast<double>(m.at<float>(r, c))));
    return v;
}

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
        std::printf("usage: test_train_chunks MODEL\n");
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
        const int n = 900, w = 112, hgt = 112;
        std::vector<Mat> images;
        unsigned s = 777;
        for (int i = 0; i < n; ++i) {
            Mat im(hgt, w, CV_8UC1);
            for (int yy = 0; yy < hgt; ++yy)
                for (int xx = 0; xx < w; ++xx) {
                    s = s * 1664525u + 1013904223u;
                    im.at<unsigned char>(yy, xx) = static_cast<unsigned char>(128 + 60 * std::sin(0.11 * xx + 0.03 * i) * std::cos(0.07 * yy + 0.01 * i) + ((s >> 24) & 31));
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
        const Regulariser reg(Regulariser::RegularisationType::MatrixNorm, 1.5f, false);
        using Opt = SupervisedDescentOptimiser<LinearRegressor<>, InterEyeDistanceNormalisation>;
        Opt whole({LinearRegressor<>(reg), LinearRegressor<>(reg)}, InterEyeDistanceNormalisation(ids, reye, leye));
        Opt chunked({LinearRegressor<>(reg), LinearRegressor<>(reg)}, InterEyeDistanceNormalisation(ids, reye, leye));
        chunked.set_rows_per_chunk(300);
        whole.train(x_gt, x0, Mat(), hog);
        chunked.train(x_gt, x0, Mat(), hog);
        for (size_t level = 0; level < 2; ++level) {
            const Mat a = whole.get_regressors()[level].x, b = chunked.get_regressors()[level].x;
            const double e = max_abs_diff(a, b) / max_abs(a);
            std::printf("WEIGHTS level %zu: %.3e\n", level, e);
            if (!(e <= 1e-5)) { std::printf("FAIL level %zu: chunked weights differ by %.3e\n", level, e); ++failures; }
        }
        const Mat t_whole = whole.test(x0, Mat(), hog);
        whole.set_rows_per_chunk(300);
        const Mat t_chunked = whole.test(x0, Mat(), hog);
        const double d = max_abs_diff(t_whole, t_chunked);
        std::printf("TEST: %.3e\n", d);
        if (d != 0.0) { std::printf("FAIL the chunked test() differs from the unchunked one\n"); ++failures; }
    } catch (const std::exception& e) {
        std::printf("EXCEPTION %s\n", e.what());
        return 2;
    }
    std::printf(failures ? "FAILED %d\n" : "ALL OK %d\n", failures);
    return failures ? 1 : 0;
}
