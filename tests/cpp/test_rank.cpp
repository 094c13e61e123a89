// The rank diagnostic of ColPivHouseholderQRSolver (regressors.hpp:245-306) on the optimiser's device route: a
// SupervisedDescentOptimiser<LinearRegressor<ColPivHouseholderQRSolver>> trained with a HogTransform.  Needs a GPU to run;
// compiling it (g++ -std=c++14) is part of the CPU test-suite.
//
//   test_rank MODEL
//     prints "RANK level L: r of D" for a MatrixNorm-regularised two-level train, then trains one level with lambda = 0 on
//     fewer samples than features: the solver prints the reference's message and train() throws with the rank in its text.
#include <cmath>
#include <cstdio>
#include <string>
#include <vector>

#include "rcr/model.hpp"

using namespace superviseddescent;
using cv::Mat;

int main(int argc, char** argv)
{
    if (argc < 2) {
        std::printf("usage: test_rank MODEL\n");
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
        const int n = 400, w = 128, hgt = 128;
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
            const cv::Rect box(12 + (i % 5), 10 + (i % 7), 100, 100);
            x_gt.push_back(align_mean(mean, box, 1.0f + 0.01f * (i % 3), 1.0f, 0.01f * (i % 4 - 2), 0.01f * (i % 5 - 2)));
            x0.push_back(align_mean(mean, box));
        }
        const std::vector<HoGParam> hp{{VlHogVariantUoctti, 3, 8, 4, 0.8f}, {VlHogVariantUoctti, 3, 6, 4, 0.5f}};
        HogTransform hog(images, hp, ids, reye, leye);
        using QrRegressor = LinearRegressor<ColPivHouseholderQRSolver>;
        {
            const Regulariser reg(Regulariser::RegularisationType::MatrixNorm, 1.5f, false);
            SupervisedDescentOptimiser<QrRegressor, InterEyeDistanceNormalisation> sdo({QrRegressor(reg), QrRegressor(reg)},
                                                                                      InterEyeDistanceNormalisation(ids, reye, leye));
            sdo.train(x_gt, x0, Mat(), hog);
            for (size_t level = 0; level < 2; ++level) {
                const int D = hog.feature_length(level);
                const int r = sdo.get_regressors()[level].get_solver().last_rank;
                std::printf("RANK level %zu: %d of %d\n", level, r, D);
                if (r != D) { std::printf("FAIL level %zu: a MatrixNorm-regularised system must have full rank\n", level); ++failures; }
            }
        }
        {
            // n = 400 samples, D = 3169 features, no regularisation: rank deficient, and the factorisation breaks down
            SupervisedDescentOptimiser<QrRegressor, InterEyeDistanceNormalisation> sdo({QrRegressor(Regulariser())},
                                                                                      InterEyeDistanceNormalisation(ids, reye, leye));
            std::printf("-- expecting the rank warning of regressors.hpp:290-293 --\n");
            try {
                sdo.train(x_gt, x0, Mat(), hog);
                std::printf("FAIL a singular system did not throw\n");
                ++failures;
            } catch (const std::runtime_error& e) {
                std::printf("expected error: %s\n", e.what());
                const int r = sdo.get_regressors()[0].get_solver().last_rank;
                std::printf("DEFICIENT level 0: %d of %d\n", r, hog.feature_length(0));
                if (!(r > 0 && r < hog.feature_length(0)) || std::string(e.what()).find("(The rank is " + std::to_string(r) + ",") == std::string::npos) {
                    std::printf("FAIL the error does not carry the rank\n");
                    ++failures;
                }
            }
        }
    } catch (const std::exception& e) {
        std::printf("EXCEPTION %s\n", e.what());
        return 2;
    }
    std::printf(failures ? "FAILED %d\n" : "ALL OK %d\n", failures);
    return failures ? 1 : 0;
}
