// Exercises the C++14 header shells exactly the way the reference's own gtest files and apps use the
// original headers (tests/test_LinearRegressorND.cpp:152-172,255-282, tests/test_LinearRegressor1D.cpp:84-103,
// tests/test_SupervisedDescentOptimiser.cpp:30-144, apps/rcr/rcr-detect.cpp:87-120).  Needs a GPU to run;
// compiling it (g++ -std=c++14) is part of the CPU test-suite.
//
//   test_shells                               regressor + optimiser known answers
//   test_shells MODEL FRAME.raw W H X Y BW BH OUT.bin   additionally: load model, detect, save model
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <iostream>
#include <vector>

#include "rcr/model.hpp"
#include "superviseddescent/regressors.hpp"
#include "superviseddescent/superviseddescent.hpp"

using namespace superviseddescent;
using cv::Mat;

static int failures = 0;
#define EXPECT_REL(expected, actual, tol)                                                                  \
    do {                                                                                                   \
        const double e_ = (expected), a_ = (actual);                                                       \
        if (!(std::fabs(a_ - e_) <= (tol) * std::max(std::fabs(e_), 1e-3))) {                              \
            std::printf("FAIL %s:%d expected %.9g got %.9g\n", __FILE__, __LINE__, e_, a_);                \
            ++failures;                                                                                    \
        }                                                                                                  \
    } while (0)

static Mat from(std::initializer_list<float> v, int rows, int cols)
{
    Mat m(rows, cols, CV_32FC1);
    int i = 0;
    for (float f : v) { m.at<float>(i / cols, i % cols) = f; ++i; }
    return m;
}

static void test_regressors()
{
    // NDimManyExamplesNDimY (test_LinearRegressorND.cpp:152-172)
    Mat data = from({1, 4, 2, 4, 9, 1, 6, 5, 2, 0, 6, 2, 6, 1, 9}, 5, 3);
    Mat labels = from({1, 1, 2, 5, 3, -2, 0, 5, 6, 3}, 5, 2);
    LinearRegressor<> lr;
    const bool ok = lr.learn(data, labels);
    if (!ok) { std::printf("FAIL learn returned false\n"); ++failures; }
    EXPECT_REL(0.489539, lr.x.at<float>(0, 0), 1e-4);
    EXPECT_REL(-0.06608297, lr.x.at<float>(1, 0), 1e-4);
    EXPECT_REL(0.339629412, lr.x.at<float>(2, 0), 1e-4);
    EXPECT_REL(-0.833899379, lr.x.at<float>(0, 1), 1e-4);
    EXPECT_REL(0.626753688, lr.x.at<float>(1, 1), 1e-4);
    EXPECT_REL(0.744218946, lr.x.at<float>(2, 1), 1e-4);
    Mat test = from({2.0f, 6.0f, 5.0f, 2.9f, -11.3f, 6.0f, -2.0f, -8.438f, 3.3f}, 3, 3);
    Mat gt = from({2.2807f, 5.8138f, 4.2042f, -5.0353f, 0.6993f, -1.1648f}, 3, 2);
    if (!(lr.test(test, gt) <= 0.000012)) { std::printf("FAIL residual %g\n", lr.test(test, gt)); ++failures; }

    // NDimManyExamplesNDimYBiasRegularisationButNotBias (:255-282)
    Regulariser r(Regulariser::RegularisationType::Manual, 50.0f, false);
    LinearRegressor<> lrb(r);
    Mat bias = Mat::ones(data.rows, 1, CV_32FC1), datab;
    cv::hconcat(data, bias, datab);
    lrb.learn(datab, labels);
    EXPECT_REL(0.2188783, lrb.x.at<float>(0, 0), 1e-4);
    EXPECT_REL(1.53583705, lrb.x.at<float>(3, 0), 1e-4);
    EXPECT_REL(-0.174922630, lrb.x.at<float>(0, 1), 1e-4);
    EXPECT_REL(1.82635951, lrb.x.at<float>(3, 1), 1e-4);

    // ColPivHouseholderQRSolver (regressors.hpp:245-306): same weights as the LU solver on a regular system, full rank reported
    {
        LinearRegressor<ColPivHouseholderQRSolver> lq;
        lq.learn(data, labels);
        EXPECT_REL(0.489539, lq.x.at<float>(0, 0), 1e-4);
        EXPECT_REL(0.744218946, lq.x.at<float>(2, 1), 1e-4);
        // a duplicated column without regularisation: rank 3 of 4, the reference's warning is printed (:290-293), learn() still
        // returns true (:349)
        Mat dup;
        cv::hconcat(data, data.colRange(1, 2), dup);
        LinearRegressor<ColPivHouseholderQRSolver> ld;
        std::printf("-- expecting the rank warning of regressors.hpp:290-293 --\n");
        const bool okd = ld.learn(dup, labels);
        if (!okd) { std::printf("FAIL QR learn returned false\n"); ++failures; }
        // with lambda > 0 the same data is regular again
        LinearRegressor<ColPivHouseholderQRSolver> lreg(Regulariser(Regulariser::RegularisationType::Manual, 1.0f, true));
        lreg.learn(dup, labels);
        if (!(lreg.x.rows == 4 && std::isfinite(lreg.x.at<float>(3, 1)))) { std::printf("FAIL regularised QR solve\n"); ++failures; }
    }

    // OneDimOneExampleTestingResidual (test_LinearRegressor1D.cpp:84-103)
    LinearRegressor<> l1;
    l1.learn(Mat::ones(1, 1, CV_32FC1), Mat::ones(1, 1, CV_32FC1));
    Mat t3 = from({0, 1, 2}, 3, 1), g3 = from({-1, 2, 2}, 3, 1);
    EXPECT_REL(0.47140452079103173, l1.test(t3, g3), 1e-5);
    Mat p = l1.predict(from({2.0f}, 1, 1));
    EXPECT_REL(2.0, p.at<float>(0), 1e-6);
}

static void test_optimiser()
{
    // SinConvergence / SinConvergenceCascade (test_SupervisedDescentOptimiser.cpp:30-144)
    auto h = [](Mat value, size_t, int) { return std::sin(value.at<float>(0)); };
    auto h_inv = [](float v) { return v >= 1.0f ? std::asin(1.0f) : std::asin(v); };
    const int n = 11;
    std::vector<float> y(n), x(n);
    float v = -1.0f;
    for (int i = 0; i < n; ++i) { y[i] = v; v += 0.2f; }
    for (int i = 0; i < n; ++i) x[i] = h_inv(y[i]);
    Mat y_tr(y, true), x_tr(x, true);
    Mat x0 = 0.5f * Mat::ones(n, 1, CV_32FC1);
    {
        SupervisedDescentOptimiser<LinearRegressor<>> sdo({LinearRegressor<>()});
        int calls = 0;
        auto check = [&](const Mat& cur) { ++calls; EXPECT_REL(0.21369851877468238, cv::norm(cur, x_tr, cv::NORM_L2) / cv::norm(x_tr, cv::NORM_L2), 1e-4); };
        sdo.train(x_tr, x0, y_tr, h, check);
        if (calls != 1) { std::printf("FAIL callback calls %d\n", calls); ++failures; }
        Mat pred = sdo.test(x0, y_tr, h);
        EXPECT_REL(0.21369851877468238, cv::norm(pred, x_tr, cv::NORM_L2) / cv::norm(x_tr, cv::NORM_L2), 1e-4);
    }
    {
        std::vector<LinearRegressor<>> regs(10);
        SupervisedDescentOptimiser<LinearRegressor<>> sdo(regs);
        sdo.train(x_tr, x0, y_tr, h);
        Mat pred = sdo.test(x0, y_tr, h);
        EXPECT_REL(0.040279395, cv::norm(pred, x_tr, cv::NORM_L2) / cv::norm(x_tr, cv::NORM_L2), 1e-4);
        Mat one = sdo.predict(x0.row(3), y_tr.row(3), [&](Mat value, size_t l, int i) { return h(value, l, i); });
        EXPECT_REL(pred.at<float>(3), one.at<float>(0), 1e-5);
    }
}

static void test_rcr_device_route(const char* model_path)
{
    // rcr-train style: HogTransform as the projection, IED normalisation, trained on the device route.
    using namespace rcr;
    detection_model pre = load_detection_model(model_path);
    Mat mean = pre.get_mean();
    const int L = mean.cols / 2;
    std::vector<std::string> ids;
    for (int i = 0; i < L; ++i) ids.emplace_back(sd_model_landmark_id(pre.native(), i));
    std::vector<std::string> reye{"37", "40"}, leye{"43", "46"};
    const int n = 40, w = 160, hgt = 160;
    std::vector<Mat> images;
    unsigned s = 12345;
    for (int i = 0; i < n; ++i) {
        Mat im(hgt, w, CV_8UC1);
        for (int yy = 0; yy < hgt; ++yy)
            for (int xx = 0; xx < w; ++xx) {
                s = s * 1664525u + 1013904223u;
                im.at<unsigned char>(yy, xx) = static_cast<unsigned char>(128 + 60 * std::sin(0.11 * xx + 0.01 * i) * std::cos(0.07 * yy) + ((s >> 24) & 15));
            }
        images.push_back(im);
    }
    Mat x_gt, x0;
    for (int i = 0; i < n; ++i) {
        cv::Rect box(20 + (i % 5), 18 + (i % 7), 110, 110);
        x_gt.push_back(align_mean(mean, box, 1.0f + 0.01f * (i % 3), 1.0f, 0.01f * (i % 4 - 2), 0.01f * (i % 5 - 2)));
        x0.push_back(align_mean(mean, box));
    }
    std::vector<HoGParam> hp{{VlHogVariantUoctti, 3, 8, 4, 0.8f}, {VlHogVariantUoctti, 3, 6, 4, 0.5f}};
    HogTransform hog(images, hp, ids, reye, leye);
    Regulariser reg(Regulariser::RegularisationType::MatrixNorm, 1.5f, false);
    std::vector<LinearRegressor<VerbosePartialPivLUSolver>> regs{LinearRegressor<VerbosePartialPivLUSolver>(reg), LinearRegressor<VerbosePartialPivLUSolver>(reg)};
    detection_model::model_type sdo(regs, InterEyeDistanceNormalisation(ids, reye, leye));
    std::vector<double> errs;
    errs.push_back(cv::norm(x0, x_gt, cv::NORM_L2) / cv::norm(x_gt, cv::NORM_L2));
    sdo.train(x_gt, x0, Mat(), hog, [&](const Mat& cur) { errs.push_back(cv::norm(cur, x_gt, cv::NORM_L2) / cv::norm(x_gt, cv::NORM_L2)); });
    std::printf("device-route training residuals: %.6f -> %.6f -> %.6f\n", errs[0], errs[1], errs[2]);
    if (!(errs.size() == 3 && errs[1] < errs[0] && errs[2] < errs[1])) { std::printf("FAIL training did not reduce the residual\n"); ++failures; }
    // the functor route must agree with the device route (same kernels, host-stacked features)
    Mat dev = sdo.test(x0, Mat(), hog);
    Mat host = sdo.test(x0, Mat(), [&](Mat row, size_t level, int idx) { return hog(row, level, idx); });
    EXPECT_REL(0.0, cv::norm(dev, host, cv::NORM_L2) / cv::norm(dev, cv::NORM_L2), 1e-3);   // tol * max(|e|,1e-3) = 1e-6
    // the multi-GPU overload with a one-rank communicator must give the same model (the exchange degenerates; two and more
    // ranks are covered by tests/test_gpu_multi.py)
    {
        sd_comm* comm = nullptr;
        sd_b200::check(sd_b200::context(), sd_comm_create(sd_b200::context(), nullptr, 0, 1, &comm), "sd_comm_create");
        std::vector<LinearRegressor<VerbosePartialPivLUSolver>> regs2{LinearRegressor<VerbosePartialPivLUSolver>(reg), LinearRegressor<VerbosePartialPivLUSolver>(reg)};
        detection_model::model_type sdo2(regs2, InterEyeDistanceNormalisation(ids, reye, leye));
        int seen_rows = 0;
        sdo2.train(x_gt, x0, Mat(), hog, [&](const Mat& cur) { seen_rows = cur.rows; }, comm, 0);
        sd_comm_destroy(comm);
        Mat dev2 = sdo2.test(x0, Mat(), hog);
        EXPECT_REL(0.0, cv::norm(dev, dev2, cv::NORM_L2) / cv::norm(dev, cv::NORM_L2), 1e-3);
        if (seen_rows != n) { std::printf("FAIL communicator route: callback saw %d rows\n", seen_rows); ++failures; }
    }
    // assemble a detection_model from the trained parts and run it
    detection_model trained(sdo, mean, ids, hp, reye, leye);
    auto lms = trained.detect(images[0], cv::Rect(20, 18, 110, 110));
    EXPECT_REL(dev.at<float>(0, 0), lms[0].coordinates[0], 1e-5);
}

static void test_hog_colour_frames_of_two_sizes(const char* model_path)
{
    // HogTransform over a grey frame and a colour frame of another size whose rows are padded (Mat::step() > 3 * cols): the
    // features must equal those of the same frames converted to grey on the host (OpenCV's BGR2GRAY fixed point)
    using namespace rcr;
    detection_model m = load_detection_model(model_path);
    Mat mean = m.get_mean();
    std::vector<std::string> ids;
    for (int i = 0; i < mean.cols / 2; ++i) ids.emplace_back(sd_model_landmark_id(m.native(), i));
    std::vector<std::string> reye{"37", "40"}, leye{"43", "46"};
    const int h0 = 70, w0 = 93, h1 = 61, w1 = 110;
    unsigned s = 777;
    auto noise = [&](int x, int y) { s = s * 1664525u + 1013904223u; return static_cast<unsigned char>(128 + 50 * std::sin(0.13 * x) * std::cos(0.09 * y) + ((s >> 24) & 31)); };
    Mat grey0(h0, w0, CV_8UC1);
    for (int y = 0; y < h0; ++y) for (int x = 0; x < w0; ++x) grey0.at<unsigned char>(y, x) = noise(x, y);
    Mat padded(h1, w1 + 7, CV_8UC3), grey1(h1, w1, CV_8UC1);
    for (int y = 0; y < h1; ++y)
        for (int x = 0; x < w1 + 7; ++x)
            for (int c = 0; c < 3; ++c) padded.ptr<unsigned char>(y)[3 * x + c] = noise(x + 40 * c, y);
    Mat colour1 = padded.colRange(0, w1);
    for (int y = 0; y < h1; ++y)
        for (int x = 0; x < w1; ++x) {
            const unsigned char* p = colour1.ptr<unsigned char>(y) + 3 * x;
            grey1.at<unsigned char>(y, x) = static_cast<unsigned char>((3735 * p[0] + 19235 * p[1] + 9798 * p[2] + (1 << 14)) >> 15);
        }
    std::vector<Mat> colour_frames{grey0, colour1}, grey_frames{grey0, grey1};
    std::vector<HoGParam> hp{{VlHogVariantUoctti, 3, 8, 4, 0.8f}};
    HogTransform hc(colour_frames, hp, ids, reye, leye), hg(grey_frames, hp, ids, reye, leye);
    const cv::Rect boxes[2] = {cv::Rect(12, 6, 64, 64), cv::Rect(-10, 4, 70, 70)};
    for (int i = 0; i < 2; ++i) {
        Mat x = align_mean(mean, boxes[i]);
        Mat a = hc(x, 0, i), b = hg(x, 0, i);
        int differ = a.cols == b.cols ? 0 : 1;
        for (int j = 0; j < a.cols && j < b.cols; ++j) differ += a.at<float>(0, j) != b.at<float>(0, j);
        if (differ) { std::printf("FAIL colour frame list: frame %d, %d features differ from the grey list\n", i, differ); ++failures; }
    }
}

int main(int argc, char** argv)
{
    try {
        test_regressors();
        test_optimiser();
        if (argc >= 2) test_rcr_device_route(argv[1]);
        if (argc >= 2) test_hog_colour_frames_of_two_sizes(argv[1]);
        if (argc >= 10) {
            rcr::detection_model m = rcr::load_detection_model(argv[1]);
            const int w = std::atoi(argv[3]), h = std::atoi(argv[4]);
            std::vector<unsigned char> raw(static_cast<size_t>(w) * h);
            std::ifstream f(argv[2], std::ios::binary);
            f.read(reinterpret_cast<char*>(raw.data()), raw.size());
            Mat image(h, w, CV_8UC1, raw.data());
            auto lms = m.detect(image, cv::Rect(std::atoi(argv[5]), std::atoi(argv[6]), std::atoi(argv[7]), std::atoi(argv[8])));
            std::printf("LANDMARKS");
            for (const auto& l : lms) std::printf(" %s %.6f %.6f", l.name.c_str(), l.coordinates[0], l.coordinates[1]);
            std::printf("\n");
            // the same frame as a colour image with B = G = R: cvtColor(BGR2GRAY) gives the grey frame back exactly, so the
            // colour routes (device-side sd_bgr2gray; box and previous-landmarks entry points) must return the same landmarks
            std::vector<unsigned char> bgr(raw.size() * 3);
            for (size_t i = 0; i < raw.size(); ++i) bgr[3 * i] = bgr[3 * i + 1] = bgr[3 * i + 2] = raw[i];
            Mat colour(h, w, CV_8UC3, bgr.data());
            const cv::Rect box(std::atoi(argv[5]), std::atoi(argv[6]), std::atoi(argv[7]), std::atoi(argv[8]));
            auto lms_c = m.detect(colour, box);
            auto lms_t = m.detect(colour, rcr::align_mean(m.get_mean(), box));
            for (size_t i = 0; i < lms.size(); ++i) {
                EXPECT_REL(lms[i].coordinates[0], lms_c[i].coordinates[0], 1e-6);
                EXPECT_REL(lms[i].coordinates[1], lms_c[i].coordinates[1], 1e-6);
                EXPECT_REL(lms[i].coordinates[0], lms_t[i].coordinates[0], 1e-6);
                EXPECT_REL(lms[i].coordinates[1], lms_t[i].coordinates[1], 1e-6);
            }
            rcr::save_detection_model(m, argv[9]);
            try {
                rcr::load_detection_model("/nonexistent/model.bin");
                std::printf("FAIL missing file did not throw\n");
                ++failures;
            } catch (const std::runtime_error& e) {
                std::printf("expected error: %s\n", e.what());
            }
        }
    } catch (const std::exception& e) {
        std::printf("EXCEPTION %s\n", e.what());
        return 2;
    }
    std::printf(failures ? "FAILED %d\n" : "ALL OK %d\n", failures);
    return failures ? 1 : 0;
}
