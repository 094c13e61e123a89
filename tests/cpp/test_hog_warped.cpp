// Warped samples in the C++14 shells.  Needs a GPU to run; compiling it (g++ -std=c++14) is part of the CPU test-suite.
//
//   test_hog_warped MODEL IN OUT
//     IN (written by tests/test_cpp_hog_warped.py): photos, per-sample warps, landmarks and boxes, and each sample's virtual frame
//     V materialised by cv2.  Trains a two-level cascade with rcr::HogTransform's `warps` on shallow copies of the photos and on
//     the V copies, prints "WEIGHTS level L: d", "TEST: d", the same on the host route ("HOST ...") and one entry through the
//     functor ("FUNCTOR: d"); detect with warps against detect on the V copies ("DETECT: d"), all of which must be 0.  OUT
//     receives the warped detect's landmarks and the helpers' results for the Python side to compare bit for bit.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <fstream>
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

template <class T> static T get(std::ifstream& in)
{
    T v;
    in.read(reinterpret_cast<char*>(&v), sizeof(T));
    return v;
}

static Mat read_image(std::ifstream& in)
{
    const int h = get<int32_t>(in), w = get<int32_t>(in), ch = get<int32_t>(in);
    Mat m(h, w, ch == 3 ? CV_8UC3 : CV_8UC1);
    for (int y = 0; y < h; ++y) in.read(reinterpret_cast<char*>(m.ptr<unsigned char>(y)), static_cast<std::streamsize>(w) * ch);
    return m;
}

int main(int argc, char** argv)
{
    if (argc < 4) {
        std::printf("usage: test_hog_warped MODEL IN OUT\n");
        return 2;
    }
    int failures = 0;
    try {
        using namespace rcr;
        detection_model model = load_detection_model(argv[1]);
        const Mat mean = model.get_mean();
        const int L = mean.cols / 2;
        std::vector<std::string> ids;
        for (int i = 0; i < L; ++i) ids.emplace_back(sd_model_landmark_id(model.native(), i));
        std::ifstream in(argv[2], std::ios::binary);
        const int photos = get<int32_t>(in);
        std::vector<Mat> loaded;
        for (int i = 0; i < photos; ++i) loaded.push_back(read_image(in));
        const int n = get<int32_t>(in);
        std::vector<int> photo(n);
        std::vector<sd_sample_warp> warps(n);
        Mat x_gt(n, 2 * L, CV_32FC1), x0(n, 2 * L, CV_32FC1);
        std::vector<cv::Rect> boxes;
        for (int i = 0; i < n; ++i) photo[i] = get<int32_t>(in);
        for (int i = 0; i < n; ++i) {
            warp_matrix m;
            for (int k = 0; k < 6; ++k) m[k] = get<double>(in);
            const int w = get<int32_t>(in), h = get<int32_t>(in);
            warps[i] = make_warp(m, w, h);
        }
        for (int i = 0; i < n; ++i) in.read(reinterpret_cast<char*>(x_gt.ptr<float>(i)), sizeof(float) * 2 * L);
        for (int i = 0; i < n; ++i) in.read(reinterpret_cast<char*>(x0.ptr<float>(i)), sizeof(float) * 2 * L);
        for (int i = 0; i < n; ++i) {
            int32_t b[4];
            in.read(reinterpret_cast<char*>(b), sizeof(b));
            boxes.emplace_back(b[0], b[1], b[2], b[3]);
        }
        std::vector<Mat> vs, in_place;
        for (int i = 0; i < n; ++i) vs.push_back(read_image(in));
        if (!in) throw std::runtime_error("short input file");
        for (int i = 0; i < n; ++i) in_place.emplace_back(loaded[photo[i]]);

        const std::vector<std::string> reye{"37", "40"}, leye{"43", "46"};
        const std::vector<HoGParam> hp{{VlHogVariantUoctti, 3, 8, 4, 0.8f}, {VlHogVariantUoctti, 3, 6, 4, 0.5f}};
        HogTransform a_h(in_place, hp, ids, reye, leye, {}, warps), b_h(vs, hp, ids, reye, leye);
        const Regulariser reg(Regulariser::RegularisationType::MatrixNorm, 1.5f, false);
        using Opt = SupervisedDescentOptimiser<LinearRegressor<>, InterEyeDistanceNormalisation>;
        Opt a({LinearRegressor<>(reg), LinearRegressor<>(reg)}, InterEyeDistanceNormalisation(ids, reye, leye));
        Opt b({LinearRegressor<>(reg), LinearRegressor<>(reg)}, InterEyeDistanceNormalisation(ids, reye, leye));
        a.train(x_gt, x0, Mat(), a_h);
        b.train(x_gt, x0, Mat(), b_h);
        std::printf("FRAMES warped %d copies %d\n", a_h.num_frames(), b_h.num_frames());
        if (a_h.num_frames() != photos || !a_h.on_device() || !b_h.on_device()) { std::printf("FAIL frame counts or route\n"); ++failures; }
        for (size_t level = 0; level < 2; ++level) {
            const double e = max_abs_diff(a.get_regressors()[level].x, b.get_regressors()[level].x);
            std::printf("WEIGHTS level %zu: %.3e\n", level, e);
            if (e != 0.0) { std::printf("FAIL level %zu: weights differ\n", level); ++failures; }
        }
        const double d = max_abs_diff(a.test(x0, Mat(), a_h), b.test(x0, Mat(), b_h));
        std::printf("TEST: %.3e\n", d);
        if (d != 0.0) { std::printf("FAIL test() differs\n"); ++failures; }
        HogTransform::device_frame_share() = 0.0;
        HogTransform on_host(in_place, hp, ids, reye, leye, {}, warps);
        Opt h({LinearRegressor<>(reg), LinearRegressor<>(reg)}, InterEyeDistanceNormalisation(ids, reye, leye));
        h.train(x_gt, x0, Mat(), on_host);
        HogTransform::device_frame_share() = 0.5;
        if (on_host.on_device()) { std::printf("FAIL host route not taken\n"); ++failures; }
        for (size_t level = 0; level < 2; ++level) {
            const double e = max_abs_diff(b.get_regressors()[level].x, h.get_regressors()[level].x);
            std::printf("HOST WEIGHTS level %zu: %.3e\n", level, e);
            if (e != 0.0) { std::printf("FAIL level %zu: host-route weights differ\n", level); ++failures; }
        }
        const double dh = max_abs_diff(b.test(x0, Mat(), b_h), h.test(x0, Mat(), on_host));
        std::printf("HOST TEST: %.3e\n", dh);
        if (dh != 0.0) { std::printf("FAIL host-route test() differs\n"); ++failures; }
        const int e = n / 2 + 1;
        const double f = max_abs_diff(a_h(x0.row(e), 0, e), b_h(x0.row(e), 0, e));
        std::printf("FUNCTOR: %.3e\n", f);
        if (f != 0.0) { std::printf("FAIL functor differs\n"); ++failures; }

        // detect: warped against the V copies (face i in V i)
        std::vector<int> own(n);
        for (int i = 0; i < n; ++i) own[i] = i;
        const std::vector<Mat> got = model.detect(loaded, photo, boxes, warps), want = model.detect(vs, own, boxes);
        const std::vector<Mat> got_init = model.detect(loaded, photo, x0, warps), want_init = model.detect(vs, own, x0);
        double dd = 0.0;
        for (int i = 0; i < n; ++i) dd = std::max({dd, max_abs_diff(got[i], want[i]), max_abs_diff(got_init[i], want_init[i])});
        std::printf("DETECT: %.3e\n", dd);
        if (dd != 0.0) { std::printf("FAIL warped detect differs\n"); ++failures; }

        // results for the Python side: detect landmarks, rotation_warp of a few (centre, angle, scale), the inverse of every warp
        // and x0 carried to the photo
        std::ofstream out(argv[3], std::ios::binary);
        for (int i = 0; i < n; ++i) out.write(reinterpret_cast<const char*>(got[i].ptr<float>(0)), sizeof(float) * 2 * L);
        const double rot[][4] = {{0, 0, 0, 1}, {320.5, 240.25, 30, 1}, {-17, 1000, -45, 1.7}, {61.5, 40.25, 180, 0.25}, {100, 80, 721, 4}};
        for (const auto& r : rot) {
            const warp_matrix m = rotation_warp(r[0], r[1], r[2], r[3]);
            out.write(reinterpret_cast<const char*>(m.data()), sizeof(double) * 6);
        }
        std::vector<warp_matrix> ms;
        for (int i = 0; i < n; ++i) {
            warp_matrix m;
            std::copy(warps[i].m, warps[i].m + 6, m.begin());
            ms.push_back(m);
            const warp_matrix inv = invert_warp(m);
            out.write(reinterpret_cast<const char*>(inv.data()), sizeof(double) * 6);
        }
        const Mat back = warp_landmarks(x0, ms);
        for (int i = 0; i < n; ++i) out.write(reinterpret_cast<const char*>(back.ptr<float>(i)), sizeof(float) * 2 * L);
    } catch (const std::exception& ex) {
        std::printf("EXCEPTION %s\n", ex.what());
        return 2;
    }
    std::printf(failures ? "FAILED %d\n" : "ALL OK %d\n", failures);
    return failures ? 1 : 0;
}
