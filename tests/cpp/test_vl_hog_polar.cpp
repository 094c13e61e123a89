// The shell's dense HOG of caller-supplied gradient fields (rcr::vl_hog_polar) on fields of different sizes.
// Needs a GPU to run; compiling it (g++ -std=c++14) is part of the CPU test-suite.
//
//   test_vl_hog_polar IN.bin OUT.bin CELL_SIZE NUM_BINS VARIANT DIRECTED BILINEAR
//     IN.bin : int32 num_fields; per field int32 width, height, then the modulus plane and the angle plane (float32)
//     OUT.bin: per field int32 rows, cols, then rows x cols float32 (dd * hogH rows of hogW features)
// Each plane is held with a row step 32 elements longer than its pixels, so the row stride is the Mat's step, not its width.
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <vector>

#include "rcr/adaptive_vlhog.hpp"

using cv::Mat;

int main(int argc, char** argv)
{
    if (argc < 8) {
        std::printf("usage: test_vl_hog_polar IN.bin OUT.bin CELL_SIZE NUM_BINS VARIANT DIRECTED BILINEAR\n");
        return 2;
    }
    int failures = 0;
    try {
        std::ifstream in(argv[1], std::ios::binary);
        auto get = [&in]() { int32_t v = 0; in.read(reinterpret_cast<char*>(&v), sizeof(v)); return v; };
        auto plane = [&in](int w, int h) {
            Mat padded(h, w + 32, CV_32FC1);
            Mat p = padded.colRange(0, w);
            for (int y = 0; y < h; ++y) in.read(reinterpret_cast<char*>(p.ptr<float>(y)), static_cast<std::streamsize>(w) * 4);
            return p;
        };
        const int num_fields = get();
        std::vector<Mat> modulus, angle;
        for (int f = 0; f < num_fields; ++f) {
            const int w = get(), h = get();
            modulus.push_back(plane(w, h));
            angle.push_back(plane(w, h));
        }
        if (!in) throw std::runtime_error("truncated input");
        const int cs = std::atoi(argv[3]), K = std::atoi(argv[4]);
        const VlHogVariant variant = std::atoi(argv[5]) == 0 ? VlHogVariantDalalTriggs : VlHogVariantUoctti;
        const bool directed = std::atoi(argv[6]) != 0, bilinear = std::atoi(argv[7]) != 0;
        const std::vector<Mat> hog = rcr::vl_hog_polar(modulus, angle, variant, cs, K, directed, bilinear);
        std::ofstream out(argv[2], std::ios::binary);
        for (size_t f = 0; f < hog.size(); ++f) {
            const int32_t rc[2] = {hog[f].rows, hog[f].cols};
            out.write(reinterpret_cast<const char*>(rc), sizeof(rc));
            for (int r = 0; r < hog[f].rows; ++r) out.write(reinterpret_cast<const char*>(hog[f].ptr<float>(r)), sizeof(float) * hog[f].cols);
        }
        // a pair of different sizes, a field of another type, a 3 x 3 field, unpaired lists and a refused configuration throw
        struct Bad { std::vector<Mat> m, a; int cs, K; };
        const std::vector<Bad> bad = {
            {{Mat::zeros(40, 40, CV_32FC1)}, {Mat::zeros(40, 41, CV_32FC1)}, cs, K},
            {{Mat::zeros(40, 40, CV_8UC1)}, {Mat::zeros(40, 40, CV_32FC1)}, cs, K},
            {{Mat::zeros(3, 3, CV_32FC1)}, {Mat::zeros(3, 3, CV_32FC1)}, cs, K},
            {{Mat::zeros(40, 40, CV_32FC1), Mat::zeros(40, 40, CV_32FC1)}, {Mat::zeros(40, 40, CV_32FC1)}, cs, K},
            {{Mat::zeros(40, 40, CV_32FC1)}, {Mat::zeros(40, 40, CV_32FC1)}, 33, K},
            {{Mat::zeros(40, 40, CV_32FC1)}, {Mat::zeros(40, 40, CV_32FC1)}, cs, 17},
        };
        for (const Bad& b : bad) {
            try {
                rcr::vl_hog_polar(b.m, b.a, variant, b.cs, b.K, directed, bilinear);
                std::printf("FAIL an invalid field did not throw\n");
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
