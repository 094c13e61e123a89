// The shell's dense HOG of multi-channel 8-bit or float frames (rcr::vl_hog) on frames of different sizes.
// Needs a GPU to run; compiling it (g++ -std=c++14) is part of the CPU test-suite.
//
//   test_vl_hog IN.bin OUT.bin CELL_SIZE NUM_BINS VARIANT BILINEAR
//     IN.bin : int32 num_frames, channels, dtype (0 = u8, 1 = f32); per frame int32 width, height, then its channel planes
//     OUT.bin: per frame int32 rows, cols, then rows x cols float32 (dd * hogH rows of hogW features)
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
    if (argc < 7) {
        std::printf("usage: test_vl_hog IN.bin OUT.bin CELL_SIZE NUM_BINS VARIANT BILINEAR\n");
        return 2;
    }
    int failures = 0;
    try {
        std::ifstream in(argv[1], std::ios::binary);
        auto get = [&in]() { int32_t v = 0; in.read(reinterpret_cast<char*>(&v), sizeof(v)); return v; };
        const int num_frames = get(), channels = get(), dtype = get();
        const int type = dtype == 0 ? CV_8UC1 : CV_32FC1;
        const int es = dtype == 0 ? 1 : 4;
        std::vector<std::vector<Mat>> frames(num_frames);
        for (int f = 0; f < num_frames; ++f) {
            const int w = get(), h = get();
            for (int c = 0; c < channels; ++c) {
                Mat padded(h, w + 32, type);
                Mat plane = padded.colRange(0, w);
                for (int y = 0; y < h; ++y) in.read(reinterpret_cast<char*>(plane.ptr<unsigned char>(y)), static_cast<std::streamsize>(w) * es);
                frames[f].push_back(plane);
            }
        }
        if (!in) throw std::runtime_error("truncated input");
        const int cs = std::atoi(argv[3]), K = std::atoi(argv[4]);
        const VlHogVariant variant = std::atoi(argv[5]) == 0 ? VlHogVariantDalalTriggs : VlHogVariantUoctti;
        const bool bilinear = std::atoi(argv[6]) != 0;
        const std::vector<Mat> hog = rcr::vl_hog(frames, variant, cs, K, bilinear);
        std::ofstream out(argv[2], std::ios::binary);
        for (size_t f = 0; f < hog.size(); ++f) {
            const int32_t rc[2] = {hog[f].rows, hog[f].cols};
            out.write(reinterpret_cast<const char*>(rc), sizeof(rc));
            for (int r = 0; r < hog[f].rows; ++r) out.write(reinterpret_cast<const char*>(hog[f].ptr<float>(r)), sizeof(float) * hog[f].cols);
        }
        // a frame of 3 x 3 pixels and planes of two types are refused
        const std::vector<std::vector<std::vector<Mat>>> bad = {
            {{Mat::zeros(3, 3, CV_8UC1)}},
            {{Mat::zeros(40, 40, CV_8UC1), Mat::zeros(40, 40, CV_32FC1)}},
        };
        for (const auto& b : bad) {
            try {
                rcr::vl_hog(b, variant, cs, K, bilinear);
                std::printf("FAIL an invalid frame did not throw\n");
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
