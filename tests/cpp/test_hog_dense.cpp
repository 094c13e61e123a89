// The shell's dense HOG of whole frames (rcr::hog_dense) on frames of different sizes, grey or colour.
// Needs a GPU to run; compiling it (g++ -std=c++14) is part of the CPU test-suite.
//
//   test_hog_dense IN.bin OUT.bin CELL_SIZE NUM_BINS VARIANT
//     IN.bin : int32 num_frames, per frame int32 width, height, channels and its packed rows
//     OUT.bin: per frame int32 rows, cols, then rows x cols float32 (dd * hogH rows of hogW features)
// Each frame is held with a row step 32 bytes longer than its pixels, so the row stride is the Mat's step, not its width.
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <vector>

#include "rcr/adaptive_vlhog.hpp"

using cv::Mat;

int main(int argc, char** argv)
{
    if (argc < 6) {
        std::printf("usage: test_hog_dense IN.bin OUT.bin CELL_SIZE NUM_BINS VARIANT\n");
        return 2;
    }
    int failures = 0;
    try {
        std::ifstream in(argv[1], std::ios::binary);
        auto get = [&in]() { int32_t v = 0; in.read(reinterpret_cast<char*>(&v), sizeof(v)); return v; };
        const int num_frames = get();
        std::vector<Mat> frames;
        for (int f = 0; f < num_frames; ++f) {
            const int w = get(), h = get(), ch = get();
            Mat padded(h, w + 32, ch == 3 ? CV_8UC3 : CV_8UC1);
            Mat frame = padded.colRange(0, w);
            for (int y = 0; y < h; ++y) in.read(reinterpret_cast<char*>(frame.ptr<unsigned char>(y)), static_cast<std::streamsize>(w) * ch);
            frames.push_back(frame);
        }
        if (!in) throw std::runtime_error("truncated input");
        const int cs = std::atoi(argv[3]), K = std::atoi(argv[4]);
        const VlHogVariant variant = std::atoi(argv[5]) == 0 ? VlHogVariantDalalTriggs : VlHogVariantUoctti;
        const std::vector<Mat> hog = rcr::hog_dense(frames, variant, cs, K);
        std::ofstream out(argv[2], std::ios::binary);
        for (size_t f = 0; f < hog.size(); ++f) {
            const int32_t rc[2] = {hog[f].rows, hog[f].cols};
            out.write(reinterpret_cast<const char*>(rc), sizeof(rc));
            for (int r = 0; r < hog[f].rows; ++r) out.write(reinterpret_cast<const char*>(hog[f].ptr<float>(r)), sizeof(float) * hog[f].cols);
        }
        // a frame of 3 x 3 pixels is refused (hog.c:545-546)
        try {
            rcr::hog_dense(std::vector<Mat>{Mat::zeros(3, 3, CV_8UC1)}, variant, cs, K);
            std::printf("FAIL a 3 x 3 frame did not throw\n");
            ++failures;
        } catch (const std::runtime_error& e) {
            std::printf("expected error: %s\n", e.what());
        }
    } catch (const std::exception& e) {
        std::printf("EXCEPTION %s\n", e.what());
        return 2;
    }
    std::printf(failures ? "FAILED %d\n" : "ALL OK %d\n", failures);
    return failures ? 1 : 0;
}
