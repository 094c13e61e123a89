// The shell's HOG pyramid and filter scores (rcr::vl_hog_pyramid, rcr::vl_hog_correlate).
// Needs a GPU to run; compiling it (g++ -std=c++14) is part of the CPU test-suite.
//
//   test_hog_filters IN.bin OUT.bin CELL_SIZE NUM_BINS VARIANT PAD_X PAD_Y
//     IN.bin : int32 num_frames, per frame int32 width, height, channels and its packed rows; int32 num_scales, float64 scales;
//              int32 Q, fw, fh, then Q filters of dd * fh x fw float32; int32 has_bias, then Q float32
//     OUT.bin: per frame and scale int32 rows, cols and rows x cols float32 (0, 0 for an empty level); then per frame and non-empty
//              level the scores of the filters on that level, int32 rows, cols and rows x cols float32
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <vector>

#include "rcr/adaptive_vlhog.hpp"

using cv::Mat;

static void put(std::ofstream& out, const Mat& m)
{
    const int32_t rc[2] = {m.empty() ? 0 : m.rows, m.empty() ? 0 : m.cols};
    out.write(reinterpret_cast<const char*>(rc), sizeof(rc));
    for (int r = 0; r < rc[0]; ++r) out.write(reinterpret_cast<const char*>(m.ptr<float>(r)), sizeof(float) * m.cols);
}

int main(int argc, char** argv)
{
    if (argc < 8) {
        std::printf("usage: test_hog_filters IN.bin OUT.bin CELL_SIZE NUM_BINS VARIANT PAD_X PAD_Y\n");
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
            Mat padded(h, w + 32, ch == 3 ? CV_8UC3 : CV_8UC1);   // a row step wider than the pixels
            Mat frame = padded.colRange(0, w);
            for (int y = 0; y < h; ++y) in.read(reinterpret_cast<char*>(frame.ptr<unsigned char>(y)), static_cast<std::streamsize>(w) * ch);
            frames.push_back(frame);
        }
        std::vector<double> scales(get());
        in.read(reinterpret_cast<char*>(scales.data()), static_cast<std::streamsize>(scales.size() * sizeof(double)));
        const int cs = std::atoi(argv[3]), K = std::atoi(argv[4]);
        const VlHogVariant variant = std::atoi(argv[5]) == 0 ? VlHogVariantDalalTriggs : VlHogVariantUoctti;
        const int pad_x = std::atoi(argv[6]), pad_y = std::atoi(argv[7]);
        const int dd = variant == VlHogVariantUoctti ? 3 * K + 4 : 4 * K;
        const int Q = get(), fw = get(), fh = get();
        std::vector<Mat> filters;
        for (int q = 0; q < Q; ++q) {
            Mat f(dd * fh, fw, CV_32FC1);
            in.read(reinterpret_cast<char*>(f.ptr<float>(0)), static_cast<std::streamsize>(sizeof(float)) * dd * fh * fw);
            filters.push_back(f);
        }
        std::vector<float> bias(get() ? Q : 0);
        in.read(reinterpret_cast<char*>(bias.data()), static_cast<std::streamsize>(bias.size() * sizeof(float)));
        if (!in) throw std::runtime_error("truncated input");

        const std::vector<std::vector<Mat>> pyr = rcr::vl_hog_pyramid(frames, scales, variant, cs, K);
        std::ofstream out(argv[2], std::ios::binary);
        for (const auto& levels : pyr)
            for (const Mat& m : levels) put(out, m);
        for (const auto& levels : pyr) {
            std::vector<Mat> maps;
            for (const Mat& m : levels)
                if (!m.empty()) maps.push_back(m);
            for (const Mat& s : rcr::vl_hog_correlate(maps, filters, variant, K, bias, pad_x, pad_y)) put(out, s);
        }
        // refused configurations throw
        try {
            rcr::vl_hog_pyramid(frames, std::vector<double>{5.0}, variant, cs, K);
            std::printf("FAIL a scale of 5 did not throw\n");
            ++failures;
        } catch (const std::runtime_error& e) {
            std::printf("expected error: %s\n", e.what());
        }
        try {
            rcr::vl_hog_correlate(std::vector<Mat>{Mat::zeros(dd * 4, 4, CV_32FC1)}, filters, variant, K, bias, fw, 0);
            std::printf("FAIL a pad of fw did not throw\n");
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
