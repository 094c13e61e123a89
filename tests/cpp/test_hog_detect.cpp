// The shell's sliding-window detector (rcr::vl_hog_detect).
// Needs a GPU to run; compiling it (g++ -std=c++14) is part of the CPU test-suite.
//
//   test_hog_detect IN.bin OUT.bin CELL_SIZE NUM_BINS VARIANT PAD_X PAD_Y THRESHOLD OVERLAP MAX_CANDIDATES MAX_DETECTIONS
//     IN.bin : int32 num_frames, per frame int32 width, height, channels and its packed rows; int32 num_scales, float64 scales;
//              int32 Q, fw, fh, then Q filters of dd * fh x fw float32; int32 has_bias, then Q float32
//     OUT.bin: per frame int32 count, then count records of int32 x, y, w, h, float32 score, int32 filter, level, cell x, cell y
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <vector>

#include "rcr/adaptive_vlhog.hpp"

using cv::Mat;

int main(int argc, char** argv)
{
    if (argc < 12) {
        std::printf("usage: test_hog_detect IN.bin OUT.bin CELL_SIZE NUM_BINS VARIANT PAD_X PAD_Y THRESHOLD OVERLAP MAX_CANDIDATES "
                    "MAX_DETECTIONS\n");
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
        const float threshold = static_cast<float>(std::atof(argv[8]));
        const double overlap = std::atof(argv[9]);
        const int max_candidates = std::atoi(argv[10]), max_detections = std::atoi(argv[11]);
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

        const std::vector<std::vector<rcr::hog_detection>> det = rcr::vl_hog_detect(frames, scales, filters, variant, cs, K, bias, pad_x,
                                                                                   pad_y, threshold, overlap, max_candidates, max_detections);
        std::ofstream out(argv[2], std::ios::binary);
        for (const auto& list : det) {
            const int32_t n = static_cast<int32_t>(list.size());
            out.write(reinterpret_cast<const char*>(&n), sizeof(n));
            for (const rcr::hog_detection& d : list) {
                int32_t rec[9] = {d.box.x, d.box.y, d.box.width, d.box.height, 0, d.filter, d.level, d.cell_x, d.cell_y};
                std::memcpy(&rec[4], &d.score, sizeof(float));
                out.write(reinterpret_cast<const char*>(rec), sizeof(rec));
            }
        }
        // refused arguments throw
        try {
            rcr::vl_hog_detect(frames, scales, filters, variant, cs, K, bias, pad_x, pad_y, threshold, 1.5, max_candidates, max_detections);
            std::printf("FAIL an overlap of 1.5 did not throw\n");
            ++failures;
        } catch (const std::runtime_error& e) {
            std::printf("expected error: %s\n", e.what());
        }
        try {
            rcr::vl_hog_detect(frames, scales, filters, variant, cs, K, bias, pad_x, pad_y, threshold, overlap, max_candidates,
                               max_candidates + 1);
            std::printf("FAIL max_detections above max_candidates did not throw\n");
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
