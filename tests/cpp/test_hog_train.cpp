// The shell's HOG filter trainer (rcr::train_hog_filter).
// Needs a GPU to run; compiling it (g++ -std=c++14) is part of the CPU test-suite.
//
//   test_hog_train IN.bin OUT.bin
//     IN.bin : int32 num_frames, per frame int32 width, height, channels and its packed rows; int32 num_scales, float64 scales;
//              int32 num_boxes, per box int32 frame, x, y, w, h; int32 cell_size, num_bins, variant, fw, fh, pad_x, pad_y;
//              the sd_hog_train_param bytes
//     OUT.bin: the filter (dd * fh x fw float32), float32 bias, int32 rounds + 1 and the sd_hog_train_report bytes of each round,
//              int32 num_negatives and the sd_hog_window bytes of each
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <vector>

#include "rcr/adaptive_vlhog.hpp"

using cv::Mat;

int main(int argc, char** argv)
{
    if (argc < 3) {
        std::printf("usage: test_hog_train IN.bin OUT.bin\n");
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
        const int nb = get();
        std::vector<int> box_frame;
        std::vector<cv::Rect> boxes;
        for (int k = 0; k < nb; ++k) {
            box_frame.push_back(get());
            const int x = get(), y = get(), w = get(), h = get();
            boxes.push_back(cv::Rect(x, y, w, h));
        }
        const int cs = get(), K = get(), v = get(), fw = get(), fh = get(), pad_x = get(), pad_y = get();
        sd_hog_train_param p;
        in.read(reinterpret_cast<char*>(&p), sizeof(p));
        if (!in) throw std::runtime_error("truncated input");
        const VlHogVariant variant = v == 0 ? VlHogVariantDalalTriggs : VlHogVariantUoctti;

        const rcr::hog_filter hf = rcr::train_hog_filter(frames, box_frame, boxes, scales, variant, cs, K, fw, fh, pad_x, pad_y, p);
        std::ofstream out(argv[2], std::ios::binary);
        for (int r = 0; r < hf.filter.rows; ++r)
            out.write(reinterpret_cast<const char*>(hf.filter.ptr<float>(r)), static_cast<std::streamsize>(sizeof(float)) * hf.filter.cols);
        out.write(reinterpret_cast<const char*>(&hf.bias), sizeof(float));
        const int32_t nr = static_cast<int32_t>(hf.rounds.size()), nn = static_cast<int32_t>(hf.negatives.size());
        out.write(reinterpret_cast<const char*>(&nr), sizeof(nr));
        out.write(reinterpret_cast<const char*>(hf.rounds.data()), static_cast<std::streamsize>(sizeof(sd_hog_train_report)) * nr);
        out.write(reinterpret_cast<const char*>(&nn), sizeof(nn));
        out.write(reinterpret_cast<const char*>(hf.negatives.data()), static_cast<std::streamsize>(sizeof(sd_hog_window)) * nn);
        // refused arguments throw
        sd_hog_train_param bad = p;
        bad.lambda = 0.f;
        try {
            rcr::train_hog_filter(frames, box_frame, boxes, scales, variant, cs, K, fw, fh, pad_x, pad_y, bad);
            std::printf("FAIL lambda 0 did not throw\n");
            ++failures;
        } catch (const std::runtime_error& e) {
            std::printf("expected error: %s\n", e.what());
        }
        try {
            rcr::train_hog_filter(frames, std::vector<int>(box_frame.size(), num_frames), boxes, scales, variant, cs, K, fw, fh, pad_x,
                                  pad_y, p);
            std::printf("FAIL a box of a missing frame did not throw\n");
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
