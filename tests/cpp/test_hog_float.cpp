// The shell's HOG calls on float frames: rcr::vl_hog_pyramid, vl_hog_detect, vl_hog_part_detect and train_hog_filter with
// multichannel and float_frames, on CV_32FC1 or CV_32FC3 frames.  Needs a GPU to run; compiling it (g++ -std=c++14) is part of
// the CPU test-suite.
//
//   test_hog_float IN.bin OUT.bin BILINEAR
//     IN.bin : int32 channels (1 or 3), int32 num_frames, per frame int32 width, height and its packed float32 rows of
//              interleaved channels; int32 num_scales, float64 scales;
//              int32 cell_size, num_bins, variant; int32 fw, fh, the filter (dd * fh x fw float32) and its float32 bias;
//              int32 P, pfw, pfh, R, the P part filters, P anchors (int32 ax, ay) and P deformations (float32 x 4);
//              int32 num_boxes, per box int32 frame, x, y, w, h; the sd_hog_train_param bytes
//     OUT.bin: per frame and scale int32 rows, cols and the level's floats; per frame int32 count and 9 int32 per detection;
//              per frame int32 count and 9 + 7 P int32 per part detection; the trained filter's floats, its float32 bias,
//              int32 num_negatives and the sd_hog_window bytes of each
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
    if (argc < 4) {
        std::printf("usage: test_hog_float IN.bin OUT.bin BILINEAR\n");
        return 2;
    }
    const bool bil = std::atoi(argv[3]) != 0;
    int failures = 0;
    try {
        std::ifstream in(argv[1], std::ios::binary);
        auto get = [&in]() { int32_t v = 0; in.read(reinterpret_cast<char*>(&v), sizeof(v)); return v; };
        auto getf = [&in]() { float v = 0; in.read(reinterpret_cast<char*>(&v), sizeof(v)); return v; };
        const int C = get(), num_frames = get();
        std::vector<Mat> frames;
        for (int f = 0; f < num_frames; ++f) {
            const int w = get(), h = get();
            Mat padded(h, w + 32, C == 3 ? CV_32FC3 : CV_32FC1);  // a row step wider than the pixels
            Mat frame = padded.colRange(0, w);
            for (int y = 0; y < h; ++y)
                in.read(reinterpret_cast<char*>(frame.ptr<float>(y)), static_cast<std::streamsize>(sizeof(float)) * w * C);
            frames.push_back(frame);
        }
        std::vector<double> scales(get());
        in.read(reinterpret_cast<char*>(scales.data()), static_cast<std::streamsize>(scales.size() * sizeof(double)));
        const int cs = get(), K = get();
        const VlHogVariant variant = get() == 0 ? VlHogVariantDalalTriggs : VlHogVariantUoctti;
        const int dd = variant == VlHogVariantUoctti ? 3 * K + 4 : 4 * K;
        auto filter = [&in, dd](int w, int h) {
            Mat f(dd * h, w, CV_32FC1);
            in.read(reinterpret_cast<char*>(f.ptr<float>(0)), static_cast<std::streamsize>(sizeof(float)) * dd * h * w);
            return f;
        };
        const int fw = get(), fh = get();
        const Mat root = filter(fw, fh);
        const float bias = getf();
        rcr::hog_part_model model;
        const int P = get(), pfw = get(), pfh = get();
        model.max_displacement = get();
        model.root.push_back(root);
        model.bias.push_back(bias);
        model.parts.resize(1);
        model.anchors.resize(1);
        model.deformation.resize(1);
        for (int p = 0; p < P; ++p) model.parts[0].push_back(filter(pfw, pfh));
        for (int p = 0; p < P; ++p) model.anchors[0].push_back({{get(), get()}});
        for (int p = 0; p < P; ++p) model.deformation[0].push_back({{getf(), getf(), getf(), getf()}});
        const int nb = get();
        std::vector<int> box_frame;
        std::vector<cv::Rect> boxes;
        for (int k = 0; k < nb; ++k) {
            box_frame.push_back(get());
            const int x = get(), y = get(), w = get(), h = get();
            boxes.push_back(cv::Rect(x, y, w, h));
        }
        sd_hog_train_param prm;
        in.read(reinterpret_cast<char*>(&prm), sizeof(prm));
        if (!in) throw std::runtime_error("truncated input");

        std::ofstream out(argv[2], std::ios::binary);
        auto put = [&out](int32_t v) { out.write(reinterpret_cast<const char*>(&v), sizeof(v)); };
        const std::vector<std::vector<Mat>> pyr = rcr::vl_hog_pyramid(frames, scales, variant, cs, K, true, bil, true);
        for (const auto& levels : pyr)
            for (const Mat& m : levels) {
                put(m.rows);
                put(m.cols);
                for (int r = 0; r < m.rows; ++r)
                    out.write(reinterpret_cast<const char*>(m.ptr<float>(r)), static_cast<std::streamsize>(sizeof(float)) * m.cols);
            }
        auto put_det = [&put](const rcr::hog_detection& d) {
            put(d.box.x); put(d.box.y); put(d.box.width); put(d.box.height);
            int32_t s;
            std::memcpy(&s, &d.score, sizeof(s));
            put(s); put(d.filter); put(d.level); put(d.cell_x); put(d.cell_y);
        };
        const auto det = rcr::vl_hog_detect(frames, scales, {root}, variant, cs, K, {bias}, 1, 0, -1.f, 0.5, 4096, 30, true, bil, true);
        for (const auto& list : det) {
            put(static_cast<int32_t>(list.size()));
            for (const auto& d : list) put_det(d);
        }
        std::vector<double> root_scales;
        for (double s : scales)
            if (s <= 2) root_scales.push_back(s);
        const auto parts = rcr::vl_hog_part_detect(frames, root_scales, model, variant, cs, K, -2.f, 0.5, 4096, 30, true, bil, true);
        for (const auto& list : parts) {
            put(static_cast<int32_t>(list.size()));
            for (const auto& d : list) {
                put_det(d.detection);
                for (const rcr::hog_part& p : d.parts) {
                    int32_t s;
                    std::memcpy(&s, &p.score, sizeof(s));
                    put(p.u); put(p.v); put(s); put(p.box.x); put(p.box.y); put(p.box.width); put(p.box.height);
                }
            }
        }
        const rcr::hog_filter hf = rcr::train_hog_filter(frames, box_frame, boxes, scales, variant, cs, K, fw, fh, 1, 0, prm, true, bil, true);
        for (int r = 0; r < hf.filter.rows; ++r)
            out.write(reinterpret_cast<const char*>(hf.filter.ptr<float>(r)), static_cast<std::streamsize>(sizeof(float)) * hf.filter.cols);
        out.write(reinterpret_cast<const char*>(&hf.bias), sizeof(float));
        put(static_cast<int32_t>(hf.negatives.size()));
        out.write(reinterpret_cast<const char*>(hf.negatives.data()), static_cast<std::streamsize>(sizeof(sd_hog_window) * hf.negatives.size()));
        // float_frames without multichannel, and 8-bit frames with float_frames, are refused
        try {
            rcr::vl_hog_pyramid(frames, scales, variant, cs, K, false, false, true);
            std::printf("FAIL float_frames without multichannel did not throw\n");
            ++failures;
        } catch (const std::runtime_error& e) {
            std::printf("expected error: %s\n", e.what());
        }
        try {
            rcr::vl_hog_pyramid({Mat(40, 48, CV_8UC3)}, scales, variant, cs, K, true, false, true);
            std::printf("FAIL 8-bit frames with float_frames did not throw\n");
            ++failures;
        } catch (const std::runtime_error& e) {
            std::printf("expected error: %s\n", e.what());
        }
    } catch (const std::exception& e) {
        std::printf("EXCEPTION %s\n", e.what());
        return 1;
    }
    if (failures) return 1;
    std::printf("ALL OK\n");
    return 0;
}
