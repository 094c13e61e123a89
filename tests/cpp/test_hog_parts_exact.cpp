// The shell's star-model detector with the exact transform (rcr::vl_hog_part_detect of a model with unbounded = true).
// Needs a GPU to run; compiling it (g++ -std=c++14) is part of the CPU test-suite.
//
//   test_hog_parts_exact IN.bin OUT.bin CELL_SIZE NUM_BINS VARIANT THRESHOLD OVERLAP MAX_CANDIDATES MAX_DETECTIONS
//     IN.bin : int32 num_frames, per frame int32 width, height, channels and its packed rows; int32 num_scales, float64 scales;
//              int32 Q, P, fw, fh, pfw, pfh, pad_x, pad_y, part_pad_x, part_pad_y, R (ignored: the model is unbounded); Q roots of dd * fh x fw float32, Q bias
//              float32, Q * P parts of dd * pfh x pfw float32, Q * P anchors of 2 int32, Q * P deformations of 4 float32
//     OUT.bin: per frame int32 count, then per detection int32 x, y, w, h, float32 score, int32 filter, level, cell x, cell y,
//              and per part int32 u, v, float32 score, int32 x, y, w, h
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
    if (argc < 10) {
        std::printf("usage: test_hog_parts_exact IN.bin OUT.bin CELL_SIZE NUM_BINS VARIANT THRESHOLD OVERLAP MAX_CANDIDATES MAX_DETECTIONS\n");
        return 2;
    }
    int failures = 0;
    try {
        std::ifstream in(argv[1], std::ios::binary);
        auto get = [&in]() { int32_t v = 0; in.read(reinterpret_cast<char*>(&v), sizeof(v)); return v; };
        auto getf = [&in]() { float v = 0; in.read(reinterpret_cast<char*>(&v), sizeof(v)); return v; };
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
        const float threshold = static_cast<float>(std::atof(argv[6]));
        const double overlap = std::atof(argv[7]);
        const int max_candidates = std::atoi(argv[8]), max_detections = std::atoi(argv[9]);
        const int dd = variant == VlHogVariantUoctti ? 3 * K + 4 : 4 * K;
        rcr::hog_part_model model;
        const int Q = get(), P = get(), fw = get(), fh = get(), pfw = get(), pfh = get();
        model.pad_x = get(); model.pad_y = get(); model.part_pad_x = get(); model.part_pad_y = get();
        model.max_displacement = get();
        model.unbounded = true;
        auto filter = [&in, dd](int w, int h) {
            Mat f(dd * h, w, CV_32FC1);
            in.read(reinterpret_cast<char*>(f.ptr<float>(0)), static_cast<std::streamsize>(sizeof(float)) * dd * h * w);
            return f;
        };
        for (int q = 0; q < Q; ++q) model.root.push_back(filter(fw, fh));
        for (int q = 0; q < Q; ++q) model.bias.push_back(getf());
        model.parts.resize(Q);
        model.anchors.resize(Q);
        model.deformation.resize(Q);
        for (int q = 0; q < Q; ++q)
            for (int p = 0; p < P; ++p) model.parts[q].push_back(filter(pfw, pfh));
        for (int q = 0; q < Q; ++q)
            for (int p = 0; p < P; ++p) {
                const int ax = get(), ay = get();
                model.anchors[q].push_back({{ax, ay}});
            }
        for (int q = 0; q < Q; ++q)
            for (int p = 0; p < P; ++p) {
                std::array<float, 4> w;
                for (float& v : w) v = getf();
                model.deformation[q].push_back(w);
            }
        if (!in) throw std::runtime_error("truncated input");

        const std::vector<std::vector<rcr::hog_part_detection>> det =
            rcr::vl_hog_part_detect(frames, scales, model, variant, cs, K, threshold, overlap, max_candidates, max_detections);
        std::ofstream out(argv[2], std::ios::binary);
        for (const auto& list : det) {
            const int32_t n = static_cast<int32_t>(list.size());
            out.write(reinterpret_cast<const char*>(&n), sizeof(n));
            for (const rcr::hog_part_detection& d : list) {
                const rcr::hog_detection& r = d.detection;
                int32_t rec[9] = {r.box.x, r.box.y, r.box.width, r.box.height, 0, r.filter, r.level, r.cell_x, r.cell_y};
                std::memcpy(&rec[4], &r.score, sizeof(float));
                out.write(reinterpret_cast<const char*>(rec), sizeof(rec));
                for (const rcr::hog_part& p : d.parts) {
                    int32_t pr[7] = {p.u, p.v, 0, p.box.x, p.box.y, p.box.width, p.box.height};
                    std::memcpy(&pr[2], &p.score, sizeof(float));
                    out.write(reinterpret_cast<const char*>(pr), sizeof(pr));
                }
            }
        }
        // refused arguments throw
        try {
            rcr::vl_hog_part_detect(frames, {4.0}, model, variant, cs, K, threshold, overlap, max_candidates, max_detections);
            std::printf("FAIL a root scale of 4 did not throw\n");
            ++failures;
        } catch (const std::runtime_error& e) {
            std::printf("expected error: %s\n", e.what());
        }
        try {
            rcr::hog_part_model bad = model;
            bad.deformation[0][0][0] = 0.0f;                      // w0 = 0: the exact transform needs w0 > 0
            rcr::vl_hog_part_detect(frames, scales, bad, variant, cs, K, threshold, overlap, max_candidates, max_detections);
            std::printf("FAIL w0 = 0 did not throw\n");
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
