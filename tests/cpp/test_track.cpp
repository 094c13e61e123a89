// The shell's tracking step (rcr::detection_model::track) and box scores (rcr::hog_box_scores).
// Needs a GPU to run; compiling it (g++ -std=c++14) is part of the CPU test-suite.
//
//   test_track MODEL IN.bin OUT.bin CELL_SIZE NUM_BINS VARIANT THRESHOLD
//     IN.bin : int32 num_frames, per frame int32 width, height, channels and its packed rows; int32 T, T int32 frame indices,
//              T x 2L float32 previous landmarks; int32 fw, fh, dd * fh x fw float32 filter, float32 bias; int32 n, n int32 frame
//              indices and n x 4 int32 boxes for hog_box_scores
//     OUT.bin: T x 2L float32 landmarks, T x 4 int32 boxes, T float32 scores, T int32 alive, n float32 box scores
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <stdexcept>
#include <vector>

#include "rcr/model.hpp"

using cv::Mat;

int main(int argc, char** argv)
{
    if (argc < 8) {
        std::printf("usage: test_track MODEL IN.bin OUT.bin CELL_SIZE NUM_BINS VARIANT THRESHOLD\n");
        return 2;
    }
    int failures = 0;
    try {
        rcr::detection_model model = rcr::load_detection_model(argv[1]);
        const int P = 2 * sd_model_num_landmarks(model.native());
        std::ifstream in(argv[2], std::ios::binary);
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
        const int T = get();
        std::vector<int> face(T);
        for (int t = 0; t < T; ++t) face[t] = get();
        Mat previous(T, P, CV_32FC1);
        in.read(reinterpret_cast<char*>(previous.ptr<float>(0)), static_cast<std::streamsize>(sizeof(float)) * T * P);
        const int cs = std::atoi(argv[4]), K = std::atoi(argv[5]);
        const VlHogVariant variant = std::atoi(argv[6]) == 0 ? VlHogVariantDalalTriggs : VlHogVariantUoctti;
        const float threshold = static_cast<float>(std::atof(argv[7]));
        const int dd = variant == VlHogVariantUoctti ? 3 * K + 4 : 4 * K;
        const int fw = get(), fh = get();
        rcr::hog_filter filter;
        filter.filter = Mat(dd * fh, fw, CV_32FC1);
        in.read(reinterpret_cast<char*>(filter.filter.ptr<float>(0)), static_cast<std::streamsize>(sizeof(float)) * dd * fh * fw);
        in.read(reinterpret_cast<char*>(&filter.bias), sizeof(float));
        const int n = get();
        std::vector<int> box_frame(n);
        for (int k = 0; k < n; ++k) box_frame[k] = get();
        std::vector<cv::Rect> boxes;
        for (int k = 0; k < n; ++k) {
            const int x = get(), y = get(), w = get(), h = get();
            boxes.push_back(cv::Rect(x, y, w, h));
        }
        if (!in) throw std::runtime_error("truncated input");

        const rcr::tracked_faces tr = model.track(frames, face, previous, filter, variant, cs, K, threshold);
        const std::vector<float> scores = rcr::hog_box_scores(frames, box_frame, boxes, filter.filter, filter.bias, variant, cs, K);
        std::ofstream out(argv[3], std::ios::binary);
        for (int t = 0; t < T; ++t) out.write(reinterpret_cast<const char*>(tr.landmarks[t].ptr<float>(0)), static_cast<std::streamsize>(sizeof(float)) * P);
        for (int t = 0; t < T; ++t) {
            const int32_t b[4] = {tr.boxes[t].x, tr.boxes[t].y, tr.boxes[t].width, tr.boxes[t].height};
            out.write(reinterpret_cast<const char*>(b), sizeof(b));
        }
        out.write(reinterpret_cast<const char*>(tr.scores.data()), static_cast<std::streamsize>(sizeof(float)) * T);
        for (int t = 0; t < T; ++t) {
            const int32_t a = tr.alive[t] ? 1 : 0;
            out.write(reinterpret_cast<const char*>(&a), sizeof(a));
        }
        out.write(reinterpret_cast<const char*>(scores.data()), static_cast<std::streamsize>(sizeof(float)) * n);

        // refusals throw: a frame index out of range, previous rows of the wrong width, a box without width
        std::vector<int> bad = face;
        bad[0] = num_frames;
        try { model.track(frames, bad, previous, filter, variant, cs, K, threshold); ++failures; std::printf("bad index not refused\n"); }
        catch (const std::runtime_error&) {}
        try { model.track(frames, face, previous.colRange(0, P - 1), filter, variant, cs, K, threshold); ++failures; std::printf("bad rows not refused\n"); }
        catch (const std::runtime_error&) {}
        std::vector<cv::Rect> empty_box{cv::Rect(0, 0, 0, 5)};
        try { rcr::hog_box_scores(frames, {0}, empty_box, filter.filter, filter.bias, variant, cs, K); ++failures; std::printf("empty box not refused\n"); }
        catch (const std::runtime_error&) {}
    } catch (const std::exception& e) {
        std::printf("exception: %s\n", e.what());
        return 1;
    }
    if (failures) return 1;
    std::printf("ALL OK\n");
    return 0;
}
