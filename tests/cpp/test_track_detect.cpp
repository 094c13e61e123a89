// The shell's tracking step with the detector inside it (rcr::detection_model::track_and_detect).
// Needs a GPU to run; compiling it (g++ -std=c++14) is part of the CPU test-suite.
//
//   test_track_detect MODEL IN.bin OUT.bin CELL_SIZE NUM_BINS THRESHOLD DETECT_THRESHOLD TRACK_OVERLAP MAX_DETECTIONS
//     IN.bin : int32 num_frames, per frame int32 width, height, channels and its packed rows; int32 T, T int32 frame indices,
//              T x 2L float32 previous landmarks; int32 fw, fh, dd * fh x fw float32 filter, float32 bias; int32 S, S float64
//              scales; int32 D, D int32 listed frames
//     OUT.bin: int32 R (T + new rows), R x 2L float32 landmarks, R x 4 int32 boxes, R float32 scores, R int32 alive, R int32 frames
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
    if (argc < 10) {
        std::printf("usage: test_track_detect MODEL IN.bin OUT.bin CELL_SIZE NUM_BINS THRESHOLD DETECT_THRESHOLD TRACK_OVERLAP MAX_DETECTIONS\n");
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
            Mat frame(h, w, ch == 3 ? CV_8UC3 : CV_8UC1);
            in.read(reinterpret_cast<char*>(frame.ptr<unsigned char>(0)), static_cast<std::streamsize>(w) * h * ch);
            frames.push_back(frame);
        }
        const int T = get();
        std::vector<int> face(T);
        for (int t = 0; t < T; ++t) face[t] = get();
        Mat previous(T, P, CV_32FC1);
        if (T) in.read(reinterpret_cast<char*>(previous.ptr<float>(0)), static_cast<std::streamsize>(sizeof(float)) * T * P);
        const int cs = std::atoi(argv[4]), K = std::atoi(argv[5]), dd = 3 * K + 4;
        const int fw = get(), fh = get();
        rcr::hog_filter filter;
        filter.filter = Mat(dd * fh, fw, CV_32FC1);
        in.read(reinterpret_cast<char*>(filter.filter.ptr<float>(0)), static_cast<std::streamsize>(sizeof(float)) * dd * fh * fw);
        in.read(reinterpret_cast<char*>(&filter.bias), sizeof(float));
        std::vector<double> scales(get());
        in.read(reinterpret_cast<char*>(scales.data()), static_cast<std::streamsize>(sizeof(double) * scales.size()));
        std::vector<int> listed(get());
        for (auto& v : listed) v = get();
        if (!in) throw std::runtime_error("truncated input");
        rcr::track_detect_params params;
        params.detect_threshold = static_cast<float>(std::atof(argv[7]));
        params.track_overlap = std::atof(argv[8]);
        params.max_detections = std::atoi(argv[9]);
        const float threshold = static_cast<float>(std::atof(argv[6]));

        const rcr::track_step r = model.track_and_detect(frames, face, previous, filter, VlHogVariantUoctti, cs, K, threshold, scales, listed,
                                                         params);
        const int32_t R = static_cast<int32_t>(r.landmarks.size());
        if (R != T + r.num_new) throw std::runtime_error("row count");
        std::ofstream out(argv[3], std::ios::binary);
        out.write(reinterpret_cast<const char*>(&R), sizeof(R));
        for (int i = 0; i < R; ++i) out.write(reinterpret_cast<const char*>(r.landmarks[i].ptr<float>(0)), static_cast<std::streamsize>(sizeof(float)) * P);
        for (int i = 0; i < R; ++i) {
            const int32_t b[4] = {r.boxes[i].x, r.boxes[i].y, r.boxes[i].width, r.boxes[i].height};
            out.write(reinterpret_cast<const char*>(b), sizeof(b));
        }
        out.write(reinterpret_cast<const char*>(r.scores.data()), static_cast<std::streamsize>(sizeof(float)) * R);
        for (int i = 0; i < R; ++i) {
            const int32_t a = r.alive[i] ? 1 : 0;
            out.write(reinterpret_cast<const char*>(&a), sizeof(a));
        }
        for (int i = 0; i < R; ++i) {
            const int32_t f = r.frame[i];
            out.write(reinterpret_cast<const char*>(&f), sizeof(f));
        }

        // refusals throw: a frame listed twice, a listed frame out of range
        try { model.track_and_detect(frames, face, previous, filter, VlHogVariantUoctti, cs, K, threshold, scales, {0, 0}, params); ++failures; std::printf("repeated frame not refused\n"); }
        catch (const std::runtime_error&) {}
        try { model.track_and_detect(frames, face, previous, filter, VlHogVariantUoctti, cs, K, threshold, scales, {num_frames}, params); ++failures; std::printf("bad frame not refused\n"); }
        catch (const std::runtime_error&) {}
    } catch (const std::exception& e) {
        std::printf("exception: %s\n", e.what());
        return 1;
    }
    if (failures) return 1;
    std::printf("ALL OK\n");
    return 0;
}
