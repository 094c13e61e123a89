// The shell's tracking steps and box scores on colour and float frames (rcr::detection_model::track and track_and_detect,
// rcr::hog_box_scores with multichannel, bilinear_orientations, float_frames and grey_images).
// Needs a GPU to run; compiling it (g++ -std=c++14) is part of the CPU test-suite.
//
//   test_track_colour MODEL IN.bin OUT.bin CELL_SIZE NUM_BINS THRESHOLD DETECT_THRESHOLD TRACK_OVERLAP MAX_DETECTIONS BILINEAR
//     IN.bin : int32 float_frames, int32 num_frames, per frame int32 width, height, channels and its packed rows (uint8, or
//              float32 when float_frames), then when float_frames per frame its packed uint8 grey rows; int32 T, T int32 frame
//              indices, T x 2L float32 previous landmarks; int32 fw, fh, dd * fh x fw float32 filter, float32 bias; int32 S, S
//              float64 scales; int32 D, D int32 listed frames
//     OUT.bin: track(): T x 2L float32 landmarks, T x 4 int32 boxes, T float32 scores, T int32 alive; hog_box_scores of those
//              boxes: T float32; track_and_detect(): int32 R, R x 2L float32 landmarks, R x 4 int32 boxes, R float32 scores,
//              R int32 alive, R int32 frames
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <stdexcept>
#include <vector>

#include "rcr/model.hpp"

using cv::Mat;

namespace {

void write_rows(std::ofstream& out, const std::vector<Mat>& landmarks, const std::vector<cv::Rect>& boxes, const std::vector<float>& scores,
                const std::vector<bool>& alive, int P)
{
    const size_t R = landmarks.size();
    for (size_t i = 0; i < R; ++i) out.write(reinterpret_cast<const char*>(landmarks[i].ptr<float>(0)), static_cast<std::streamsize>(sizeof(float)) * P);
    for (size_t i = 0; i < R; ++i) {
        const int32_t b[4] = {boxes[i].x, boxes[i].y, boxes[i].width, boxes[i].height};
        out.write(reinterpret_cast<const char*>(b), sizeof(b));
    }
    out.write(reinterpret_cast<const char*>(scores.data()), static_cast<std::streamsize>(sizeof(float) * R));
    for (size_t i = 0; i < R; ++i) {
        const int32_t a = alive[i] ? 1 : 0;
        out.write(reinterpret_cast<const char*>(&a), sizeof(a));
    }
}

}  // namespace

int main(int argc, char** argv)
{
    if (argc < 11) {
        std::printf("usage: test_track_colour MODEL IN.bin OUT.bin CELL_SIZE NUM_BINS THRESHOLD DETECT_THRESHOLD TRACK_OVERLAP "
                    "MAX_DETECTIONS BILINEAR\n");
        return 2;
    }
    int failures = 0;
    try {
        rcr::detection_model model = rcr::load_detection_model(argv[1]);
        const int P = 2 * sd_model_num_landmarks(model.native());
        std::ifstream in(argv[2], std::ios::binary);
        auto get = [&in]() { int32_t v = 0; in.read(reinterpret_cast<char*>(&v), sizeof(v)); return v; };
        const bool float_frames = get() != 0;
        const int num_frames = get();
        std::vector<Mat> frames, grey;
        for (int f = 0; f < num_frames; ++f) {
            const int w = get(), h = get(), ch = get();
            const int type = float_frames ? (ch == 3 ? CV_32FC3 : CV_32FC1) : (ch == 3 ? CV_8UC3 : CV_8UC1);
            Mat frame(h, w, type);
            in.read(reinterpret_cast<char*>(frame.ptr<unsigned char>(0)),
                    static_cast<std::streamsize>(w) * h * ch * (float_frames ? sizeof(float) : 1));
            frames.push_back(frame);
        }
        if (float_frames)
            for (int f = 0; f < num_frames; ++f) {
                Mat g(frames[f].rows, frames[f].cols, CV_8UC1);
                in.read(reinterpret_cast<char*>(g.ptr<unsigned char>(0)), static_cast<std::streamsize>(g.rows) * g.cols);
                grey.push_back(g);
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
        const bool bil = std::atoi(argv[10]) != 0;
        const std::vector<Mat>* grey_images = float_frames ? &grey : nullptr;

        std::ofstream out(argv[3], std::ios::binary);
        const rcr::tracked_faces t = model.track(frames, face, previous, filter, VlHogVariantUoctti, cs, K, threshold, true, bil, float_frames,
                                                 grey_images);
        write_rows(out, t.landmarks, t.boxes, t.scores, t.alive, P);
        const std::vector<float> sc = rcr::hog_box_scores(frames, face, t.boxes, filter.filter, filter.bias, VlHogVariantUoctti, cs, K, true,
                                                          bil, float_frames);
        out.write(reinterpret_cast<const char*>(sc.data()), static_cast<std::streamsize>(sizeof(float) * sc.size()));
        const rcr::track_step r = model.track_and_detect(frames, face, previous, filter, VlHogVariantUoctti, cs, K, threshold, scales, listed,
                                                         params, true, bil, float_frames, grey_images);
        const int32_t R = static_cast<int32_t>(r.landmarks.size());
        if (R != T + r.num_new) throw std::runtime_error("row count");
        out.write(reinterpret_cast<const char*>(&R), sizeof(R));
        write_rows(out, r.landmarks, r.boxes, r.scores, r.alive, P);
        for (int i = 0; i < R; ++i) {
            const int32_t f = r.frame[i];
            out.write(reinterpret_cast<const char*>(&f), sizeof(f));
        }

        // refusals throw: float frames without grey_images, bilinear orientations without multichannel, grey frames of other sizes
        if (float_frames) {
            try { model.track(frames, face, previous, filter, VlHogVariantUoctti, cs, K, threshold, true, bil, true); ++failures; std::printf("float frames without grey_images not refused\n"); }
            catch (const std::runtime_error&) {}
            std::vector<Mat> small;
            for (const Mat& g : grey) small.push_back(Mat(g.rows, g.cols - 1, CV_8UC1));
            try { model.track(frames, face, previous, filter, VlHogVariantUoctti, cs, K, threshold, true, bil, true, &small); ++failures; std::printf("grey frames of other sizes not refused\n"); }
            catch (const std::runtime_error&) {}
        }
        try { model.track(frames, face, previous, filter, VlHogVariantUoctti, cs, K, threshold, false, true); ++failures; std::printf("bilinear without multichannel not refused\n"); }
        catch (const std::runtime_error&) {}
        // hog_box_scores refuses the flags before anything else, with no boxes too
        try { rcr::hog_box_scores(frames, {}, {}, filter.filter, filter.bias, VlHogVariantUoctti, cs, K, false, true); ++failures; std::printf("hog_box_scores: bilinear without multichannel not refused\n"); }
        catch (const std::runtime_error&) {}
    } catch (const std::exception& e) {
        std::printf("exception: %s\n", e.what());
        return 1;
    }
    if (failures) return 1;
    std::printf("ALL OK\n");
    return 0;
}
