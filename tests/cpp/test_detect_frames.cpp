// The shell's detect overloads for several faces in frames of different sizes, grey or colour
// (rcr::detection_model::detect(images, face_image, faceboxes) and detect(images, face_image, initialisations)).
// Needs a GPU to run; compiling it (g++ -std=c++14) is part of the CPU test-suite.
//
//   test_detect_frames MODEL IN.bin OUT.bin
//     IN.bin : int32 num_frames, per frame int32 width, height, channels and its packed rows;
//              int32 num_faces, per face int32 frame, x, y, w, h
//     OUT.bin: num_faces x 2L float32 landmarks of detect(images, face_image, faceboxes)
// Each frame is held with a row step 32 bytes longer than its pixels, so the row stride is the Mat's step, not its width.
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <vector>

#include "rcr/model.hpp"

using cv::Mat;

static int failures = 0;

static bool same(const Mat& a, const Mat& b)
{
    return a.cols == b.cols && std::memcmp(a.ptr<float>(0), b.ptr<float>(0), sizeof(float) * a.cols) == 0;
}

int main(int argc, char** argv)
{
    if (argc < 4) {
        std::printf("usage: test_detect_frames MODEL IN.bin OUT.bin\n");
        return 2;
    }
    try {
        std::ifstream in(argv[2], std::ios::binary);
        auto get = [&in]() { int32_t v = 0; in.read(reinterpret_cast<char*>(&v), sizeof(v)); return v; };
        const int num_frames = get();
        std::vector<Mat> frames;
        for (int f = 0; f < num_frames; ++f) {
            const int w = get(), h = get(), ch = get();
            const int type = ch == 3 ? CV_8UC3 : CV_8UC1;
            Mat padded(h, w + 32, type);
            Mat frame = padded.colRange(0, w);
            for (int y = 0; y < h; ++y) in.read(reinterpret_cast<char*>(frame.ptr<unsigned char>(y)), static_cast<std::streamsize>(w) * ch);
            frames.push_back(frame);
        }
        const int num_faces = get();
        std::vector<int> face_image(num_faces);
        std::vector<cv::Rect> boxes(num_faces);
        for (int i = 0; i < num_faces; ++i) {
            face_image[i] = get();
            const int x = get(), y = get(), w = get(), h = get();
            boxes[i] = cv::Rect(x, y, w, h);
        }
        if (!in) throw std::runtime_error("truncated input");

        rcr::detection_model m = rcr::load_detection_model(argv[1]);
        const std::vector<Mat> lms = m.detect(frames, face_image, boxes);
        // tracking: starting from align_mean(box) is the box route
        const Mat mean = m.get_mean();
        Mat x0(num_faces, mean.cols, CV_32FC1);
        for (int i = 0; i < num_faces; ++i) {
            const Mat a = rcr::align_mean(mean, boxes[i]);
            std::memcpy(x0.ptr<float>(i), a.ptr<float>(0), sizeof(float) * mean.cols);
        }
        const std::vector<Mat> tracked = m.detect(frames, face_image, x0);
        for (int i = 0; i < num_faces; ++i) {
            if (!same(lms[i], tracked[i])) { std::printf("FAIL face %d: initialisation route differs from the box route\n", i); ++failures; }
            // one frame, one face: the single-image entry point
            const auto single = m.detect(frames[face_image[i]], boxes[i]);
            for (size_t l = 0; l < single.size(); ++l)
                if (single[l].coordinates[0] != lms[i].at<float>(0, static_cast<int>(l)) ||
                    single[l].coordinates[1] != lms[i].at<float>(0, static_cast<int>(l + single.size()))) {
                    std::printf("FAIL face %d landmark %zu: single-frame detect differs\n", i, l);
                    ++failures;
                    break;
                }
        }
        std::ofstream out(argv[3], std::ios::binary);
        for (const Mat& r : lms) out.write(reinterpret_cast<const char*>(r.ptr<float>(0)), sizeof(float) * r.cols);
        // a face that refers to a frame that does not exist is refused
        try {
            m.detect(frames, std::vector<int>{num_frames}, std::vector<cv::Rect>{boxes[0]});
            std::printf("FAIL an out-of-range frame index did not throw\n");
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
