// The shell's aligned face chips (rcr::face_chips).  Needs a GPU to run; compiling it (g++ -std=c++14) is part of the CPU
// test-suite.
//
//   test_face_chips MODEL IN.bin OUT.bin CHIP_WIDTH CHIP_HEIGHT PADDING [LANDMARK_ID ...]
//     IN.bin : int32 float_frames, int32 num_frames, per frame int32 width, height, channels and its packed rows (uint8, or float32
//              when float_frames); int32 N, N int32 frame indices, N x 2L float32 landmarks
//     OUT.bin: N chips (packed rows), N x 6 float64 chip_to_frame, N x 6 float64 frame_to_chip, N int32 valid
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <stdexcept>
#include <string>
#include <vector>

#include "rcr/model.hpp"

using cv::Mat;

namespace {

template <class F>
bool throws(F f)
{
    try {
        f();
    } catch (const std::runtime_error&) {
        return true;
    }
    return false;
}

}  // namespace

int main(int argc, char** argv)
{
    if (argc < 7) {
        std::printf("usage: test_face_chips MODEL IN.bin OUT.bin CHIP_WIDTH CHIP_HEIGHT PADDING [LANDMARK_ID ...]\n");
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
        std::vector<Mat> frames;
        for (int f = 0; f < num_frames; ++f) {
            const int w = get(), h = get(), c = get();
            const int type = float_frames ? (c == 3 ? CV_32FC3 : CV_32FC1) : (c == 3 ? CV_8UC3 : CV_8UC1);
            Mat m(h, w, type);
            in.read(reinterpret_cast<char*>(m.ptr<unsigned char>(0)), static_cast<std::streamsize>(m.step() * h));
            frames.push_back(m);
        }
        const int N = get();
        std::vector<int> face(N);
        for (int& v : face) v = get();
        Mat lms(N, P, CV_32FC1);
        in.read(reinterpret_cast<char*>(lms.ptr<float>(0)), static_cast<std::streamsize>(sizeof(float)) * N * P);
        const int cw = std::atoi(argv[4]), ch = std::atoi(argv[5]);
        const double padding = std::atof(argv[6]);
        std::vector<std::string> ids;
        for (int a = 7; a < argc; ++a) ids.push_back(argv[a]);

        const rcr::face_chip_set r = rcr::face_chips(frames, face, lms, model, cw, ch, padding, ids);
        if (static_cast<int>(r.chips.size()) != N || static_cast<int>(r.valid.size()) != N) {
            std::printf("FAIL: %zu chips for %d faces\n", r.chips.size(), N);
            ++failures;
        }
        std::ofstream out(argv[3], std::ios::binary);
        for (const Mat& c : r.chips) out.write(reinterpret_cast<const char*>(c.ptr<unsigned char>(0)), static_cast<std::streamsize>(c.step() * c.rows));
        for (const auto& m : r.chip_to_frame) out.write(reinterpret_cast<const char*>(m.data()), sizeof(double) * 6);
        for (const auto& m : r.frame_to_chip) out.write(reinterpret_cast<const char*>(m.data()), sizeof(double) * 6);
        for (bool v : r.valid) {
            const int32_t b = v ? 1 : 0;
            out.write(reinterpret_cast<const char*>(&b), sizeof(b));
        }

        // refused arguments throw
        std::vector<int> bad_face = face;
        bad_face[0] = num_frames;
        const struct { const char* what; bool ok; } cases[] = {
            {"frame index out of range", throws([&] { rcr::face_chips(frames, bad_face, lms, model, cw, ch, padding, ids); })},
            {"unknown landmark id", throws([&] { rcr::face_chips(frames, face, lms, model, cw, ch, padding, {"no-such-id", "x"}); })},
            {"one landmark", throws([&] { rcr::face_chips(frames, face, lms, model, cw, ch, padding, {std::string(sd_model_landmark_id(model.native(), 0))}); })},
            {"chip width 0", throws([&] { rcr::face_chips(frames, face, lms, model, 0, ch, padding, ids); })},
            {"padding -0.5", throws([&] { rcr::face_chips(frames, face, lms, model, cw, ch, -0.5, ids); })},
            {"landmarks of the wrong width", throws([&] { rcr::face_chips(frames, face, lms.colRange(0, P - 2), model, cw, ch, padding, ids); })},
        };
        for (const auto& c : cases)
            if (!c.ok) {
                std::printf("FAIL: %s did not throw\n", c.what);
                ++failures;
            }
    } catch (const std::exception& e) {
        std::printf("FAIL: %s\n", e.what());
        return 1;
    }
    if (failures) return 1;
    std::printf("ALL OK\n");
    return 0;
}
