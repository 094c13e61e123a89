// Host batch projections (feature_length / project_host, and RowwiseProjection over a per-row functor) through
// SupervisedDescentOptimiser::train / test / predict on the device route (sd_train_level_host_projected /
// sd_apply_level_host_projected).  Needs a GPU to run; compiling it (g++ -std=c++14) is part of the CPU test-suite.
//
//   test_host_projection
//     POSE      the pose example's projection through rowwise(...) against the plain-functor route: weights within 1e-3, the
//               final landmarks and the prediction of the hand-labelled frame within 1e-4 (the bars of the pose suite)
//     CHUNKS    a class with project_host trains in one chunk and with set_rows_per_chunk: the exact call sequence, chunked
//               against one chunk within 1e-4, two chunked runs and the communicator overload bit for bit, test == predict
//     RETHROWN  an exception of project_host, and of a functor inside rowwise(...), comes out of train() / test()
#include <cmath>
#include <cstdio>
#include <cstring>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "superviseddescent/superviseddescent.hpp"

using namespace superviseddescent;
using cv::Mat;

static double rel_err(const Mat& a, const Mat& b)
{
    double diff = 0, ref = 1e-30;
    for (int r = 0; r < b.rows; ++r)
        for (int c = 0; c < b.cols; ++c) {
            diff = std::fmax(diff, std::fabs(static_cast<double>(a.at<float>(r, c)) - b.at<float>(r, c)));
            ref = std::fmax(ref, std::fabs(static_cast<double>(b.at<float>(r, c))));
        }
    return diff / ref;
}

static bool same(const Mat& a, const Mat& b)
{
    if (a.rows != b.rows || a.cols != b.cols) return false;
    for (int r = 0; r < a.rows; ++r)
        if (std::memcmp(a.ptr<float>(r), b.ptr<float>(r), sizeof(float) * a.cols) != 0) return false;
    return true;
}

// ---- the pose example (tests/pose_example.py): 6 pose parameters -> 10 projected model points, normalised ---------------------
static const float kFaceModel[4][10] = {
    {-0.287526f, -0.11479f, -46.1668f, -18.926f, 19.2574f, 46.1914f, -23.7552f, -0.0753515f, 23.7138f, 0.125511f},
    {-2.0203f, -17.2056f, 34.7219f, 31.5432f, 31.5767f, 34.452f, -35.7461f, -28.3064f, -35.7886f, -44.7427f},
    {3.33725f, -13.5569f, -35.938f, -29.9641f, -30.229f, -36.1317f, -28.2573f, -12.8984f, -28.5949f, -17.1411f},
    {1.f, 1.f, 1.f, 1.f, 1.f, 1.f, 1.f, 1.f, 1.f, 1.f}};

struct M4 {
    float m[4][4];
};
static M4 identity()
{
    M4 r{};
    for (int i = 0; i < 4; ++i) r.m[i][i] = 1.f;
    return r;
}
static M4 mul(const M4& a, const M4& b)
{
    M4 r{};
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j)
            for (int k = 0; k < 4; ++k) r.m[i][j] += a.m[i][k] * b.m[k][j];
    return r;
}
// rotation by deg degrees in the (i, j) plane: [[c, -s], [s, c]] on rows / columns i, j
static M4 rotation(int i, int j, float deg)
{
    const float a = deg * 3.14159265358979f / 180.f, c = std::cos(a), s = std::sin(a);
    M4 r = identity();
    r.m[i][i] = c; r.m[i][j] = -s; r.m[j][i] = s; r.m[j][j] = c;
    return r;
}

struct PoseFunctor {
    Mat operator()(Mat p, size_t /*level*/, int /*index*/) const
    {
        const float focal = 1800.f;
        M4 t = identity();
        t.m[0][3] = p.at<float>(0, 3); t.m[1][3] = p.at<float>(0, 4); t.m[2][3] = p.at<float>(0, 5);
        const M4 model = mul(mul(mul(t, rotation(2, 0, p.at<float>(0, 1))), rotation(1, 2, p.at<float>(0, 0))), rotation(0, 1, p.at<float>(0, 2)));
        const float fovy = 2.f * std::atan(1000.f / (2.f * focal)) * 180.f / 3.14159265358979f;
        const float rad = fovy / 2.f * 3.14159265358979f / 180.f, cot = std::cos(rad) / std::sin(rad), n = 1.f, f = 5000.f;
        M4 persp{};
        persp.m[0][0] = cot; persp.m[1][1] = cot; persp.m[2][2] = -(n + f) / (f - n); persp.m[2][3] = -2 * n * f / (f - n); persp.m[3][2] = -1.f;
        const M4 pm = mul(persp, model);
        Mat out(1, 20, CV_32FC1);
        for (int k = 0; k < 10; ++k) {
            float clip[4];
            for (int i = 0; i < 4; ++i) {
                clip[i] = 0.f;
                for (int j = 0; j < 4; ++j) clip[i] += pm.m[i][j] * kFaceModel[j][k];
            }
            const float xs = (clip[0] / clip[3] + 1.f) * 500.f, ys = 1000.f - (clip[1] / clip[3] + 1.f) * 500.f;
            out.at<float>(0, k) = (xs - 500.f) / focal;
            out.at<float>(0, 10 + k) = (ys - 500.f) / focal;
        }
        return out;
    }
};

// ---- random features: cos(x W_l + b_l) and a last column of ones, written for a batch at once ---------------------------------
struct RandomFeatures {
    int P, F;
    std::vector<std::vector<float>> W, b;              // per level: P x F, F
    std::vector<std::pair<long long, int>>* calls;
    bool fail = false;
    RandomFeatures(int P_, int F_, int levels, std::vector<std::pair<long long, int>>* calls_) : P(P_), F(F_), calls(calls_)
    {
        unsigned s = 77;
        auto uniform = [&s]() { s = s * 1664525u + 1013904223u; return static_cast<float>(s >> 8) / 16777216.f; };
        for (int l = 0; l < levels; ++l) {
            W.emplace_back(static_cast<size_t>(P) * F);
            b.emplace_back(F);
            for (auto& w : W.back()) w = 2.f * uniform() - 1.f;
            for (auto& v : b.back()) v = 6.2831853f * uniform();
        }
    }
    int feature_length(size_t) const { return F + 1; }
    int project_host(size_t level, const float* x, int64_t ldx, int64_t first_row, int rows, float* out, int64_t ld)
    {
        calls->emplace_back(first_row, rows);
        if (fail) throw std::runtime_error("host projection failed on purpose");
        for (int r = 0; r < rows; ++r) {
            for (int j = 0; j < F; ++j) {
                float v = b[level][j];
                for (int p = 0; p < P; ++p) v += x[r * ldx + p] * W[level][static_cast<size_t>(p) * F + j];
                out[r * ld + j] = std::cos(v);
            }
            out[r * ld + F] = 1.f;
        }
        return 0;
    }
};

int main()
{
    int failures = 0;
    try {
        // ---- POSE -------------------------------------------------------------------------------------------------------------
        {
            static_assert(detail::is_host_batch_projection<RowwiseProjection<PoseFunctor>>::value &&
                              !detail::is_device_batch_projection<RowwiseProjection<PoseFunctor>>::value &&
                              !detail::takes_device_route<PoseFunctor>::value,
                          "rowwise(...) takes the host batch route, the plain functor its own");
            const int n = 500;
            unsigned s = 42;
            Mat x_tr(n, 6, CV_32FC1), x0 = Mat::zeros(n, 6, CV_32FC1), y_tr;
            for (int i = 0; i < n; ++i) {
                for (int j = 0; j < 6; ++j) {
                    s = s * 1664525u + 1013904223u;
                    x_tr.at<float>(i, j) = j < 3 ? 60.f * (static_cast<float>(s >> 8) / 16777216.f) - 30.f : 0.f;
                }
                x_tr.at<float>(i, 5) = -2000.f;
                x0.at<float>(i, 5) = -2000.f;
                y_tr.push_back(PoseFunctor()(x_tr.row(i), 0, i));
            }
            const Regulariser reg(Regulariser::RegularisationType::MatrixNorm, 2.0f, true);
            using Opt = SupervisedDescentOptimiser<LinearRegressor<>>;
            Opt plain({LinearRegressor<>(reg), LinearRegressor<>(reg), LinearRegressor<>(reg)});
            Opt piped({LinearRegressor<>(reg), LinearRegressor<>(reg), LinearRegressor<>(reg)});
            Mat xp, xh;
            plain.train(x_tr, x0, y_tr, PoseFunctor(), [&](const Mat& x) { xp = x.clone(); });
            piped.train(x_tr, x0, y_tr, rowwise(PoseFunctor(), 20), [&](const Mat& x) { xh = x.clone(); });
            double e_w = 0;
            for (int l = 0; l < 3; ++l) e_w = std::fmax(e_w, rel_err(piped.get_regressors()[l].x, plain.get_regressors()[l].x));
            const float lm[20] = {498, 504, 479, 498, 529, 553, 489, 503, 527, 503, 502, 513, 457, 465, 471, 471, 522, 522, 530, 536};
            Mat test_lms(1, 20, CV_32FC1), test_init = Mat::zeros(1, 6, CV_32FC1);
            for (int k = 0; k < 20; ++k) test_lms.at<float>(0, k) = (lm[k] - 500.f) / 1800.f;
            test_init.at<float>(0, 5) = -2000.f;
            const Mat pp = plain.predict(test_init, test_lms, PoseFunctor()), ph = piped.predict(test_init, test_lms, rowwise(PoseFunctor(), 20));
            const double e_x = rel_err(xh, xp), e_p = rel_err(ph, pp);
            std::printf("POSE rowwise vs plain functor: weights %.2e, final x %.2e, prediction %.2e; pitch/yaw/roll %.2f %.2f %.2f\n", e_w, e_x,
                        e_p, ph.at<float>(0, 0), ph.at<float>(0, 1), ph.at<float>(0, 2));
            if (!(e_w <= 1e-3 && e_x <= 1e-4 && e_p <= 1e-4)) { std::printf("FAIL pose: rowwise is not the plain-functor route\n"); ++failures; }
        }
        // ---- CHUNKS -----------------------------------------------------------------------------------------------------------
        {
            const int n = 3000, P = 10, F = 300;
            unsigned s = 9;
            auto uniform = [&s]() { s = s * 1664525u + 1013904223u; return static_cast<float>(s >> 8) / 16777216.f; };
            Mat x_gt(n, P, CV_32FC1), x0(n, P, CV_32FC1);
            for (int i = 0; i < n; ++i)
                for (int j = 0; j < P; ++j) {
                    x_gt.at<float>(i, j) = 2.f * uniform() - 1.f;
                    x0.at<float>(i, j) = x_gt.at<float>(i, j) + 0.6f * (uniform() - 0.5f);
                }
            std::vector<std::pair<long long, int>> calls;
            RandomFeatures rf(P, F, 2, &calls);
            static_assert(detail::is_host_batch_projection<RandomFeatures>::value && detail::takes_device_route<RandomFeatures>::value,
                          "a class with project_host takes the host batch route");
            const Regulariser reg(Regulariser::RegularisationType::MatrixNorm, 1.5f, false);
            using Opt = SupervisedDescentOptimiser<LinearRegressor<>>;
            auto make = [&reg]() { return Opt({LinearRegressor<>(reg), LinearRegressor<>(reg)}); };
            Opt one = make(), a = make(), b = make(), c = make();
            Mat x_one, x_a, x_b, x_c;
            one.train(x_gt, x0, Mat(), rf, [&](const Mat& x) { x_one = x.clone(); });
            const size_t calls_one = calls.size();
            calls.clear();
            a.set_rows_per_chunk(700);
            b.set_rows_per_chunk(700);
            a.train(x_gt, x0, Mat(), rf, [&](const Mat& x) { x_a = x.clone(); });
            std::vector<std::pair<long long, int>> want;
            for (int level = 0; level < 2; ++level) {
                for (int r0 = 0; r0 < n; r0 += 700) want.emplace_back(r0, n - r0 < 700 ? n - r0 : 700);   // the Gram pass
                for (int r0 = 0; r0 + 700 < n; r0 += 700) want.emplace_back(r0, 700);                    // the update pass
            }
            const bool seq = calls_one == 2 && calls == want;
            b.train(x_gt, x0, Mat(), rf, [&](const Mat& x) { x_b = x.clone(); });
            c.train(x_gt, x0, Mat(), rf, [&](const Mat& x) { x_c = x.clone(); }, nullptr, 0);     // the communicator overload, one rank
            double e_w = 0;
            bool repro = same(x_a, x_b) && same(x_c, x_one);
            for (int l = 0; l < 2; ++l) {
                e_w = std::fmax(e_w, rel_err(a.get_regressors()[l].x, one.get_regressors()[l].x));
                repro = repro && same(a.get_regressors()[l].x, b.get_regressors()[l].x) && same(c.get_regressors()[l].x, one.get_regressors()[l].x);
            }
            const double e_x = rel_err(x_a, x_one);
            one.set_rows_per_chunk(1000);
            const Mat t = one.test(x0, Mat(), rf), p = one.predict(x0, Mat(), rf);
            const bool applied = same(t, p) && t.rows == n && t.cols == P;
            std::printf("CHUNKS D = %d, 5 chunks vs one: weights %.2e, x %.2e; call sequence %s, reproducible %s, test == predict %s\n", F + 1, e_w,
                        e_x, seq ? "ok" : "WRONG", repro ? "yes" : "NO", applied ? "yes" : "NO");
            if (!(seq && repro && applied && e_w <= 1e-4 && e_x <= 1e-4)) { std::printf("FAIL chunks\n"); ++failures; }
            // ---- RETHROWN -----------------------------------------------------------------------------------------------------
            rf.fail = true;
            try {
                make().train(x_gt, x0, Mat(), rf);
                std::printf("FAIL train() returned although project_host threw\n");
                ++failures;
            } catch (const std::runtime_error& e) {
                const bool ok = std::string(e.what()) == "host projection failed on purpose";
                std::printf(ok ? "RETHROWN project_host\n" : "FAIL wrong exception: %s\n", e.what());
                failures += ok ? 0 : 1;
            }
            auto throwing = [](Mat, size_t, int i) -> Mat {
                if (i == 1234) throw std::runtime_error("functor failed on row 1234");
                return Mat::zeros(1, 301, CV_32FC1);
            };
            try {
                one.test(x0, Mat(), rowwise(throwing, 301));
                std::printf("FAIL test() returned although the functor threw\n");
                ++failures;
            } catch (const std::runtime_error& e) {
                const bool ok = std::string(e.what()) == "functor failed on row 1234";
                std::printf(ok ? "RETHROWN rowwise\n" : "FAIL wrong exception: %s\n", e.what());
                failures += ok ? 0 : 1;
            }
        }
    } catch (const std::exception& e) {
        std::printf("EXCEPTION %s\n", e.what());
        return 2;
    }
    std::printf(failures ? "FAILED %d\n" : "ALL OK %d\n", failures);
    return failures ? 1 : 0;
}
