// H100 drop-in for the reference's include/superviseddescent/regressors.hpp.
//
// Same names and call signatures: Regressor (regressors.hpp:43-77), Regulariser (:87-169),
// PartialPivLUSolver (:180-235), ColPivHouseholderQRSolver (:245-306), LinearRegressor<Solver>
// (:318-400, public member `x`).  The arithmetic is NOT here: Solver::solve forwards to sd_learn and
// predict/test to sd_predict / sd_test_residual of libsd_b200.so (hand-written sm_90a kernels);
// there is no CPU path.
#pragma once

#include <iostream>
#include <limits>
#include <stdexcept>
#include <string>
#include <utility>

#include "sd_b200/device.hpp"

namespace superviseddescent {

class Regressor {
public:
    virtual ~Regressor() {}
    virtual bool learn(cv::Mat data, cv::Mat labels) = 0;
    virtual double test(cv::Mat data, cv::Mat labels) = 0;
    virtual cv::Mat predict(cv::Mat values) = 0;
};

class Regulariser {
public:
    enum class RegularisationType { Manual, MatrixNorm };

    Regulariser(RegularisationType regularisation_type = RegularisationType::Manual, float param = 0.0f, bool regularise_last_row = true)
        : regularisation_type(regularisation_type), lambda(param), regularise_last_row(regularise_last_row) {}

    // The C-ABI view of this regulariser; the lambda rule itself (regressors.hpp:126-148) runs on the device.
    sd_regulariser c() const
    {
        sd_regulariser r;
        r.type = regularisation_type == RegularisationType::MatrixNorm ? 1 : 0;
        r.param = lambda;
        r.regularise_last_row = regularise_last_row ? 1 : 0;
        return r;
    }
    static Regulariser from_c(const sd_regulariser& r)
    {
        return Regulariser(r.type == 1 ? RegularisationType::MatrixNorm : RegularisationType::Manual, r.param, r.regularise_last_row != 0);
    }

private:
    RegularisationType regularisation_type;
    float lambda;
    bool regularise_last_row;
};

// The solver behind every Solver name of the reference: Gram on tensor cores + LU / Cholesky on the device.
class B200Solver {
public:
    cv::Mat solve(cv::Mat data, cv::Mat labels, Regulariser regulariser)
    {
        if (data.empty() || labels.empty() || data.rows != labels.rows) throw std::runtime_error("solve: data/labels shape mismatch");
        sd_ctx* ctx = sd_b200::context();
        const int N = data.rows, D = data.cols, M = labels.cols;
        // one extended operand [A | B] so that A^T B rides along in the same SYRK
        const int64_t ld = (static_cast<int64_t>(D) + M + 3) / 4 * 4;
        sd_b200::DeviceBuffer ext(static_cast<size_t>(N) * ld * sizeof(float)), dX(static_cast<size_t>(D) * M * sizeof(float));
        // [A | B] side by side on the device: two strided copies
        sd_b200::check(ctx, sd_memcpy2d_h2d(ctx, ext.as<float>(), ld * sizeof(float), data.ptr<float>(0), data.step(), sizeof(float) * D, N), "solve");
        sd_b200::check(ctx, sd_memcpy2d_h2d(ctx, ext.as<float>() + D, ld * sizeof(float), labels.ptr<float>(0), labels.step(), sizeof(float) * M, N), "solve");
        const sd_regulariser reg = regulariser.c();
        // the private copy is centred in place (no-op for D <= 256): see sd_centre_features in sd_b200.h
        sd_b200::DeviceBuffer mu(static_cast<size_t>(D) * sizeof(float));
        sd_b200::check(ctx, sd_centre_features(ctx, nullptr, ext.as<float>(), ld, N, D, N, &reg, mu.as<float>()), "sd_centre_features");
        sd_b200::check(ctx, sd_learn_centred(ctx, nullptr, ext.as<float>(), ld, ext.as<float>() + D, ld, N, D, M, &reg, N, 0, mu.as<float>(),
                                             dX.as<float>(), nullptr, &last_lambda), "sd_learn_centred");
        return sd_b200::download(dX.as<float>(), D, M, M);
    }
    // called by the optimiser's device route after a level was learned (VerbosePartialPivLUSolver prints here)
    void report() const {}
    float last_lambda = 0.0f;
};

using PartialPivLUSolver = B200Solver;          // regressors.hpp:180-235

// regressors.hpp:245-306: the solver that "can check for invertibility".  Same system and solve as above, plus the numerical
// rank of the regularised AtA from a diagonally pivoted Cholesky on the device (sd_learn_rank_revealing); a deficient rank is
// reported with the reference's message (regressors.hpp:290-293) and learning continues, as there.  The optimiser's device
// route learns through sd_learn_centred instead; it asks the library for the rank (sd_set_rank_diagnostic) and hands it over
// with report_rank().
class ColPivHouseholderQRSolver {
public:
    cv::Mat solve(cv::Mat data, cv::Mat labels, Regulariser regulariser)
    {
        if (data.empty() || labels.empty() || data.rows != labels.rows) throw std::runtime_error("solve: data/labels shape mismatch");
        sd_ctx* ctx = sd_b200::context();
        const int N = data.rows, D = data.cols, M = labels.cols;
        const int64_t ld = (static_cast<int64_t>(D) + M + 3) / 4 * 4;
        sd_b200::DeviceBuffer ext(static_cast<size_t>(N) * ld * sizeof(float)), dX(static_cast<size_t>(D) * M * sizeof(float));
        sd_b200::check(ctx, sd_memcpy2d_h2d(ctx, ext.as<float>(), ld * sizeof(float), data.ptr<float>(0), data.step(), sizeof(float) * D, N), "solve");
        sd_b200::check(ctx, sd_memcpy2d_h2d(ctx, ext.as<float>() + D, ld * sizeof(float), labels.ptr<float>(0), labels.step(), sizeof(float) * M, N), "solve");
        const sd_regulariser reg = regulariser.c();
        int rank = -1;
        const int rc = sd_learn_rank_revealing(ctx, ext.as<float>(), ld, ext.as<float>() + D, ld, N, D, M, &reg, dX.as<float>(), &last_lambda, &rank);
        report_rank(rank, D);
        if (rc == SD_ERR_NUMERIC && last_rank >= 0 && last_rank < D) {
            // the reference would hand back whatever Eigen's inverse of a singular matrix contains; here the factorisation stops
            cv::Mat nan_x(D, M, CV_32FC1);
            for (int r = 0; r < D; ++r) for (int c = 0; c < M; ++c) nan_x.at<float>(r, c) = std::numeric_limits<float>::quiet_NaN();
            return nan_x;
        }
        sd_b200::check(ctx, rc, "sd_learn_rank_revealing");
        return sd_b200::download(dX.as<float>(), D, M, M);
    }
    void report() const {}
    // the rank of a system of D unknowns that was learned; a deficient one prints the reference's message
    void report_rank(int rank, int D)
    {
        last_rank = rank;
        if (rank >= 0 && rank < D)
            std::cout << "The regularised AtA is not invertible. We continued learning, but Eigen may return garbage (their docu is not very specific). (The rank is "
                      << std::to_string(rank) << ", full rank would be " << std::to_string(D) << "). Increase lambda." << std::endl;
    }
    float last_lambda = 0.0f;
    int last_rank = -1;       // numerical rank of the last system learned (-1: not computed, the distributed factorisation)
};

template <class Solver = PartialPivLUSolver>
class LinearRegressor : public Regressor {
public:
    LinearRegressor(Regulariser regulariser = Regulariser()) : x(), regulariser(regulariser) {}
    // copies share the host model (cv::Mat is reference counted, as in the reference) but never the device copy
    LinearRegressor(const LinearRegressor& o) : x(o.x), regulariser(o.regulariser), solver(o.solver), dirty(true) {}
    LinearRegressor& operator=(const LinearRegressor& o)
    {
        if (this != &o) { x = o.x; regulariser = o.regulariser; solver = o.solver; dirty = true; }
        return *this;
    }

    bool learn(cv::Mat data, cv::Mat labels) override
    {
        this->x = solver.solve(data, labels, regulariser);
        dirty = true;
        return true;   // regressors.hpp:349
    }

    double test(cv::Mat data, cv::Mat labels) override
    {
        sd_ctx* ctx = sd_b200::context();
        sd_b200::DeviceBuffer dV, dL;
        sd_b200::upload(data, dV, data.cols);
        sd_b200::upload(labels, dL, labels.cols);
        double residual = 0;
        sd_b200::check(ctx, sd_test_residual(ctx, dV.as<float>(), data.cols, dL.as<float>(), labels.cols, data.rows, data.cols, device_x(), x.cols, &residual), "sd_test_residual");
        return residual;
    }

    cv::Mat predict(cv::Mat values) override
    {
        sd_ctx* ctx = sd_b200::context();
        sd_b200::DeviceBuffer dV, dO(static_cast<size_t>(values.rows) * x.cols * sizeof(float));
        sd_b200::upload(values, dV, values.cols);
        sd_b200::check(ctx, sd_predict(ctx, dV.as<float>(), values.cols, values.rows, values.cols, device_x(), x.cols, dO.as<float>(), x.cols), "sd_predict");
        return sd_b200::download(dO.as<float>(), values.rows, x.cols, x.cols);
    }

    cv::Mat x;   // the learned D x M model, public as in the reference (regressors.hpp:383)

    // device-resident copy of x for the cascade kernels (uploaded lazily after x changes)
    const float* device_x()
    {
        if (dirty || dx.bytes() == 0) { sd_b200::upload(x, dx, x.cols); dirty = false; }
        return dx.template as<float>();
    }
    void set_x(cv::Mat new_x) { x = new_x; dirty = true; }
    void report_solver() { solver.report(); }
    // only for solvers that report a rank (ColPivHouseholderQRSolver): the optimiser's device route calls it after each level
    template <class S = Solver>
    auto report_rank(int rank, int D) -> decltype(std::declval<S&>().report_rank(rank, D)) { return solver.report_rank(rank, D); }
    const Solver& get_solver() const { return solver; }
    const Regulariser& get_regulariser() const { return regulariser; }

private:
    Regulariser regulariser;
    Solver solver;
    sd_b200::DeviceBuffer dx;
    bool dirty = true;
};

}  // namespace superviseddescent
