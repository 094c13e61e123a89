// H100 drop-in for include/superviseddescent/verbose_solver.hpp: the solver type baked into
// rcr::detection_model::model_type (model.hpp:125).  Prints the same four phase lines as the reference
// (verbose_solver.hpp:66-103), measured with CUDA events on the device.
#pragma once

#include <iostream>

#include "superviseddescent/regressors.hpp"

namespace superviseddescent {

class VerbosePartialPivLUSolver {
public:
    cv::Mat solve(cv::Mat data, cv::Mat labels, Regulariser regulariser)
    {
        cv::Mat x = inner.solve(data, labels, regulariser);
        report();
        return x;
    }

    // the four phase lines of verbose_solver.hpp:66-103, from CUDA events of the last learn on this context
    void report() const
    {
        float ms[4] = {0, 0, 0, 0};
        sd_solver_timings(sd_b200::context(), ms);
        std::cout << "At * A (ms): " << ms[0] << std::endl;
        std::cout << "AtA + Reg (ms): " << ms[1] << std::endl;
        std::cout << "Decomposition (ms): " << ms[2] << std::endl;
        std::cout << "solve() (ms): " << ms[3] << std::endl;
    }

private:
    B200Solver inner;
};

}  // namespace superviseddescent
