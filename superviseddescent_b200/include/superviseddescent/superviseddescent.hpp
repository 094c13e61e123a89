// H100 drop-in for the reference's include/superviseddescent/superviseddescent.hpp.
//
// SupervisedDescentOptimiser<RegressorType, NormalisationStrategy> keeps train / test / predict with the
// reference's signatures (superviseddescent.hpp:85-361) and its callback types (:52-54).  Two routes:
//
//   device route   RegressorType is this package's LinearRegressor<>, the projection is a device
//                  projection (rcr::HogTransform, or a batch projection with feature_length / project_device,
//                  see is_device_batch_projection) or a host batch projection (feature_length / project_host,
//                  see is_host_batch_projection; RowwiseProjection wraps a per-row functor) and the
//                  normalisation maps to sd_normalisation: targets, Gram, solve and update all stay in HBM,
//                  one sd_train_level / sd_apply_level call (sd_*_level_projected, sd_*_level_host_projected for
//                  a batch projection) per level through a buffer of feature rows that holds the whole level
//                  when it fits, and chunks of it otherwise (set_rows_per_chunk).
//   functor route  any other projection functor h(row, level, idx) -> Mat | float is USER host code; it is
//                  evaluated on a pool of host threads exactly as the reference does (:173-189) and the
//                  stacked feature matrix goes through RegressorType::learn / predict (which are GPU calls
//                  for LinearRegressor<>).  That is the reference's API for user functors, not a fallback.
#pragma once

#include <exception>
#include <functional>
#include <thread>
#include <type_traits>
#include <utility>
#include <vector>

#include "superviseddescent/regressors.hpp"

namespace superviseddescent {

inline void no_eval(const cv::Mat& /*current_predictions*/) {}   // superviseddescent.hpp:52-54

class NoNormalisation {   // superviseddescent.hpp:60-74
public:
    inline cv::Mat operator()(cv::Mat params) { return cv::Mat::ones(1, params.cols, params.type()); }
    sd_normalisation c_normalisation() const { sd_normalisation n{}; n.kind = 0; return n; }
};

namespace detail {

template <class...> struct voider { using type = void; };
template <class... T> using void_t = typename voider<T...>::type;

// projection whose frames a level call reads, projected on the device for all rows at once (rcr::HogTransform)
template <class P, class = void> struct is_device_projection : std::false_type {};
template <class P> struct is_device_projection<P, void_t<decltype(std::declval<P&>().level_frames(0)), decltype(std::declval<P&>().hog_param(size_t(0)))>> : std::true_type {};

// projection that writes the feature rows of a chunk on the device itself (sd_level_projection):
//   int feature_length(size_t level);
//   int project_device(sd_ctx* ctx, size_t level, const float* d_x, int64_t ldx, int64_t first_row, int rows, float* d_out, int64_t ld);
// project_device follows the callback contract of include/sd_b200.h (work ordered on sd_ctx_stream(ctx), columns [0, D) only,
// deterministic); a non-zero return or an exception fails the level, and the exception is rethrown from train() / test().
template <class P, class = void> struct is_device_batch_projection : std::false_type {};
template <class P> struct is_device_batch_projection<P, void_t<
    decltype(static_cast<int>(std::declval<P&>().feature_length(size_t(0)))),
    decltype(static_cast<int>(std::declval<P&>().project_device(std::declval<sd_ctx*>(), size_t(0), std::declval<const float*>(), int64_t(0),
                                                                int64_t(0), 0, std::declval<float*>(), int64_t(0))))>> : std::true_type {};

// projection that writes the feature rows of a batch on the host (sd_level_host_projection):
//   int feature_length(size_t level);
//   int project_host(size_t level, const float* x, int64_t ldx, int64_t first_row, int rows, float* out, int64_t ld);
// x: the batch's parameter rows (pitch ldx = P); out: a pinned staging half (pitch ld), columns [0, D) of `rows` rows to write.
// project_host follows the host callback contract of include/sd_b200.h (deterministic, no calls into the library's context); a
// non-zero return or an exception fails the level, and the exception is rethrown from train() / test().  RowwiseProjection makes
// one from a per-row functor.
template <class P, class = void> struct is_host_batch_projection : std::false_type {};
template <class P> struct is_host_batch_projection<P, void_t<
    decltype(static_cast<int>(std::declval<P&>().feature_length(size_t(0)))),
    decltype(static_cast<int>(std::declval<P&>().project_host(size_t(0), std::declval<const float*>(), int64_t(0), int64_t(0), 0,
                                                              std::declval<float*>(), int64_t(0))))>> : std::true_type {};

template <class P> struct takes_device_route
    : std::integral_constant<bool, is_device_projection<P>::value || is_device_batch_projection<P>::value ||
                                       is_host_batch_projection<P>::value> {};

// Where the device route's levels get their feature rows: a HogTransform's frames (sd_train_level / sd_apply_level), a device
// batch projection's callback (sd_train_level_projected / sd_apply_level_projected) or a host batch projection's callback
// (sd_train_level_host_projected / sd_apply_level_host_projected), tried in that order.
enum { kHogSource, kDeviceSource, kHostSource };
template <class P> struct source_kind
    : std::integral_constant<int, is_device_projection<P>::value ? kHogSource : (is_device_batch_projection<P>::value ? kDeviceSource : kHostSource)> {};

template <class P, int Kind = source_kind<P>::value> class LevelSource;

// an exception of the projection, kept while the C call unwound normally, for rethrow() after the call
class CallbackError {
public:
    void rethrow()
    {
        if (!error) return;
        std::exception_ptr e = error;
        error = nullptr;
        std::rethrow_exception(e);
    }

protected:
    std::exception_ptr error;
};

template <class P> class LevelSource<P, kHogSource> {
public:
    LevelSource(P& projection, int n) : h(projection), eyes(projection.eyes()), frames(projection.level_frames(n)) {}
    const sd_level_frames* level_frames() const { return &frames; }
    int train(sd_ctx* ctx, sd_comm* c, size_t level, const float* d_x, const float* d_gt, int n, int Pd, int64_t n_global,
              const sd_normalisation& norm, const float* tmpl, int64_t ldt, const sd_regulariser& reg, int route, float* chunk,
              int64_t ld, int rows, float* X, float* x_next)
    {
        const sd_hog_param hp = h.hog_param(level);
        return sd_train_level(ctx, c, &frames, d_x, d_gt, n, Pd / 2, n_global, &eyes, &hp, &norm, tmpl, ldt, &reg, route, chunk, ld, rows,
                              X, x_next, nullptr);
    }
    int apply(sd_ctx* ctx, size_t level, const float* d_x, int n, int Pd, const sd_normalisation& norm, const float* tmpl, int64_t ldt,
              const float* X, float* chunk, int64_t ld, int rows, float* x_next)
    {
        const sd_hog_param hp = h.hog_param(level);
        return sd_apply_level(ctx, &frames, d_x, n, Pd / 2, &eyes, &hp, &norm, tmpl, ldt, X, chunk, ld, rows, x_next);
    }
    void rethrow() {}

private:
    P& h;
    sd_normalisation eyes;
    sd_level_frames frames;
};

template <class P> class LevelSource<P, kDeviceSource> : public CallbackError {
public:
    LevelSource(P& projection, int /*n*/) : h(projection) {}
    const sd_level_frames* level_frames() const { return nullptr; }
    int train(sd_ctx* ctx, sd_comm* c, size_t level, const float* d_x, const float* d_gt, int n, int Pd, int64_t n_global,
              const sd_normalisation& norm, const float* tmpl, int64_t ldt, const sd_regulariser& reg, int route, float* chunk,
              int64_t ld, int rows, float* X, float* x_next)
    {
        const sd_level_projection proj = descriptor(level);
        return sd_train_level_projected(ctx, c, &proj, d_x, d_gt, n, Pd, n_global, &norm, tmpl, ldt, &reg, route, chunk, ld, rows, X,
                                        x_next, nullptr);
    }
    int apply(sd_ctx* ctx, size_t level, const float* d_x, int n, int Pd, const sd_normalisation& norm, const float* tmpl, int64_t ldt,
              const float* X, float* chunk, int64_t ld, int rows, float* x_next)
    {
        const sd_level_projection proj = descriptor(level);
        return sd_apply_level_projected(ctx, &proj, d_x, n, Pd, &norm, tmpl, ldt, X, chunk, ld, rows, x_next);
    }

private:
    sd_level_projection descriptor(size_t level)
    {
        sd_level_projection proj{};
        proj.fn = &LevelSource::call;
        proj.user = this;
        proj.level = static_cast<int32_t>(level);
        proj.feature_length = h.feature_length(level);
        return proj;
    }
    static int call(void* user, sd_ctx* ctx, int level, const float* d_x, int64_t ldx, int64_t first_row, int rows, float* d_out, int64_t ld)
    {
        LevelSource* self = static_cast<LevelSource*>(user);
        try {
            return self->h.project_device(ctx, static_cast<size_t>(level), d_x, ldx, first_row, rows, d_out, ld);
        } catch (...) {                          // nothing may unwind through the library's frames
            self->error = std::current_exception();
            return -1;
        }
    }
    P& h;
};

template <class P> class LevelSource<P, kHostSource> : public CallbackError {
public:
    LevelSource(P& projection, int /*n*/) : h(projection) {}
    const sd_level_frames* level_frames() const { return nullptr; }
    int train(sd_ctx* ctx, sd_comm* c, size_t level, const float* d_x, const float* d_gt, int n, int Pd, int64_t n_global,
              const sd_normalisation& norm, const float* tmpl, int64_t ldt, const sd_regulariser& reg, int route, float* chunk,
              int64_t ld, int rows, float* X, float* x_next)
    {
        const sd_level_host_projection proj = descriptor(level);
        return sd_train_level_host_projected(ctx, c, &proj, d_x, d_gt, n, Pd, n_global, &norm, tmpl, ldt, &reg, route, chunk, ld, rows, X,
                                             x_next, nullptr);
    }
    int apply(sd_ctx* ctx, size_t level, const float* d_x, int n, int Pd, const sd_normalisation& norm, const float* tmpl, int64_t ldt,
              const float* X, float* chunk, int64_t ld, int rows, float* x_next)
    {
        const sd_level_host_projection proj = descriptor(level);
        return sd_apply_level_host_projected(ctx, &proj, d_x, n, Pd, &norm, tmpl, ldt, X, chunk, ld, rows, x_next);
    }

private:
    sd_level_host_projection descriptor(size_t level)
    {
        sd_level_host_projection proj{};
        proj.fn = &LevelSource::call;
        proj.user = this;
        proj.level = static_cast<int32_t>(level);
        proj.feature_length = h.feature_length(level);
        proj.stage_half_bytes = 0;               // the library's default
        return proj;
    }
    static int call(void* user, int level, const float* x, int64_t ldx, int64_t first_row, int rows, float* out, int64_t ld)
    {
        LevelSource* self = static_cast<LevelSource*>(user);
        try {
            return self->h.project_host(static_cast<size_t>(level), x, ldx, first_row, rows, out, ld);
        } catch (...) {                          // nothing may unwind through the library's frames
            self->error = std::current_exception();
            return -1;
        }
    }
    P& h;
};

template <class N, class = void> struct has_c_normalisation : std::false_type {};
template <class N> struct has_c_normalisation<N, void_t<decltype(std::declval<const N&>().c_normalisation())>> : std::true_type {};

// regressors whose solver reports the rank of the system (ColPivHouseholderQRSolver)
template <class R, class = void> struct reports_rank : std::false_type {};
template <class R> struct reports_rank<R, void_t<decltype(std::declval<R&>().report_rank(0, 0))>> : std::true_type {};
template <class R> void report_rank(R& r, int rank, int D, std::true_type) { r.report_rank(rank, D); }
template <class R> void report_rank(R&, int, int, std::false_type) {}

template <class R, class = void> struct is_device_regressor : std::false_type {};
template <class R> struct is_device_regressor<R, void_t<decltype(std::declval<R&>().device_x()), decltype(std::declval<R&>().get_regulariser())>> : std::true_type {};

inline cv::Mat as_row(float v) { cv::Mat m(1, 1, CV_32FC1); m.at<float>(0, 0) = v; return m; }
inline cv::Mat as_row(double v) { return as_row(static_cast<float>(v)); }
inline cv::Mat as_row(const cv::Mat& m) { return m; }

// h(current_x.row(i), level, i) for every row, on hardware_concurrency() host threads (superviseddescent.hpp:173-189)
template <class ProjectionFunction>
cv::Mat project_on_host(const cv::Mat& current_x, size_t level, ProjectionFunction projection)
{
    const int n = current_x.rows;
    std::vector<cv::Mat> rows(n);
    unsigned threads = std::thread::hardware_concurrency();
    if (threads == 0) threads = 4;
    if (threads > static_cast<unsigned>(n)) threads = n > 0 ? n : 1;
    std::vector<std::thread> pool;
    for (unsigned t = 0; t < threads; ++t) {
        pool.emplace_back([&, t, projection]() mutable {      // each worker owns a copy of the functor
            for (int i = t; i < n; i += threads) rows[i] = as_row(projection(current_x.row(i), level, i)).clone();
        });
    }
    for (auto& th : pool) th.join();
    cv::Mat features;
    for (int i = 0; i < n; ++i) features.push_back(rows[i]);
    return features;
}

}  // namespace detail

// A reference-style projection functor h(cv::Mat row, size_t level, int index) -> Mat | float as a host batch projection, so that
// the optimiser runs it through the level pipeline (chunks, several ranks, the host filling rows while the GPU works) instead of
// the functor route.  project_host evaluates a batch's rows on hardware_concurrency() threads, each worker with its own copy of
// the functor, as the functor route does; the rows h sees are views of the library's pinned copy of the parameters.
// feature_length: one D for every level, or one per level.
template <class H>
class RowwiseProjection {
public:
    RowwiseProjection(H h, int feature_length) : h(std::move(h)), lengths(1, feature_length) {}
    RowwiseProjection(H h, std::vector<int> feature_lengths) : h(std::move(h)), lengths(std::move(feature_lengths)) {}

    int feature_length(size_t level) const { return lengths.size() == 1 ? lengths[0] : lengths.at(level); }

    int project_host(size_t level, const float* x, int64_t ldx, int64_t first_row, int rows, float* out, int64_t ld)
    {
        const int D = feature_length(level);
        unsigned threads = std::thread::hardware_concurrency();
        if (threads == 0) threads = 4;
        if (threads > static_cast<unsigned>(rows)) threads = rows > 0 ? rows : 1;
        std::vector<std::exception_ptr> errors(threads);
        auto work = [&](unsigned t, H& projection) {
            try {
                for (int i = static_cast<int>(t); i < rows; i += static_cast<int>(threads)) {
                    const cv::Mat row(1, static_cast<int>(ldx), CV_32FC1, const_cast<float*>(x + static_cast<int64_t>(i) * ldx));
                    const cv::Mat f = detail::as_row(projection(row, level, static_cast<int>(first_row + i)));
                    if (f.type() != CV_32FC1 || f.rows * f.cols != D)
                        throw std::runtime_error("RowwiseProjection: the functor returned " + std::to_string(f.rows * f.cols) + " values for row " +
                                                 std::to_string(first_row + i) + ", feature_length is " + std::to_string(D));
                    float* dst = out + static_cast<int64_t>(i) * ld;
                    for (int k = 0; k < D; ++k) dst[k] = f.at<float>(k);
                }
            } catch (...) {
                errors[t] = std::current_exception();
            }
        };
        if (threads == 1) {
            work(0, h);
        } else {
            std::vector<std::thread> pool;
            for (unsigned t = 0; t < threads; ++t)
                pool.emplace_back([&work, t, projection = h]() mutable { work(t, projection); });   // each worker owns a copy
            for (auto& th : pool) th.join();
        }
        for (auto& e : errors)
            if (e) std::rethrow_exception(e);
        return 0;
    }

private:
    H h;
    std::vector<int> lengths;
};

template <class H> RowwiseProjection<H> rowwise(H h, int feature_length) { return RowwiseProjection<H>(std::move(h), feature_length); }
template <class H> RowwiseProjection<H> rowwise(H h, std::vector<int> feature_lengths)
{
    return RowwiseProjection<H>(std::move(h), std::move(feature_lengths));
}

template <class RegressorType, class NormalisationStrategy = NoNormalisation>
class SupervisedDescentOptimiser {
public:
    SupervisedDescentOptimiser() = default;
    SupervisedDescentOptimiser(std::vector<RegressorType> regressors, NormalisationStrategy normalisation = NormalisationStrategy())
        : regressors(std::move(regressors)), normalisation_strategy(std::move(normalisation)) {}

    template <class ProjectionFunction>
    void train(cv::Mat parameters, cv::Mat initialisations, cv::Mat templates, ProjectionFunction projection)
    {
        want_callback = false;   // no host copy of current_x per level when nobody listens (SURVEY 5, "Metrics")
        train(parameters, initialisations, templates, projection, no_eval);
        want_callback = true;
    }

    // Multi-GPU (one process per GPU, each passing ITS shard of the rows): the optional communicator of the C ABI.  Per level
    // the local [AtA | Atb] is exchanged and solved by sd_learn_dist; every rank ends with the same regressors.  route: 0 =
    // all-reduce + every rank solves, 1 = reduce to the panel owners + distributed Cholesky, 2 = all-reduce + CG shared by the
    // ranks.  The callback receives the rows of ALL ranks (superviseddescent.hpp:217).
    template <class ProjectionFunction, class OnTrainingEpochCallback>
    void train(cv::Mat parameters, cv::Mat initialisations, cv::Mat templates, ProjectionFunction projection,
               OnTrainingEpochCallback on_training_epoch_callback, sd_comm* communicator, int route = 0)
    {
        static_assert(detail::takes_device_route<ProjectionFunction>::value && detail::has_c_normalisation<NormalisationStrategy>::value &&
                          detail::is_device_regressor<RegressorType>::value,
                      "multi-GPU training needs the device route (HogTransform, device or host batch projection, device regressors)");
        comm = communicator;
        comm_route = route;
        train_impl(parameters, initialisations, templates, projection, on_training_epoch_callback, std::true_type());
        comm = nullptr;
    }

    // superviseddescent.hpp:165-219
    template <class ProjectionFunction, class OnTrainingEpochCallback>
    void train(cv::Mat parameters, cv::Mat initialisations, cv::Mat templates, ProjectionFunction projection,
               OnTrainingEpochCallback on_training_epoch_callback)
    {
        train_impl(parameters, initialisations, templates, projection, on_training_epoch_callback,
                   std::integral_constant<bool, detail::takes_device_route<ProjectionFunction>::value &&
                                                    detail::has_c_normalisation<NormalisationStrategy>::value &&
                                                    detail::is_device_regressor<RegressorType>::value>());
    }

    template <class ProjectionFunction>
    cv::Mat test(cv::Mat initialisations, cv::Mat templates, ProjectionFunction projection)
    {
        want_callback = false;
        cv::Mat out = test(initialisations, templates, projection, no_eval);
        want_callback = true;
        return out;
    }

    // superviseddescent.hpp:262-306
    template <class ProjectionFunction, class OnRegressorIterationCallback>
    cv::Mat test(cv::Mat initialisations, cv::Mat templates, ProjectionFunction projection,
                 OnRegressorIterationCallback on_regressor_iteration_callback)
    {
        return test_impl(initialisations, templates, projection, on_regressor_iteration_callback,
                         std::integral_constant<bool, detail::takes_device_route<ProjectionFunction>::value &&
                                                          detail::has_c_normalisation<NormalisationStrategy>::value &&
                                                          detail::is_device_regressor<RegressorType>::value>());
    }

    // superviseddescent.hpp:323-344 (single row or batch; same arithmetic as test without a callback)
    template <class ProjectionFunction>
    cv::Mat predict(cv::Mat initialisations, cv::Mat templates, ProjectionFunction projection)
    {
        return test(initialisations, templates, projection);
    }

    std::vector<RegressorType>& get_regressors() { return regressors; }
    NormalisationStrategy& get_normalisation() { return normalisation_strategy; }

    // Device route: feature rows per chunk of a level in train() / test() / predict().  0 (the default): as many as fit on the
    // device beside the solve (sd_level_chunk_rows) -- the whole level whenever it fits.  Templates always take one chunk.  The
    // automatic chunk leaves a batch projection's project_device only the library's 512 MB reserve for its own temporaries: one
    // that needs more per row sets the chunk here.
    void set_rows_per_chunk(int rows) { rows_per_chunk = rows < 0 ? 0 : rows; }

private:
    std::vector<RegressorType> regressors;
    NormalisationStrategy normalisation_strategy;
    bool want_callback = true;
    int rows_per_chunk = 0;

    // ------------------------------------------------------------------ functor route (host projection)
    template <class P, class CB>
    void train_impl(cv::Mat parameters, cv::Mat initialisations, cv::Mat templates, P projection, CB cb, std::false_type)
    {
        using cv::Mat;
        Mat current_x = initialisations;
        for (size_t level = 0; level < regressors.size(); ++level) {
            Mat features = detail::project_on_host(current_x, level, projection);
            Mat observed = templates.empty() ? features : Mat(features - templates);              // :191-197
            Mat b(current_x.rows, current_x.cols, CV_32FC1);                                     // :199-205
            for (int i = 0; i < current_x.rows; ++i) {
                Mat n = normalisation_strategy(current_x.row(i));
                for (int j = 0; j < current_x.cols; ++j)
                    b.at<float>(i, j) = (current_x.at<float>(i, j) - parameters.at<float>(i, j)) * n.at<float>(0, j);
            }
            regressors[level].learn(observed, b);                                                // :207
            current_x = update_on_host(level, observed, current_x);                              // :209-215
            cb(current_x);                                                                       // :217
        }
    }

    template <class P, class CB>
    cv::Mat test_impl(cv::Mat initialisations, cv::Mat templates, P projection, CB cb, std::false_type)
    {
        using cv::Mat;
        Mat current_x = initialisations;
        for (size_t level = 0; level < regressors.size(); ++level) {
            Mat features = detail::project_on_host(current_x, level, projection);
            Mat observed = templates.empty() ? features : Mat(features - templates);
            current_x = update_on_host(level, observed, current_x);
            cb(current_x);                                                                       // :303
        }
        return current_x;
    }

    cv::Mat update_on_host(size_t level, const cv::Mat& observed, const cv::Mat& current_x)
    {
        cv::Mat update = regressors[level].predict(observed);      // one batched GPU GEMM instead of N GEMVs
        cv::Mat x_k(current_x.rows, current_x.cols, CV_32FC1);
        for (int i = 0; i < current_x.rows; ++i) {
            cv::Mat n = normalisation_strategy(current_x.row(i));
            for (int j = 0; j < current_x.cols; ++j)
                x_k.at<float>(i, j) = current_x.at<float>(i, j) - update.at<float>(i, j) * (1.0f / n.at<float>(0, j));
        }
        return x_k;
    }

    sd_comm* comm = nullptr;     // set for the duration of a multi-GPU train()
    int comm_route = 0;

    // feature rows per chunk of a device-route level: set_rows_per_chunk's (at most n), or as many as fit
    int chunk_rows(sd_ctx* ctx, sd_comm* c, const sd_level_frames* frames, int n, int D, int Pd, int route) const
    {
        if (rows_per_chunk > 0) return rows_per_chunk < n ? rows_per_chunk : (n > 0 ? n : 1);
        int rows = 0;
        sd_b200::check(ctx, sd_level_chunk_rows(ctx, c, frames, n, D, Pd, route, 0, &rows), "sd_level_chunk_rows");
        return rows;
    }

    // ------------------------------------------------------------------ device route
    template <class P, class CB>
    void train_impl(cv::Mat parameters, cv::Mat initialisations, cv::Mat templates, P projection, CB cb, std::true_type)
    {
        sd_ctx* ctx = sd_b200::context();
        const int n = initialisations.rows, Pd = initialisations.cols;
        sd_b200::DeviceBuffer d_gt, d_cur, d_next(static_cast<size_t>(n) * Pd * sizeof(float)), d_tmpl;
        sd_b200::upload(parameters, d_gt, Pd);
        sd_b200::upload(initialisations, d_cur, Pd);
        const sd_normalisation norm = normalisation_strategy.c_normalisation();
        detail::LevelSource<P> src(projection, n);
        if (!templates.empty()) sd_b200::upload(templates, d_tmpl, templates.cols);
        sd_b200::DeviceBuffer X;
        int64_t n_global = n;
        const int nranks = comm ? sd_comm_size(comm) : 1;
        if (nranks > 1) sd_b200::check(ctx, sd_comm_sum_int64(ctx, comm, &n_global), "sd_comm_sum_int64");
        sd_comm* c = nranks > 1 ? comm : nullptr;
        const int route = nranks > 1 ? comm_route : 0;
        for (size_t level = 0; level < regressors.size(); ++level) {
            const int D = projection.feature_length(level);
            const int64_t ld = (static_cast<int64_t>(D) + Pd + 3) / 4 * 4;
            const sd_regulariser reg = regressors[level].get_regulariser().c();
            const bool want_rank = detail::reports_rank<RegressorType>::value;
            if (want_rank) sd_b200::check(ctx, sd_set_rank_diagnostic(ctx, 1), "sd_set_rank_diagnostic");   // counted by the chunk query
            // 1)-4) :173-215 -- features, targets, Gram, exchange, solve and update through a buffer of `rows` feature rows
            const int rows = templates.empty() ? chunk_rows(ctx, c, src.level_frames(), n, D, Pd, route) : (n > 0 ? n : 1);
            sd_b200::DeviceBuffer chunk(static_cast<size_t>(rows) * ld * sizeof(float));
            X.allocate(static_cast<size_t>(D) * Pd * sizeof(float));
            const float* tmpl = templates.empty() ? nullptr : d_tmpl.as<float>();
            const int rc = src.train(ctx, c, level, d_cur.as<float>(), d_gt.as<float>(), n, Pd, n_global, norm, tmpl, templates.cols, reg, route,
                                     chunk.as<float>(), ld, rows, X.as<float>(), d_next.as<float>());
            if (want_rank) {
                sd_set_rank_diagnostic(ctx, 0);
                detail::report_rank(regressors[level], sd_last_rank(ctx), D, detail::reports_rank<RegressorType>());
            }
            src.rethrow();
            // a factorisation that broke down throws (with the rank in the message): NaN weights would poison the next level
            sd_b200::check(ctx, rc, "sd_train_level");
            regressors[level].set_x(sd_b200::download(X.as<float>(), D, Pd, Pd));
            regressors[level].report_solver();
            std::swap(d_cur, d_next);
            if (want_callback) {                                                                             // 5) :217
                if (nranks > 1) {
                    // every rank contributes its rows; shards are padded to the largest one for the gather
                    int64_t most = n;
                    std::vector<int64_t> counts(nranks, 0);
                    for (int r = 0; r < nranks; ++r) {
                        int64_t v = (r == sd_comm_rank(comm)) ? n : 0;
                        sd_b200::check(ctx, sd_comm_sum_int64(ctx, comm, &v), "sd_comm_sum_int64");
                        counts[r] = v;
                        most = v > most ? v : most;
                    }
                    const size_t row_bytes = static_cast<size_t>(Pd) * sizeof(float);
                    sd_b200::DeviceBuffer send(static_cast<size_t>(most) * row_bytes), recv(static_cast<size_t>(most) * row_bytes * nranks);
                    sd_b200::check(ctx, sd_memset(ctx, send.as<float>(), 0, static_cast<size_t>(most) * row_bytes), "gather");
                    sd_b200::check(ctx, sd_memcpy2d_d2d(ctx, send.as<float>(), row_bytes, d_cur.as<float>(), row_bytes, row_bytes, n), "gather");
                    sd_b200::check(ctx, sd_comm_allgather(ctx, comm, send.as<float>(), static_cast<size_t>(most) * row_bytes, recv.as<float>()), "sd_comm_allgather");
                    cv::Mat all;
                    for (int r = 0; r < nranks; ++r)
                        if (counts[r] > 0) all.push_back(sd_b200::download(recv.as<float>() + static_cast<size_t>(r) * most * Pd, static_cast<int>(counts[r]), Pd, Pd));
                    cb(all);
                } else {
                    cb(sd_b200::download(d_cur.as<float>(), n, Pd, Pd));
                }
            }
        }
    }

    template <class P, class CB>
    cv::Mat test_impl(cv::Mat initialisations, cv::Mat templates, P projection, CB cb, std::true_type)
    {
        sd_ctx* ctx = sd_b200::context();
        const int n = initialisations.rows, Pd = initialisations.cols;
        sd_b200::DeviceBuffer d_cur, d_next(static_cast<size_t>(n) * Pd * sizeof(float)), d_tmpl;
        sd_b200::upload(initialisations, d_cur, Pd);
        const sd_normalisation norm = normalisation_strategy.c_normalisation();
        detail::LevelSource<P> src(projection, n);
        if (!templates.empty()) sd_b200::upload(templates, d_tmpl, templates.cols);
        for (size_t level = 0; level < regressors.size(); ++level) {
            const int D = projection.feature_length(level);
            const int64_t ld = (static_cast<int64_t>(D) + 3) / 4 * 4;
            const int rows = chunk_rows(ctx, nullptr, src.level_frames(), n, D, Pd, 0);
            sd_b200::DeviceBuffer chunk(static_cast<size_t>(rows) * ld * sizeof(float));
            const float* tmpl = templates.empty() ? nullptr : d_tmpl.as<float>();
            const int rc = src.apply(ctx, level, d_cur.as<float>(), n, Pd, norm, tmpl, templates.cols, regressors[level].device_x(),
                                     chunk.as<float>(), ld, rows, d_next.as<float>());
            src.rethrow();
            sd_b200::check(ctx, rc, "sd_apply_level");
            std::swap(d_cur, d_next);
            if (want_callback) cb(sd_b200::download(d_cur.as<float>(), n, Pd, Pd));                          // :303
        }
        return sd_b200::download(d_cur.as<float>(), n, Pd, Pd);
    }
};

}  // namespace superviseddescent
