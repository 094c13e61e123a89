// Minimal row-major matrix type standing in for cv::Mat in the header shells.
//
// The reference's public interface speaks cv::Mat (OpenCV is an external, un-vendored dependency and
// its C++ headers are not installed in this image).  The shells therefore bring the small subset of
// cv::Mat / cv::Rect / cv::Vec2f that the reference's call sites on the hot path actually use
// (SURVEY.md 7.2): rows, cols, type(), ptr<T>(), at<T>(), row(i), colRange, clone(), push_back(),
// empty(), Mat::ones / zeros, channels(), isContinuous().  Storage is reference counted like cv::Mat,
// so passing by value is shallow, exactly as the reference's signatures assume
// (regressors.hpp:199 takes cv::Mat by value).  With -DSD_B200_USE_OPENCV the real OpenCV types are
// used instead and this file defines nothing.
#pragma once

#ifdef SD_B200_USE_OPENCV
#include "opencv2/core/core.hpp"
#else

#include <cassert>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <memory>
#include <stdexcept>
#include <vector>

#define CV_8UC1 0
#define CV_8UC3 16
#define CV_32FC1 5
#define CV_32FC3 21

namespace cv {

struct Rect {
    int x = 0, y = 0, width = 0, height = 0;
    Rect() = default;
    Rect(int x_, int y_, int w_, int h_) : x(x_), y(y_), width(w_), height(h_) {}
};

struct Vec2f {
    float val[2] = {0.f, 0.f};
    Vec2f() = default;
    Vec2f(float a, float b) { val[0] = a; val[1] = b; }
    float& operator[](int i) { return val[i]; }
    const float& operator[](int i) const { return val[i]; }
};

class Mat {
public:
    int rows = 0, cols = 0;

    Mat() = default;
    Mat(int r, int c, int type) { create(r, c, type); }
    // view on external memory (no ownership), like cv::Mat(rows, cols, type, void* data)
    Mat(int r, int c, int type, void* data) : rows(r), cols(c), type_(type), step_(static_cast<size_t>(c) * elem_size(type)), data_(static_cast<unsigned char*>(data)) {}
    // column vector from std::vector<float> (copy), like cv::Mat(const std::vector<T>&, true)
    Mat(const std::vector<float>& v, bool /*copy*/) { create(static_cast<int>(v.size()), 1, CV_32FC1); if (!v.empty()) std::memcpy(data_, v.data(), v.size() * sizeof(float)); }

    void create(int r, int c, int type)
    {
        rows = r; cols = c; type_ = type;
        step_ = static_cast<size_t>(c) * elem_size(type);
        const size_t bytes = step_ * static_cast<size_t>(r);
        store_ = std::shared_ptr<unsigned char>(new unsigned char[bytes ? bytes : 1], std::default_delete<unsigned char[]>());
        data_ = store_.get();
    }

    static Mat zeros(int r, int c, int type) { Mat m(r, c, type); std::memset(m.data_, 0, m.step_ * r); return m; }
    static Mat ones(int r, int c, int type)
    {
        Mat m(r, c, type);
        assert(type == CV_32FC1);
        for (int i = 0; i < r; ++i) for (int j = 0; j < c; ++j) m.at<float>(i, j) = 1.0f;
        return m;
    }

    int type() const { return type_; }
    int channels() const { return type_ == CV_8UC3 || type_ == CV_32FC3 ? 3 : 1; }
    bool empty() const { return data_ == nullptr || rows == 0 || cols == 0; }
    bool isContinuous() const { return step_ == static_cast<size_t>(cols) * elem_size(type_); }
    size_t step() const { return step_; }
    size_t elemSize() const { return elem_size(type_); }
    unsigned char* data() const { return data_; }

    template <class T> T* ptr(int r = 0) { return reinterpret_cast<T*>(data_ + step_ * r); }
    template <class T> const T* ptr(int r = 0) const { return reinterpret_cast<const T*>(data_ + step_ * r); }
    template <class T> T& at(int r, int c) { return ptr<T>(r)[c]; }
    template <class T> const T& at(int r, int c) const { return ptr<T>(r)[c]; }
    // single-index access: i-th element of a row or column vector (cv::Mat::at<T>(int))
    template <class T> T& at(int i) { return rows == 1 ? ptr<T>(0)[i] : (cols == 1 ? ptr<T>(i)[0] : ptr<T>(i / cols)[i % cols]); }
    template <class T> const T& at(int i) const { return const_cast<Mat*>(this)->at<T>(i); }

    Mat row(int r) const { Mat m = *this; m.rows = 1; m.data_ = data_ + step_ * r; return m; }
    Mat rowRange(int r0, int r1) const { Mat m = *this; m.rows = r1 - r0; m.data_ = data_ + step_ * r0; return m; }
    Mat colRange(int c0, int c1) const { Mat m = *this; m.cols = c1 - c0; m.data_ = data_ + c0 * elem_size(type_); return m; }

    Mat clone() const
    {
        Mat m(rows, cols, type_);
        const size_t line = static_cast<size_t>(cols) * elem_size(type_);
        for (int r = 0; r < rows; ++r) std::memcpy(m.data_ + m.step_ * r, data_ + step_ * r, line);
        return m;
    }

    // append the rows of `other` (cv::Mat::push_back); amortised doubling instead of realloc-per-row
    void push_back(const Mat& other)
    {
        if (other.empty()) return;
        if (empty()) { *this = other.clone(); capacity_rows_ = rows; return; }
        if (other.cols != cols || other.type_ != type_) throw std::runtime_error("Mat::push_back: shape/type mismatch");
        const int need = rows + other.rows;
        if (!isContinuous() || !store_ || need > capacity_rows_ || data_ != store_.get()) {
            int cap = capacity_rows_ > 0 ? capacity_rows_ : rows;
            while (cap < need) cap *= 2;
            Mat grown(cap, cols, type_);
            const size_t line = static_cast<size_t>(cols) * elem_size(type_);
            for (int r = 0; r < rows; ++r) std::memcpy(grown.data_ + grown.step_ * r, data_ + step_ * r, line);
            grown.rows = rows;
            grown.capacity_rows_ = cap;
            *this = grown;
        }
        const size_t line = static_cast<size_t>(cols) * elem_size(type_);
        for (int r = 0; r < other.rows; ++r) std::memcpy(data_ + step_ * (rows + r), other.data_ + other.step_ * r, line);
        rows = need;
    }
    void push_back(float v) { Mat m(1, 1, CV_32FC1); m.at<float>(0, 0) = v; push_back(m); }

    template <class T> T* begin() { return ptr<T>(0); }
    template <class T> T* end() { return ptr<T>(0) + static_cast<size_t>(rows) * cols; }

private:
    static size_t elem_size(int type) { return type == CV_32FC1 ? 4 : type == CV_8UC3 ? 3 : type == CV_32FC3 ? 12 : 1; }
    int type_ = CV_32FC1;
    size_t step_ = 0;
    unsigned char* data_ = nullptr;
    std::shared_ptr<unsigned char> store_;
    int capacity_rows_ = 0;
};

// element-wise helpers the reference's call sites use on row vectors
inline Mat operator-(const Mat& a, const Mat& b)
{
    Mat o(a.rows, a.cols, CV_32FC1);
    for (int r = 0; r < a.rows; ++r) for (int c = 0; c < a.cols; ++c) o.at<float>(r, c) = a.at<float>(r, c) - b.at<float>(r, c);
    return o;
}
inline Mat operator*(float s, const Mat& a)
{
    Mat o(a.rows, a.cols, CV_32FC1);
    for (int r = 0; r < a.rows; ++r) for (int c = 0; c < a.cols; ++c) o.at<float>(r, c) = s * a.at<float>(r, c);
    return o;
}
// cv::norm(a, b, NORM_L2) / cv::norm(a, NORM_L2) on CV_32F: float difference, double accumulation
enum { NORM_L2 = 4 };
inline double norm(const Mat& a, int /*type*/ = NORM_L2)
{
    double s = 0;
    for (int r = 0; r < a.rows; ++r) for (int c = 0; c < a.cols; ++c) { const double v = a.at<float>(r, c); s += v * v; }
    return std::sqrt(s);
}
inline double norm(const Mat& a, const Mat& b, int /*type*/ = NORM_L2)
{
    double s = 0;
    for (int r = 0; r < a.rows; ++r) for (int c = 0; c < a.cols; ++c) { const double v = static_cast<double>(a.at<float>(r, c) - b.at<float>(r, c)); s += v * v; }
    return std::sqrt(s);
}
inline void hconcat(const Mat& a, const Mat& b, Mat& dst)
{
    Mat o(a.rows, a.cols + b.cols, CV_32FC1);
    for (int r = 0; r < a.rows; ++r) {
        std::memcpy(o.ptr<float>(r), a.ptr<float>(r), sizeof(float) * a.cols);
        std::memcpy(o.ptr<float>(r) + a.cols, b.ptr<float>(r), sizeof(float) * b.cols);
    }
    dst = o;
}

}  // namespace cv

#endif  // SD_B200_USE_OPENCV
