// H100 drop-in for the hot-path part of include/rcr/helpers.hpp: to_row (:45-55),
// to_landmark_collection (:66-75) and get_ied (:136-160).  Drawing / check_face are visualisation and
// dataset hygiene (out of scope, SURVEY.md 2 #8).
#pragma once

#include <cmath>
#include <stdexcept>
#include <string>
#include <vector>

#include "rcr/landmark.hpp"

namespace rcr {

inline cv::Mat to_row(LandmarkCollection<cv::Vec2f> landmarks)
{
    const int n = static_cast<int>(landmarks.size());
    cv::Mat row(1, n * 2, CV_32FC1);
    for (int i = 0; i < n; ++i) {
        row.at<float>(i) = landmarks[i].coordinates[0];
        row.at<float>(i + n) = landmarks[i].coordinates[1];
    }
    return row;
}

inline LandmarkCollection<cv::Vec2f> to_landmark_collection(cv::Mat model_instance, std::vector<std::string> model_landmarks_list)
{
    LandmarkCollection<cv::Vec2f> collection;
    const int n = model_instance.cols / 2;
    if (n != static_cast<int>(model_landmarks_list.size())) throw std::runtime_error("to_landmark_collection: landmark count mismatch");
    for (int i = 0; i < n; ++i)
        collection.emplace_back(Landmark<cv::Vec2f>{model_landmarks_list[i], cv::Vec2f(model_instance.at<float>(i), model_instance.at<float>(i + n))});
    return collection;
}

// row indices of the named landmarks; throws with the reference's messages (helpers.hpp:144,153)
inline std::vector<int> eye_indices(const std::vector<std::string>& ids, const std::vector<std::string>& eye_ids, const char* which)
{
    std::vector<int> out;
    for (const auto& e : eye_ids) {
        int found = -1;
        for (size_t i = 0; i < ids.size(); ++i) if (ids[i] == e) { found = static_cast<int>(i); break; }
        if (found < 0) throw std::runtime_error(std::string("one of given ") + which + "EyeIdentifiers ids not present in lms");
        out.push_back(found);
    }
    return out;
}

// Inter-eye distance of a handful of landmarks (host side; the kernels evaluate the same expression on the device).
inline double get_ied(LandmarkCollection<cv::Vec2f> lms, std::vector<std::string> right_eye_identifiers, std::vector<std::string> left_eye_identifiers)
{
    std::vector<std::string> names;
    for (const auto& l : lms) names.push_back(l.name);
    const auto r = eye_indices(names, right_eye_identifiers, "right");
    const auto l = eye_indices(names, left_eye_identifiers, "left");
    float rx = 0.f, ry = 0.f, lx = 0.f, ly = 0.f;
    for (int i : r) { rx += lms[i].coordinates[0]; ry += lms[i].coordinates[1]; }
    for (int i : l) { lx += lms[i].coordinates[0]; ly += lms[i].coordinates[1]; }
    const float ir = 1.f / static_cast<float>(r.size()), il = 1.f / static_cast<float>(l.size());
    rx *= ir; ry *= ir; lx *= il; ly *= il;
    const double dx = static_cast<double>(rx - lx), dy = static_cast<double>(ry - ly);
    return std::sqrt(dx * dx + dy * dy);
}

}  // namespace rcr
