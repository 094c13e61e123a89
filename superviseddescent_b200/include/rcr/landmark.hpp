// H100 drop-in for include/rcr/landmark.hpp (:34-64): Landmark<T>, LandmarkCollection<T>, filter().
#pragma once

#include <algorithm>
#include <string>
#include <vector>

#include "sd_b200/mat.hpp"

namespace rcr {

template <class LandmarkType>
struct Landmark {
    std::string name;
    LandmarkType coordinates;
};

template <class LandmarkType>
using LandmarkCollection = std::vector<Landmark<LandmarkType>>;

// keeps the landmarks whose name is in `filter` (landmark.hpp:51-64)
template <class T>
LandmarkCollection<T> filter(const LandmarkCollection<T>& landmarks, const std::vector<std::string>& filter)
{
    LandmarkCollection<T> out;
    std::copy_if(landmarks.begin(), landmarks.end(), std::back_inserter(out), [&](const Landmark<T>& lm) {
        return std::find(filter.begin(), filter.end(), lm.name) != filter.end();
    });
    return out;
}

}  // namespace rcr
