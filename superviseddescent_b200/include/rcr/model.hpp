// H100 drop-in for include/rcr/model.hpp: align_mean (:64-76), InterEyeDistanceNormalisation (:84-116),
// detection_model (:122-183) and load/save_detection_model (:192-219).  detect() runs the whole cascade
// on the GPU through sd_detect_faces_host; the file format is byte compatible with the reference's
// cereal archives (face_landmarks_model_rcr_22.bin loads unchanged).
#pragma once

#include <array>
#include <string>
#include <vector>

#include "rcr/adaptive_vlhog.hpp"
#include "rcr/helpers.hpp"
#include "superviseddescent/superviseddescent.hpp"
#include "superviseddescent/verbose_solver.hpp"

namespace rcr {

inline cv::Mat align_mean(cv::Mat mean, cv::Rect facebox, float scaling_x = 1.0f, float scaling_y = 1.0f, float translation_x = 0.0f, float translation_y = 0.0f)
{
    cv::Mat aligned(1, mean.cols, CV_32FC1);
    const int rc = sd_align_mean(mean.ptr<float>(0), mean.cols / 2, facebox.x, facebox.y, facebox.width, facebox.height, scaling_x, scaling_y,
                                 translation_x, translation_y, aligned.ptr<float>(0));
    if (rc != SD_OK) throw std::runtime_error("align_mean: bad arguments");
    return aligned;
}

// ---- mirrored samples (the landmark correspondence of a left-right flip; Python: mirror_permutation / mirror_landmarks / mirror_box)
// perm[l] = the position of landmark l's mirror partner in the list, under ibug-68 ids (the rcr_22 and ibug-68 lists use them):
// the pairs 1-17 .. 8-10, 18-27 .. 22-23, 32-36, 33-35, 37-46, 38-45, 39-44, 40-43, 41-48, 42-47, 49-55, 50-54, 51-53, 56-60,
// 57-59, 61-65, 62-64, 66-68; every other id is its own mirror.  Throws when an id is not an ibug-68 id or its partner is not in
// the list; a caller with another id scheme passes its own permutation to mirror_landmarks.
inline std::vector<int> mirror_permutation(const std::vector<std::string>& landmark_ids)
{
    static const int pairs[][2] = {{1, 17}, {2, 16}, {3, 15}, {4, 14}, {5, 13}, {6, 12}, {7, 11}, {8, 10}, {18, 27}, {19, 26},
                                   {20, 25}, {21, 24}, {22, 23}, {32, 36}, {33, 35}, {37, 46}, {38, 45}, {39, 44}, {40, 43},
                                   {41, 48}, {42, 47}, {49, 55}, {50, 54}, {51, 53}, {56, 60}, {57, 59}, {61, 65}, {62, 64}, {66, 68}};
    int partner[69];
    for (int i = 0; i <= 68; ++i) partner[i] = i;
    for (const auto& p : pairs) { partner[p[0]] = p[1]; partner[p[1]] = p[0]; }
    std::vector<int> perm(landmark_ids.size());
    for (size_t k = 0; k < landmark_ids.size(); ++k) {
        const std::string& id = landmark_ids[k];
        int n = 0;
        bool digits = !id.empty() && id.size() <= 2;
        for (char c : id) digits = digits && c >= '0' && c <= '9';
        if (digits) n = std::stoi(id);
        if (!digits || n < 1 || n > 68) throw std::runtime_error("mirror_permutation: landmark id " + id + " is not an ibug-68 id");
        const std::string want = std::to_string(partner[n]);
        size_t j = 0;
        while (j < landmark_ids.size() && landmark_ids[j] != want) ++j;
        if (j == landmark_ids.size()) throw std::runtime_error("mirror_permutation: the mirror partner " + want + " of landmark " + id + " is not in the list");
        perm[k] = static_cast<int>(j);
    }
    return perm;
}

// Landmark rows [x_0 .. x_{L-1}, y_0 .. y_{L-1}] (CV_32FC1, one per row) of left-right mirrored frames: x'[l] = W - 1 - x[perm[l]],
// y'[l] = y[perm[l]], in float, with frame_width[r] the width of row r's frame (one entry: the same width for every row).
inline cv::Mat mirror_landmarks(cv::Mat x, const std::vector<int>& frame_width, const std::vector<int>& perm)
{
    const int L = x.cols / 2;
    if (x.cols != 2 * L || static_cast<int>(perm.size()) != L || frame_width.empty() ||
        (frame_width.size() != 1 && static_cast<int>(frame_width.size()) != x.rows))
        throw std::runtime_error("mirror_landmarks: x must be N x 2L, perm L long and frame_width 1 or N long");
    cv::Mat out(x.rows, x.cols, CV_32FC1);
    for (int r = 0; r < x.rows; ++r) {
        const float w1 = static_cast<float>(frame_width[frame_width.size() == 1 ? 0 : r]) - 1.0f;
        for (int l = 0; l < L; ++l) {
            out.at<float>(r, l) = w1 - x.at<float>(r, perm[l]);
            out.at<float>(r, L + l) = x.at<float>(r, L + perm[l]);
        }
    }
    return out;
}

// a box of a frame of width W as a box of its left-right mirror: (W - x - w, y, w, h)
inline cv::Rect mirror_box(cv::Rect box, int frame_width) { return cv::Rect(frame_width - box.x - box.width, box.y, box.width, box.height); }

// ---- warped samples (Python: rotation_warp / invert_warp / warp_landmarks).  A warp matrix is 2 x 3 doubles, row-major, mapping a
// pixel of the virtual frame V to a position in its frame (include/sd_b200.h, sd_sample_warp); every helper computes in double with
// each operation rounded on its own, in the order of the Python helper, so that both give the same bits.
using warp_matrix = std::array<double, 6>;

// A sample warp: M over a V of width x height
inline sd_sample_warp make_warp(const warp_matrix& m, int width, int height)
{
    sd_sample_warp w{};
    for (int k = 0; k < 6; ++k) w.m[k] = m[k];
    w.width = width;
    w.height = height;
    return w;
}

// The exact algebraic inverse of M; throws when M is singular or not finite
inline warp_matrix invert_warp(const warp_matrix& m)
{
    const double det = m[0] * m[4] - m[1] * m[3];
    if (det == 0 || !std::isfinite(det)) throw std::runtime_error("invert_warp: the matrix is singular or not finite");
    const double ia = m[4] / det, ib = -m[1] / det, id = -m[3] / det, ie = m[0] / det;
    return warp_matrix{ia, ib, -(ia * m[2] + ib * m[5]), id, ie, -(id * m[2] + ie * m[5])};
}

// The V-to-frame matrix whose V is the frame rotated by angle degrees (counter-clockwise) about (cx, cy) and scaled by scale: the
// inverse of cv::getRotationMatrix2D(centre, angle, scale).  Its V is what cv::warpAffine with that matrix gives.
inline warp_matrix rotation_warp(double cx, double cy, double angle, double scale = 1.0)
{
    const double a = angle * (3.141592653589793 / 180.0);
    const double alpha = std::cos(a) * scale, beta = std::sin(a) * scale;
    return invert_warp(warp_matrix{alpha, beta, (1 - alpha) * cx - beta * cy, -beta, alpha, beta * cx + (1 - alpha) * cy});
}

// Landmark rows [x_0 .. x_{L-1}, y_0 .. y_{L-1}] (CV_32FC1, one per row) mapped through one matrix (m.size() == 1) or one per row,
// in double, returned as float: ground truth into a warp's V with invert_warp, results back to the frame with the warp.
inline cv::Mat warp_landmarks(cv::Mat x, const std::vector<warp_matrix>& m)
{
    const int L = x.cols / 2;
    if (x.cols != 2 * L || L < 1 || m.empty() || (m.size() != 1 && static_cast<int>(m.size()) != x.rows))
        throw std::runtime_error("warp_landmarks: x must be N x 2L and m 1 or N long");
    cv::Mat out(x.rows, x.cols, CV_32FC1);
    for (int r = 0; r < x.rows; ++r) {
        const warp_matrix& w = m[m.size() == 1 ? 0 : r];
        for (int l = 0; l < L; ++l) {
            const double px = x.at<float>(r, l), py = x.at<float>(r, L + l);
            out.at<float>(r, l) = static_cast<float>(w[0] * px + w[1] * py + w[2]);
            out.at<float>(r, L + l) = static_cast<float>(w[3] * px + w[4] * py + w[5]);
        }
    }
    return out;
}

class InterEyeDistanceNormalisation {
public:
    InterEyeDistanceNormalisation() = default;
    InterEyeDistanceNormalisation(std::vector<std::string> modelLandmarksList, std::vector<std::string> rightEyeIdentifiers, std::vector<std::string> leftEyeIdentifiers)
        : modelLandmarksList(modelLandmarksList), rightEyeIdentifiers(rightEyeIdentifiers), leftEyeIdentifiers(leftEyeIdentifiers) {}

    // 1 / IED of the given landmark row, replicated (model.hpp:94-98)
    inline cv::Mat operator()(cv::Mat params)
    {
        const double ied = get_ied(to_landmark_collection(params, modelLandmarksList), rightEyeIdentifiers, leftEyeIdentifiers);
        const float n = static_cast<float>(1.0 / ied);
        cv::Mat out(1, params.cols, CV_32FC1);
        for (int i = 0; i < params.cols; ++i) out.at<float>(0, i) = n;
        return out;
    }

    sd_normalisation c_normalisation() const
    {
        sd_normalisation nrm{};
        nrm.kind = 1;
        const auto r = eye_indices(modelLandmarksList, rightEyeIdentifiers, "right");
        const auto l = eye_indices(modelLandmarksList, leftEyeIdentifiers, "left");
        nrm.n_right = static_cast<int>(r.size());
        nrm.n_left = static_cast<int>(l.size());
        for (size_t i = 0; i < r.size() && i < 4; ++i) nrm.right_idx[i] = r[i];
        for (size_t i = 0; i < l.size() && i < 4; ++i) nrm.left_idx[i] = l[i];
        return nrm;
    }

private:
    std::vector<std::string> modelLandmarksList, rightEyeIdentifiers, leftEyeIdentifiers;
};

// One tracking step's result (detection_model::track): per track its new landmarks (1 x 2L), the box of those landmarks, that
// box's face-filter score (NaN for a degenerate box) and whether the track is still alive.
struct tracked_faces {
    std::vector<cv::Mat> landmarks;
    std::vector<cv::Rect> boxes;
    std::vector<float> scores;
    std::vector<bool> alive;
};

// The detector's side of detection_model::track_and_detect: sd_track_detect_param without its scales.
struct track_detect_params {
    int pad_x = 0, pad_y = 0;
    float detect_threshold = 0.f;
    double nms_overlap = 0.5, track_overlap = 0.5;
    int max_candidates = 4096, max_detections = 16;
};

// One step of detection_model::track_and_detect: rows 0..T-1 are the old tracks, rows T.. the num_new new ones; frame[r] is the
// frame row r lies in.
struct track_step : tracked_faces {
    std::vector<int> frame;
    int num_new = 0;
};

class detection_model {
public:
    using model_type = superviseddescent::SupervisedDescentOptimiser<superviseddescent::LinearRegressor<superviseddescent::VerbosePartialPivLUSolver>, InterEyeDistanceNormalisation>;

    detection_model() = default;

    // model.hpp:128-129: a model assembled from a trained optimiser
    detection_model(model_type optimised_model, cv::Mat mean, std::vector<std::string> landmark_ids, std::vector<rcr::HoGParam> hog_params,
                    std::vector<std::string> right_eye_ids, std::vector<std::string> left_eye_ids)
        : landmark_ids(landmark_ids)
    {
        auto& regs = optimised_model.get_regressors();
        std::vector<const float*> w;
        std::vector<sd_regulariser> r;
        std::vector<sd_hog_param> hp;
        std::vector<cv::Mat> keep;
        for (size_t i = 0; i < regs.size(); ++i) {
            keep.push_back(regs[i].x.isContinuous() ? regs[i].x : regs[i].x.clone());
            w.push_back(keep.back().ptr<float>(0));
            r.push_back(regs[i].get_regulariser().c());
            hp.push_back(hog_params[i].c());
        }
        std::vector<const char*> ids, rid, lid;
        for (auto& s : landmark_ids) ids.push_back(s.c_str());
        for (auto& s : right_eye_ids) rid.push_back(s.c_str());
        for (auto& s : left_eye_ids) lid.push_back(s.c_str());
        sd_ctx* ctx = sd_b200::context();
        sd_model* m = nullptr;
        sd_b200::check(ctx, sd_model_create(ctx, static_cast<int>(regs.size()), static_cast<int>(landmark_ids.size()), w.data(), r.data(), hp.data(),
                                            mean.ptr<float>(0), ids.data(), rid.data(), static_cast<int>(rid.size()), lid.data(), static_cast<int>(lid.size()), &m),
                       "sd_model_create");
        handle.reset(m, sd_model_destroy);
    }

    // Run the model from a face box: init with the aligned mean, then optimise (model.hpp:132-144)
    LandmarkCollection<cv::Vec2f> detect(cv::Mat image, cv::Rect facebox)
    {
        return to_landmark_collection(detect(std::vector<cv::Mat>{image}, std::vector<int>{0}, std::vector<cv::Rect>{facebox})[0], landmark_ids);
    }

    // Run the model from a landmark initialisation, e.g. the previous frame (model.hpp:147-157)
    LandmarkCollection<cv::Vec2f> detect(cv::Mat image, cv::Mat initialisation)
    {
        return to_landmark_collection(detect(std::vector<cv::Mat>{image}, std::vector<int>{0}, initialisation)[0], landmark_ids);
    }

    // Batched detect: one face box per frame, frames of any sizes; returns one 1 x 2L row per frame.
    std::vector<cv::Mat> detect(const std::vector<cv::Mat>& images, const std::vector<cv::Rect>& faceboxes)
    {
        if (images.empty() || images.size() != faceboxes.size()) throw std::runtime_error("detect: images / faceboxes size mismatch");
        std::vector<int> face_image(images.size());
        for (size_t i = 0; i < images.size(); ++i) face_image[i] = static_cast<int>(i);
        return detect(images, face_image, faceboxes);
    }

    // Several faces per frame: face i lies in images[face_image[i]]; frames 8UC1 or 8UC3 (B,G,R), any sizes and row steps.
    // Returns one 1 x 2L row per face.
    std::vector<cv::Mat> detect(const std::vector<cv::Mat>& images, const std::vector<int>& face_image, const std::vector<cv::Rect>& faceboxes)
    {
        if (face_image.size() != faceboxes.size()) throw std::runtime_error("detect: face_image / faceboxes size mismatch");
        std::vector<int32_t> boxes(4 * faceboxes.size());
        for (size_t i = 0; i < faceboxes.size(); ++i) {
            boxes[4 * i] = faceboxes[i].x; boxes[4 * i + 1] = faceboxes[i].y; boxes[4 * i + 2] = faceboxes[i].width; boxes[4 * i + 3] = faceboxes[i].height;
        }
        return detect_faces(images, face_image, boxes.data(), nullptr);
    }

    // Several faces per frame, each from a landmark initialisation (one 1 x 2L row per face, e.g. the previous frame's result).
    std::vector<cv::Mat> detect(const std::vector<cv::Mat>& images, const std::vector<int>& face_image, cv::Mat initialisations)
    {
        const int P = 2 * sd_model_num_landmarks(handle.get());
        if (initialisations.rows != static_cast<int>(face_image.size()) || initialisations.cols != P)
            throw std::runtime_error("detect: initialisations must be one 1 x 2L row per face");
        const cv::Mat x0 = initialisations.isContinuous() ? initialisations : initialisations.clone();
        return detect_faces(images, face_image, nullptr, x0.ptr<float>(0));
    }

    // Warped faces (sd_detect_faces_device_warped): face i is a face of the virtual frame V_i = cv::warpAffine(grey
    // images[face_image[i]], warps[i].m, (warps[i].width, warps[i].height), INTER_LINEAR | WARP_INVERSE_MAP) (rcr::make_warp,
    // rcr::rotation_warp); its box and its landmarks are in V_i's coordinates, bit for bit detect() on V_i.  The frames are
    // uploaded once (sd_upload_frames) and V_i is never built.  Returns one 1 x 2L row per face.
    std::vector<cv::Mat> detect(const std::vector<cv::Mat>& images, const std::vector<int>& face_image, const std::vector<cv::Rect>& faceboxes,
                                const std::vector<sd_sample_warp>& warps)
    {
        if (face_image.size() != faceboxes.size()) throw std::runtime_error("detect: face_image / faceboxes size mismatch");
        const cv::Mat mean = get_mean();
        cv::Mat x0(static_cast<int>(faceboxes.size()), mean.cols, CV_32FC1);
        for (size_t i = 0; i < faceboxes.size(); ++i) {
            const cv::Mat row = align_mean(mean, faceboxes[i]);
            std::memcpy(x0.ptr<float>(static_cast<int>(i)), row.ptr<float>(0), sizeof(float) * mean.cols);
        }
        return detect_warped(images, face_image, x0, warps);
    }

    std::vector<cv::Mat> detect(const std::vector<cv::Mat>& images, const std::vector<int>& face_image, cv::Mat initialisations,
                                const std::vector<sd_sample_warp>& warps)
    {
        const int P = 2 * sd_model_num_landmarks(handle.get());
        if (initialisations.rows != static_cast<int>(face_image.size()) || initialisations.cols != P)
            throw std::runtime_error("detect: initialisations must be one 1 x 2L row per face");
        return detect_warped(images, face_image, initialisations.isContinuous() ? initialisations : initialisations.clone(), warps);
    }

    // One tracking step (sd_track_faces; the rule is in include/sd_b200.h): track t lies in images[face_frame[t]] and had the
    // landmarks previous.row(t) (T x 2L, CV_32FC1).  Each track restarts the cascade from align_mean of the box of its previous
    // landmarks (bit for bit detect() from that box), and its new landmarks' box is scored by the face filter; it stays alive
    // while that box is valid, its score exceeds threshold and no cascade level had an empty patch.  A track whose previous box
    // is degenerate dies and keeps its previous landmarks.  images: 8UC1 or 8UC3 (B,G,R) frames of any sizes, uploaded as grey
    // (hog_batch::upload_grey).  There is no tracker state: drop the dead tracks and start new ones from vl_hog_detect boxes.
    // multichannel, bilinear_orientations and float_frames as vl_hog_detect takes them (sd_track_faces_images): a filter trained
    // on colour or float frames scores the boxes on the frames as given, while the cascade reads grey frames -- 8UC3 frames
    // converted on the device after one upload, 8UC1 frames as they are, or *grey_images (needed for CV_32FC1 / CV_32FC3 frames;
    // hog_batch::upload_track_frames).  Throws std::runtime_error where sd_track_faces or sd_track_faces_images refuses.
    tracked_faces track(const std::vector<cv::Mat>& images, const std::vector<int>& face_frame, cv::Mat previous, const hog_filter& filter,
                        VlHogVariant variant, int cell_size, int num_bins, float threshold, bool multichannel = false,
                        bool bilinear_orientations = false, bool float_frames = false, const std::vector<cv::Mat>* grey_images = nullptr)
    {
        const int P = 2 * sd_model_num_landmarks(handle.get()), T = static_cast<int>(face_frame.size());
        if (images.empty()) throw std::runtime_error("track: no frames");
        if (previous.rows != T || previous.cols != P || previous.type() != CV_32FC1)
            throw std::runtime_error("track: previous must be one 1 x 2L CV_32FC1 row per track");
        const int dd = sd_b200::hog_dimension(variant, num_bins);
        if (filter.filter.type() != CV_32FC1 || filter.filter.empty() || filter.filter.rows % dd != 0)
            throw std::runtime_error("track: the filter must be a CV_32FC1 Mat of dd * fh rows and fw columns");
        tracked_faces out;
        if (T == 0) return out;
        sd_ctx* ctx = sd_b200::context();
        sd_b200::DeviceBuffer d_filter, d_prev, d_frame(static_cast<size_t>(T) * sizeof(int32_t));
        sd_b200::DeviceBuffer d_lms(static_cast<size_t>(T) * P * sizeof(float)), d_boxes(static_cast<size_t>(T) * 4 * sizeof(int32_t));
        sd_b200::DeviceBuffer d_scores(static_cast<size_t>(T) * sizeof(float)), d_alive(static_cast<size_t>(T));
        hog_batch::TrackFrames fr;
        hog_batch::upload_track_frames(ctx, images, multichannel, bilinear_orientations, float_frames, grey_images, fr, "track upload");
        sd_b200::upload(filter.filter, d_filter, filter.filter.cols);
        sd_b200::upload(previous, d_prev, P);
        const std::vector<int32_t> idx(face_frame.begin(), face_frame.end());
        sd_b200::check(ctx, sd_memcpy_h2d(ctx, d_frame.as<int32_t>(), idx.data(), idx.size() * sizeof(int32_t)), "track");
        if (multichannel)
            sd_b200::check(ctx, sd_track_faces_images(ctx, handle.get(), &fr.grey, &fr.colour, bilinear_orientations ? 1 : 0, d_frame.as<int32_t>(),
                                                      d_prev.as<float>(), T, d_filter.as<float>(), filter.filter.cols, filter.filter.rows / dd,
                                                      filter.bias, cell_size, num_bins, variant, threshold, d_lms.as<float>(),
                                                      d_boxes.as<int32_t>(), d_scores.as<float>(), d_alive.as<uint8_t>()),
                           "sd_track_faces_images");
        else
            sd_b200::check(ctx, sd_track_faces(ctx, handle.get(), &fr.grey, d_frame.as<int32_t>(), d_prev.as<float>(), T, d_filter.as<float>(),
                                               filter.filter.cols, filter.filter.rows / dd, filter.bias, cell_size, num_bins, variant, threshold,
                                               d_lms.as<float>(), d_boxes.as<int32_t>(), d_scores.as<float>(), d_alive.as<uint8_t>()),
                           "sd_track_faces");
        std::vector<int32_t> boxes(static_cast<size_t>(T) * 4);
        std::vector<uint8_t> alive(T);
        out.scores.resize(T);
        sd_b200::check(ctx, sd_memcpy_d2h(ctx, boxes.data(), d_boxes.as<int32_t>(), boxes.size() * sizeof(int32_t)), "track");
        sd_b200::check(ctx, sd_memcpy_d2h(ctx, out.scores.data(), d_scores.as<float>(), out.scores.size() * sizeof(float)), "track");
        sd_b200::check(ctx, sd_memcpy_d2h(ctx, alive.data(), d_alive.as<uint8_t>(), alive.size()), "track");
        const cv::Mat lms = sd_b200::download(d_lms.as<float>(), T, P, P);   // synchronises
        for (int t = 0; t < T; ++t) {
            out.landmarks.push_back(lms.row(t).clone());
            out.boxes.push_back(cv::Rect(boxes[4 * t], boxes[4 * t + 1], boxes[4 * t + 2], boxes[4 * t + 3]));
            out.alive.push_back(alive[t] != 0);
        }
        return out;
    }

    // One tracking step that also detects (sd_track_detect_faces; the rule is in include/sd_b200.h): the tracks step as in
    // track(), the face filter runs as vl_hog_detect on the frames detect_frames lists (distinct indices; the pyramid's scales),
    // a detection that no alive track of its frame overlaps by IoU > params.track_overlap starts a new row from its box, and
    // within each frame the alive rows are kept greedily (old rows first, then by score) unless a kept row overlaps them.  The
    // frames are uploaded once (hog_batch::upload_grey).  previous may be empty when face_frame is.  multichannel,
    // bilinear_orientations, float_frames and grey_images as track() takes them: the box scores and the detector
    // (vl_hog_detect with the same options) read the frames as given, the cascade their grey (sd_track_detect_faces_images).
    // Throws std::runtime_error where sd_track_detect_faces or sd_track_detect_faces_images refuses.
    track_step track_and_detect(const std::vector<cv::Mat>& images, const std::vector<int>& face_frame, cv::Mat previous,
                                const hog_filter& filter, VlHogVariant variant, int cell_size, int num_bins, float threshold,
                                const std::vector<double>& scales, const std::vector<int>& detect_frames, const track_detect_params& params,
                                bool multichannel = false, bool bilinear_orientations = false, bool float_frames = false,
                                const std::vector<cv::Mat>* grey_images = nullptr)
    {
        const int P = 2 * sd_model_num_landmarks(handle.get()), T = static_cast<int>(face_frame.size());
        if (images.empty()) throw std::runtime_error("track_and_detect: no frames");
        if (T > 0 && (previous.rows != T || previous.cols != P || previous.type() != CV_32FC1))
            throw std::runtime_error("track_and_detect: previous must be one 1 x 2L CV_32FC1 row per track");
        const int dd = sd_b200::hog_dimension(variant, num_bins);
        if (filter.filter.type() != CV_32FC1 || filter.filter.empty() || filter.filter.rows % dd != 0)
            throw std::runtime_error("track_and_detect: the filter must be a CV_32FC1 Mat of dd * fh rows and fw columns");
        if (params.max_detections < 1) throw std::runtime_error("track_and_detect: max_detections must be at least 1");
        const size_t R = static_cast<size_t>(T) + detect_frames.size() * static_cast<size_t>(params.max_detections);
        sd_ctx* ctx = sd_b200::context();
        sd_b200::DeviceBuffer d_filter, d_prev, d_face(static_cast<size_t>(T) * sizeof(int32_t) + 4);
        sd_b200::DeviceBuffer d_lms(R * P * sizeof(float) + 4), d_boxes(R * 4 * sizeof(int32_t) + 4), d_scores(R * sizeof(float) + 4);
        sd_b200::DeviceBuffer d_alive(R + 4), d_frame(R * sizeof(int32_t) + 4);
        hog_batch::TrackFrames fr;
        hog_batch::upload_track_frames(ctx, images, multichannel, bilinear_orientations, float_frames, grey_images, fr,
                                       "track_and_detect upload");
        sd_b200::upload(filter.filter, d_filter, filter.filter.cols);
        if (T > 0) sd_b200::upload(previous, d_prev, P);
        const std::vector<int32_t> idx(face_frame.begin(), face_frame.end()), listed(detect_frames.begin(), detect_frames.end());
        if (T > 0) sd_b200::check(ctx, sd_memcpy_h2d(ctx, d_face.as<int32_t>(), idx.data(), idx.size() * sizeof(int32_t)), "track_and_detect");
        sd_track_detect_param p;
        p.h_scales = scales.data();
        p.num_scales = static_cast<int32_t>(scales.size());
        p.pad_x = params.pad_x; p.pad_y = params.pad_y;
        p.detect_threshold = params.detect_threshold;
        p.nms_overlap = params.nms_overlap; p.track_overlap = params.track_overlap;
        p.max_candidates = params.max_candidates; p.max_detections = params.max_detections;
        int32_t num_new = 0;
        if (multichannel)
            sd_b200::check(ctx, sd_track_detect_faces_images(ctx, handle.get(), &fr.grey, &fr.colour, bilinear_orientations ? 1 : 0,
                                                             d_face.as<int32_t>(), d_prev.as<float>(), T, d_filter.as<float>(), filter.filter.cols,
                                                             filter.filter.rows / dd, filter.bias, cell_size, num_bins, variant, threshold,
                                                             listed.data(), static_cast<int>(listed.size()), &p, d_lms.as<float>(),
                                                             d_boxes.as<int32_t>(), d_scores.as<float>(), d_alive.as<uint8_t>(),
                                                             d_frame.as<int32_t>(), &num_new),
                           "sd_track_detect_faces_images");
        else
            sd_b200::check(ctx, sd_track_detect_faces(ctx, handle.get(), &fr.grey, d_face.as<int32_t>(), d_prev.as<float>(), T, d_filter.as<float>(),
                                                      filter.filter.cols, filter.filter.rows / dd, filter.bias, cell_size, num_bins, variant,
                                                      threshold, listed.data(), static_cast<int>(listed.size()), &p, d_lms.as<float>(),
                                                      d_boxes.as<int32_t>(), d_scores.as<float>(), d_alive.as<uint8_t>(), d_frame.as<int32_t>(),
                                                      &num_new),
                           "sd_track_detect_faces");
        const int rows = T + num_new;
        track_step out;
        out.num_new = num_new;
        if (rows == 0) return out;
        std::vector<int32_t> boxes(static_cast<size_t>(rows) * 4), frame(rows);
        std::vector<uint8_t> alive(rows);
        out.scores.resize(rows);
        sd_b200::check(ctx, sd_memcpy_d2h(ctx, boxes.data(), d_boxes.as<int32_t>(), boxes.size() * sizeof(int32_t)), "track_and_detect");
        sd_b200::check(ctx, sd_memcpy_d2h(ctx, out.scores.data(), d_scores.as<float>(), out.scores.size() * sizeof(float)), "track_and_detect");
        sd_b200::check(ctx, sd_memcpy_d2h(ctx, alive.data(), d_alive.as<uint8_t>(), alive.size()), "track_and_detect");
        sd_b200::check(ctx, sd_memcpy_d2h(ctx, frame.data(), d_frame.as<int32_t>(), frame.size() * sizeof(int32_t)), "track_and_detect");
        const cv::Mat lms = sd_b200::download(d_lms.as<float>(), rows, P, P);   // synchronises
        for (int r = 0; r < rows; ++r) {
            out.landmarks.push_back(lms.row(r).clone());
            out.boxes.push_back(cv::Rect(boxes[4 * r], boxes[4 * r + 1], boxes[4 * r + 2], boxes[4 * r + 3]));
            out.alive.push_back(alive[r] != 0);
            out.frame.push_back(frame[r]);
        }
        return out;
    }

    cv::Mat get_mean()
    {
        cv::Mat mean(1, 2 * sd_model_num_landmarks(handle.get()), CV_32FC1);
        sd_model_get_mean(handle.get(), mean.ptr<float>(0));
        return mean;
    }

    sd_model* native() const { return handle.get(); }

private:
    friend detection_model load_detection_model(std::string filename);
    // sd_detect_faces_host: frames stay in host memory (Mat::step() is the row stride), landmarks come back in face order
    std::vector<cv::Mat> detect_warped(const std::vector<cv::Mat>& images, const std::vector<int>& face_image, const cv::Mat& x0,
                                       const std::vector<sd_sample_warp>& warps)
    {
        const size_t n = face_image.size();
        if (warps.size() != n) throw std::runtime_error("detect: warps needs one entry per face");
        std::vector<cv::Mat> out;
        if (n == 0) return out;
        for (int f : face_image)
            if (f < 0 || f >= static_cast<int>(images.size())) throw std::runtime_error("detect: a face refers to a frame that is not in the list");
        sd_ctx* ctx = sd_b200::context();
        const int P = 2 * sd_model_num_landmarks(handle.get());
        sd_b200::DeviceBuffer frames, didx(n * sizeof(int32_t)), dw(n * sizeof(sd_sample_warp)), dx0(n * P * sizeof(float)),
            dout(n * P * sizeof(float));
        const sd_image_batch batch = hog_batch::upload_grey(ctx, sd_b200::host_frames(images), frames, "detect upload");
        const std::vector<int32_t> idx(face_image.begin(), face_image.end());
        sd_b200::check(ctx, sd_memcpy_h2d(ctx, didx.as<int32_t>(), idx.data(), n * sizeof(int32_t)), "detect");
        sd_b200::check(ctx, sd_memcpy_h2d(ctx, dw.as<sd_sample_warp>(), warps.data(), n * sizeof(sd_sample_warp)), "detect");
        sd_b200::check(ctx, sd_memcpy_h2d(ctx, dx0.as<float>(), x0.ptr<float>(0), n * P * sizeof(float)), "detect");
        sd_b200::check(ctx, sd_detect_faces_device_warped(ctx, handle.get(), &batch, didx.as<int32_t>(), dw.as<sd_sample_warp>(), dx0.as<float>(),
                                                          static_cast<int>(n), dout.as<float>()), "sd_detect_faces_device_warped");
        const cv::Mat all = sd_b200::download(dout.as<float>(), static_cast<int>(n), P, P);
        for (size_t i = 0; i < n; ++i) {
            cv::Mat row(1, P, CV_32FC1);
            std::memcpy(row.ptr<float>(0), all.ptr<float>(static_cast<int>(i)), sizeof(float) * P);
            out.push_back(row);
        }
        return out;
    }

    std::vector<cv::Mat> detect_faces(const std::vector<cv::Mat>& images, const std::vector<int>& face_image, const int32_t* boxes, const float* x0)
    {
        sd_ctx* ctx = sd_b200::context();
        const int P = 2 * sd_model_num_landmarks(handle.get());
        const std::vector<sd_host_frame> frames = sd_b200::host_frames(images);
        const std::vector<int32_t> idx(face_image.begin(), face_image.end());
        std::vector<float> lms(face_image.size() * P);
        sd_b200::check(ctx, sd_detect_faces_host(ctx, handle.get(), frames.data(), static_cast<int>(frames.size()), idx.data(), static_cast<int>(idx.size()),
                                                 boxes, x0, lms.data()), "sd_detect_faces_host");
        std::vector<cv::Mat> out;
        for (size_t i = 0; i < face_image.size(); ++i) {
            cv::Mat row(1, P, CV_32FC1);
            std::memcpy(row.ptr<float>(0), &lms[i * P], sizeof(float) * P);
            out.push_back(row);
        }
        return out;
    }

    std::shared_ptr<sd_model> handle;
    std::vector<std::string> landmark_ids;
};

// model.hpp:192-205
inline detection_model load_detection_model(std::string filename)
{
    sd_ctx* ctx = sd_b200::context();
    sd_model* m = nullptr;
    const int rc = sd_model_load(ctx, filename.c_str(), &m);
    if (rc != SD_OK) throw std::runtime_error(sd_last_error(ctx));   // "The given model file could not be opened: ..." (model.hpp:199)
    detection_model model;
    model.handle.reset(m, sd_model_destroy);
    for (int i = 0; i < sd_model_num_landmarks(m); ++i) model.landmark_ids.emplace_back(sd_model_landmark_id(m, i));
    return model;
}

// model.hpp:214-219
inline void save_detection_model(detection_model model, std::string filename)
{
    sd_ctx* ctx = sd_b200::context();
    sd_b200::check(ctx, sd_model_save(ctx, model.native(), filename.c_str()), "save_detection_model");
}

// Aligned face chips (sd_face_chips; the rule is in include/sd_b200.h): chips[i] is cv::warpAffine(images[face_frame[i]], M_i,
// (chip_width, chip_height), INTER_LINEAR | WARP_INVERSE_MAP, BORDER_CONSTANT, 0), bit for bit, with M_i = chip_to_frame[i] (row-major
// 2 x 3) the least-squares similarity from the default template (sd_face_chip_template at padding) to landmarks.row(i).
// frame_to_chip[i] is its inverse, and valid[i] is false for a face the rule calls invalid (a zero chip and zero transforms).
struct face_chip_set {
    std::vector<cv::Mat> chips;              // the images' type: CV_8UC1 / CV_8UC3 or CV_32FC1 / CV_32FC3
    std::vector<std::array<double, 6>> chip_to_frame, frame_to_chip;
    std::vector<bool> valid;
};

// images: all CV_8UC1, all CV_8UC3, all CV_32FC1 or all CV_32FC3, of any sizes; landmarks: one 1 x 2L CV_32FC1 row per face
// (e.g. a track_step's landmarks stacked); landmark_ids: the landmarks to fit, by id (empty: all of the model's).  Throws
// std::runtime_error where sd_face_chip_template or sd_face_chips refuses.
inline face_chip_set face_chips(const std::vector<cv::Mat>& images, const std::vector<int>& face_frame, const cv::Mat& landmarks,
                                const detection_model& model, int chip_width, int chip_height, double padding = 0.25,
                                const std::vector<std::string>& landmark_ids = {})
{
    sd_model* m = model.native();
    const int L = sd_model_num_landmarks(m), n = static_cast<int>(face_frame.size());
    if (images.empty()) throw std::runtime_error("face_chips: no frames");
    if (n > 0 && (landmarks.type() != CV_32FC1 || landmarks.cols != 2 * L || landmarks.rows != n))
        throw std::runtime_error("face_chips: landmarks must be one 1 x 2L CV_32FC1 row per face");
    std::vector<int32_t> idx;
    for (const std::string& id : landmark_ids) {
        int k = 0;
        while (k < L && id != sd_model_landmark_id(m, k)) ++k;
        if (k == L) throw std::runtime_error("face_chips: landmark id " + id + " is not one of the model's");
        idx.push_back(k);
    }
    if (idx.empty())
        for (int k = 0; k < L; ++k) idx.push_back(k);
    std::vector<double> tmpl(2 * idx.size());
    if (sd_face_chip_template(m, chip_width, chip_height, padding, static_cast<int>(idx.size()), idx.data(), tmpl.data()) != SD_OK)
        throw std::runtime_error("face_chips: sd_face_chip_template refused the chip size, padding or landmarks");
    sd_ctx* ctx = sd_b200::context();
    const int type = images[0].type();
    const bool is_float = type == CV_32FC1 || type == CV_32FC3;
    hog_batch::WindowFrames fr;
    hog_batch::upload_window_frames(ctx, images, true, false, is_float, fr, "face_chips upload");
    const sd_hog_images& frames = fr.colour;
    const size_t chip_bytes = static_cast<size_t>(chip_width) * chip_height * frames.channels * (is_float ? sizeof(float) : 1);
    const size_t rows = static_cast<size_t>(n > 0 ? n : 1), P = 2 * static_cast<size_t>(L);
    sd_b200::DeviceBuffer d_frame(rows * sizeof(int32_t)), d_lms(rows * P * sizeof(float)), d_chips(chip_bytes * rows),
        d_c2f(rows * 6 * sizeof(double)), d_f2c(rows * 6 * sizeof(double)), d_valid(rows);
    const std::vector<int32_t> ff(face_frame.begin(), face_frame.end());
    if (n > 0) {
        sd_b200::check(ctx, sd_memcpy_h2d(ctx, d_frame.as<int32_t>(), ff.data(), ff.size() * sizeof(int32_t)), "face_chips");
        sd_b200::check(ctx, sd_memcpy2d_h2d(ctx, d_lms.as<float>(), P * sizeof(float), landmarks.ptr<float>(0), landmarks.step(),
                                            P * sizeof(float), static_cast<size_t>(n)), "face_chips");
    }
    const sd_face_chip_param p{chip_width, chip_height, static_cast<int32_t>(idx.size()), idx.data(), tmpl.data()};
    sd_b200::check(ctx, sd_face_chips(ctx, &frames, d_frame.as<int32_t>(), d_lms.as<float>(), static_cast<int64_t>(P), n, L, &p,
                                      d_chips.as<void>(), d_c2f.as<double>(), d_f2c.as<double>(), d_valid.as<uint8_t>()), "sd_face_chips");
    face_chip_set out;
    out.chip_to_frame.resize(n);
    out.frame_to_chip.resize(n);
    std::vector<uint8_t> valid(n);
    for (int i = 0; i < n; ++i) {
        out.chips.emplace_back(chip_height, chip_width, type);
        sd_b200::check(ctx, sd_memcpy_d2h(ctx, out.chips[i].ptr<unsigned char>(0), d_chips.as<unsigned char>() + chip_bytes * i, chip_bytes),
                       "face_chips");
    }
    if (n > 0) {
        sd_b200::check(ctx, sd_memcpy_d2h(ctx, out.chip_to_frame.data(), d_c2f.as<double>(), n * 6 * sizeof(double)), "face_chips");
        sd_b200::check(ctx, sd_memcpy_d2h(ctx, out.frame_to_chip.data(), d_f2c.as<double>(), n * 6 * sizeof(double)), "face_chips");
        sd_b200::check(ctx, sd_memcpy_d2h(ctx, valid.data(), d_valid.as<uint8_t>(), valid.size()), "face_chips");
    }
    sd_b200::check(ctx, sd_sync(ctx), "face_chips");
    for (int i = 0; i < n; ++i) out.valid.push_back(valid[i] != 0);
    return out;
}

}  // namespace rcr
