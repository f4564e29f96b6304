// landmark_selection.cpp -- the landmark gate in front of solve(): LandmarkSelector and the schemes the production node
// chains (reference: landmark_selector.hpp:118-253, src/landmark_selection_scheme_{cheirality,voxel,add_depth,helpers}.cpp).
// Host code like in the reference; no PCL / boost: the voxel scheme restates those library steps (see its header).
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <limits>
#include <iterator>
#include <stdexcept>

#include "keyframe_bundle_adjustment/landmark_selector.hpp"
#include "keyframe_bundle_adjustment/internal/landmark_selection_scheme_helpers.hpp"

namespace keyframe_bundle_adjustment {

// ---- cheirality (landmark_selection_scheme_cheirality.cpp:22-60) -----------------------------------------------------------
std::set<LandmarkId> LandmarkRejectionSchemeCheirality::getSelection(const LandmarkMap& landmarks,
                                                                     const KeyframeMap& keyframes) const {
    std::set<LandmarkId> out;
    for (const auto& lm_el : landmarks) {
        bool ok = true;
        for (const auto& id_kf : keyframes) {
            if (!id_kf.second->is_active_) continue;
            for (const auto& cam_lm : id_kf.second->getProjectedLandmarkPosition(lm_el))
                if (cam_lm.second.z() < 0.) { ok = false; break; }
            if (!ok) break;
        }
        if (ok) out.insert(lm_el.first);
    }
    return out;
}

// ---- helpers (landmark_selection_scheme_helpers.cpp) -------------------------------------------------------------------------
namespace landmark_helpers {

std::vector<LandmarkId> chooseNearLmIds(size_t max_num_lms, const std::vector<LandmarkId>& near_ids,
                                        const std::map<LandmarkId, double>& map_flow) {
    std::vector<LandmarkId> with_flow;  // tracks seen once have no flow value
    for (const auto& id : near_ids)
        if (map_flow.count(id)) with_flow.push_back(id);
    std::vector<LandmarkId> out(std::min(max_num_lms, with_flow.size()));
    const auto it = std::partial_sort_copy(with_flow.cbegin(), with_flow.cend(), out.begin(), out.end(),
                                           [&](const LandmarkId& a, const LandmarkId& b) { return map_flow.at(a) > map_flow.at(b); });
    if (it != out.end()) throw std::runtime_error("In LandmarkSelectionSchemeHelpers: Not all chosen ids of near field have been copied!");
    return out;
}

std::vector<LandmarkId> chooseMiddleLmIds(size_t max_num, const std::vector<LandmarkId>& middle_ids) {
    std::vector<LandmarkId> a(middle_ids);
    // std::random_shuffle(first, last) of libstdc++ (removed from the language in C++17): driven by std::rand()
    for (size_t i = 1; i < a.size(); ++i) {
        const size_t j = size_t(std::rand()) % (i + 1);
        if (i != j) std::swap(a[i], a[j]);
    }
    a.resize(std::min(max_num, a.size()));
    return a;
}

std::vector<LandmarkId> chooseFarLmIds(size_t max_num, const std::vector<LandmarkId>& ids_far,
                                       const std::map<KeyframeId, Keyframe::ConstPtr>& keyframes) {
    std::map<LandmarkId, unsigned int> seen;  // keyframes observing the landmark
    for (const auto& id : ids_far) {
        unsigned int n = 0;
        for (const auto& kf : keyframes) n += kf.second->hasMeasurement(id) ? 1u : 0u;
        seen[id] = n;
    }
    return chooseFarLmIds(max_num, ids_far, seen);
}

std::vector<LandmarkId> chooseFarLmIds(size_t max_num, const std::vector<LandmarkId>& ids_far,
                                       const std::map<LandmarkId, unsigned int>& seen) {
    std::vector<LandmarkId> out(std::min(max_num, ids_far.size()));
    std::partial_sort_copy(ids_far.cbegin(), ids_far.cend(), out.begin(), out.end(),
                           [&](const LandmarkId& a, const LandmarkId& b) { return seen.at(a) > seen.at(b); });
    return out;
}

std::map<LandmarkId, double> calcFlow(const std::vector<LandmarkId>& lm_ids, const std::vector<Keyframe::ConstPtr>& sorted_kfs,
                                      bool use_mean) {
    std::map<LandmarkId, double> out;
    for (const auto& lm_id : lm_ids) {
        std::map<CameraId, Measurement> last;
        std::map<CameraId, double> flow;
        std::map<CameraId, int> count;
        for (const auto& kf : sorted_kfs)
            for (const auto& cam_meas : kf->getMeasurements(lm_id)) {
                auto it = last.find(cam_meas.first);
                if (it != last.end()) {
                    flow[cam_meas.first] += (it->second.toEigen2d() - cam_meas.second.toEigen2d()).norm();
                    count[cam_meas.first] += 1;
                }
                last[cam_meas.first] = cam_meas.second;
            }
        if (use_mean)
            for (auto& el : flow) el.second /= count.at(el.first);
        // maximum over the cameras; the reference dereferences max_element of an empty map for a track seen once
        // (helpers.cpp:127-129, undefined behaviour) -- such a landmark simply gets no flow value here
        if (flow.empty()) continue;
        out[lm_id] = std::max_element(flow.cbegin(), flow.cend(), [](const auto& a, const auto& b) { return a.second < b.second; })->second;
    }
    return out;
}

std::map<LandmarkId, double> calcFlow(const std::vector<LandmarkId>& lm_ids, const std::map<KeyframeId, Keyframe::ConstPtr>& keyframes,
                                      bool use_mean) {
    // The reference sorts the shared_ptrs themselves (`a < b` on the pointers, helpers.cpp:206), i.e. by address; flow is a
    // sum of distances between consecutive observations, so any other order than time would be meaningless: time order.
    std::vector<Keyframe::ConstPtr> kfs;
    for (const auto& el : keyframes) kfs.push_back(el.second);
    std::sort(kfs.begin(), kfs.end(), [](const auto& a, const auto& b) { return a->timestamp_ < b->timestamp_; });
    return calcFlow(lm_ids, kfs, use_mean);
}

}  // namespace landmark_helpers

namespace keyframe_helpers {
std::vector<Keyframe::ConstPtr> getSortedKeyframes(const std::map<KeyframeId, Keyframe::ConstPtr>& keyframes) {
    std::vector<Keyframe::ConstPtr> out;
    for (const auto& kf : keyframes)
        if (kf.second->is_active_) out.push_back(kf.second);
    std::sort(out.begin(), out.end(), [](const auto& a, const auto& b) { return a->timestamp_ > b->timestamp_; });
    return out;
}
}  // namespace keyframe_helpers

// ---- voxel sparsification (landmark_selection_scheme_voxel.cpp:116-234) ---------------------------------------------------
namespace {

struct LabelledPoint { float x, y, z; uint32_t label; };  // pcl::PointXYZL

// boost::geometry::distance(point, linestring): distance to the nearest segment (to the point, for a one-point path)
double distance_to_path(const LabelledPoint& p, const std::vector<Eigen::Vector3d>& path) {
    const Eigen::Vector3d q(p.x, p.y, p.z);
    if (path.size() == 1) return (q - path[0]).norm();
    double best = std::numeric_limits<double>::max();
    for (size_t i = 0; i + 1 < path.size(); ++i) {
        const Eigen::Vector3d v = path[i + 1] - path[i], w = q - path[i];
        const double c1 = w.dot(v), c2 = v.dot(v);
        double d2;
        if (c1 <= 0.) d2 = w.squaredNorm();
        else if (c2 <= c1) d2 = (q - path[i + 1]).squaredNorm();
        else d2 = (q - (path[i] + v * (c1 / c2))).squaredNorm();
        best = std::min(best, d2);
    }
    return std::sqrt(best);
}

// filterPipe (voxel.cpp:90-113): points closer than `thres` to the keyframe path go on, the labels of the others are kept
void filter_pipe(const std::vector<LabelledPoint>& in, const std::vector<Eigen::Vector3d>& path, double thres,
                 std::vector<LabelledPoint>& kept, std::set<uint32_t>& removed) {
    for (const auto& p : in) {
        if (distance_to_path(p, path) < thres) kept.push_back(p);
        else removed.insert(p.label);
    }
}

// pcl::VoxelGrid<PointXYZL>::applyFilter with downsample_all_data (PCL 1.8): voxel index from floor(p / leaf) relative to
// the cloud's minimum, output in ascending voxel index, one centroid per voxel (float accumulation), label = the most
// frequent one, ties to the smallest (labels are unique here, so: the smallest label of the voxel)
std::vector<LabelledPoint> voxel_grid(const std::vector<LabelledPoint>& in, const std::array<double, 3>& leaf) {
    std::vector<LabelledPoint> out;
    if (in.empty()) return out;
    const float inv[3] = {1.0f / float(leaf[0]), 1.0f / float(leaf[1]), 1.0f / float(leaf[2])};
    float mn[3] = {in[0].x, in[0].y, in[0].z}, mx[3] = {in[0].x, in[0].y, in[0].z};
    for (const auto& p : in) {
        const float c[3] = {p.x, p.y, p.z};
        for (int a = 0; a < 3; ++a) { mn[a] = std::min(mn[a], c[a]); mx[a] = std::max(mx[a], c[a]); }
    }
    int min_b[3], div_b[3];
    for (int a = 0; a < 3; ++a) {
        min_b[a] = int(std::floor(mn[a] * inv[a]));
        div_b[a] = int(std::floor(mx[a] * inv[a])) - min_b[a] + 1;
    }
    const long long mul[3] = {1, div_b[0], (long long)div_b[0] * div_b[1]};
    std::vector<std::pair<long long, size_t>> index;  // (voxel, point)
    index.reserve(in.size());
    for (size_t i = 0; i < in.size(); ++i) {
        const float c[3] = {in[i].x, in[i].y, in[i].z};
        long long idx = 0;
        for (int a = 0; a < 3; ++a) idx += (long long)(int(std::floor(c[a] * inv[a]) - float(min_b[a]))) * mul[a];
        index.emplace_back(idx, i);
    }
    std::sort(index.begin(), index.end());  // PCL sorts by voxel only; the centroid and the label do not depend on the order inside
    for (size_t a = 0; a < index.size();) {
        size_t b = a;
        float sx = 0.f, sy = 0.f, sz = 0.f;
        uint32_t label = std::numeric_limits<uint32_t>::max();
        for (; b < index.size() && index[b].first == index[a].first; ++b) {
            const LabelledPoint& p = in[index[b].second];
            sx += p.x; sy += p.y; sz += p.z;
            label = std::min(label, p.label);
        }
        const float n = float(b - a);
        out.push_back({sx / n, sy / n, sz / n, label});
        a = b;
    }
    return out;
}

}  // namespace

std::set<LandmarkId> LandmarkSparsificationSchemeVoxel::getSelection(const LandmarkMap& landmarks, const KeyframeMap& keyframes) const {
    std::set<LandmarkId> out;
    for (const auto& el : getCategorizedSelection(landmarks, keyframes)) out.insert(el.first);
    return out;
}

std::map<LandmarkId, LandmarkCategorizatonInterface::Category> LandmarkSparsificationSchemeVoxel::getCategorizedSelection(
    const LandmarkMap& lms, const KeyframeMap& keyframes) const {
    std::map<LandmarkId, Category> out;
    if (keyframes.empty()) return out;
    const auto newest = std::max_element(keyframes.cbegin(), keyframes.cend(), [](const auto& a, const auto& b) {
        return a.second->timestamp_ < b.second->timestamp_;
    });
    const EigenPose cur = newest->second->getEigenPose();
    // 1. + 2. landmarks in the newest keyframe's frame, labelled by position in id order (32-bit labels, ids may be wider)
    std::vector<LandmarkId> lut;
    std::vector<LabelledPoint> cloud;
    for (const auto& id_lm : lms) {
        const Eigen::Vector3d p = cur * Eigen::Vector3d(id_lm.second->pos[0], id_lm.second->pos[1], id_lm.second->pos[2]);
        const LabelledPoint q{float(p[0]), float(p[1]), float(p[2]), uint32_t(lut.size())};
        lut.push_back(id_lm.first);
        if (std::isfinite(q.z) && q.z >= -20.f && q.z <= 100.f) cloud.push_back(q);  // PassThrough("z", -20, 100)
    }
    // keyframe positions (origin frame) seen from the newest keyframe, in id order: the path of filterPipe
    std::vector<Eigen::Vector3d> path;
    for (const auto& kf : keyframes) path.push_back(cur * kf.second->getEigenPose().inverse().translation());
    // 3. far bin
    std::vector<LabelledPoint> inside, near_pts;
    std::set<uint32_t> labels_far, labels_middle;
    filter_pipe(cloud, path, params_.roi_far_xyz[0], inside, labels_far);
    // 4. one point per voxel, 5. middle bin
    const std::vector<LabelledPoint> voxels = voxel_grid(inside, params_.voxel_size_xyz);
    filter_pipe(voxels, path, params_.roi_middle_xyz[0], near_pts, labels_middle);
    // 6. rank inside the bins
    std::vector<LandmarkId> ids_near, ids_middle, ids_far;
    for (const auto& p : near_pts) ids_near.push_back(lut.at(p.label));
    for (const auto& l : labels_middle) ids_middle.push_back(lut.at(l));
    for (const auto& l : labels_far) ids_far.push_back(lut.at(l));
    std::map<LandmarkId, unsigned int> seen;  // keyframes observing each far landmark (chooseFarLmIds)
    for (const auto& id : ids_far) {
        unsigned int n = 0;
        for (const auto& kf : keyframes) n += kf.second->hasMeasurement(id) ? 1u : 0u;
        seen[id] = n;
    }
    return rankBins(ids_near, landmark_helpers::calcFlow(ids_near, keyframes, false), ids_middle, ids_far, seen);
}

std::map<LandmarkId, LandmarkCategorizatonInterface::Category> LandmarkSparsificationSchemeVoxel::rankBins(
    const std::vector<LandmarkId>& ids_near, const std::map<LandmarkId, double>& flow, const std::vector<LandmarkId>& ids_middle,
    const std::vector<LandmarkId>& ids_far, const std::map<LandmarkId, unsigned int>& seen) const {
    std::map<LandmarkId, Category> out;
    for (const auto& id : landmark_helpers::chooseNearLmIds(params_.max_num_landmarks_near, ids_near, flow)) out[id] = Category::NearField;
    for (const auto& id : landmark_helpers::chooseMiddleLmIds(params_.max_num_landmarks_middle, ids_middle)) out[id] = Category::MiddleField;
    for (const auto& id : landmark_helpers::chooseFarLmIds(params_.max_num_landmarks_far, ids_far, seen)) out[id] = Category::FarField;
    return out;
}

// ---- add depth (landmark_selection_scheme_add_depth.cpp:16-75) ------------------------------------------------------------
std::set<LandmarkId> LandmarkSelectionSchemeAddDepth::getSelection(const LandmarkMap& landmarks, const KeyframeMap& keyframes) const {
    std::set<LandmarkId> out;
    std::vector<Keyframe::ConstPtr> oldest_first = keyframe_helpers::getSortedKeyframes(keyframes);
    std::reverse(oldest_first.begin(), oldest_first.end());
    for (const auto& el : params_.params_per_keyframe) {
        const FrameIndex ind = std::get<0>(el);
        const NumberLandmarks wanted = std::get<1>(el);
        const Comparator& eligible = std::get<2>(el);
        const Sorter& cost_of = std::get<3>(el);
        if (ind > int(oldest_first.size()) - 1) continue;
        const Keyframe& kf = *oldest_first[ind];
        std::vector<std::pair<LandmarkId, double>> cost;  // per eligible landmark of this keyframe: worst camera's value
        for (const auto& m : kf.measurements_) {
            const auto it = landmarks.find(m.first);
            if (it == landmarks.cend() || !eligible(it->second)) continue;
            const Eigen::Vector3d local = kf.getEigenPose() * Eigen::Vector3d(it->second->pos.data());
            double worst = -std::numeric_limits<double>::max();
            for (const auto& cam_meas : m.second) worst = std::max(worst, double(cost_of(cam_meas.second, local)));
            cost.emplace_back(m.first, worst);
        }
        const int n = std::min(wanted, int(cost.size()));
        std::partial_sort(cost.begin(), cost.begin() + n, cost.end(), [](const auto& a, const auto& b) { return a.second < b.second; });
        for (int i = 0; i < n; ++i) out.insert(cost[i].first);
    }
    return out;
}

// ---- the selector (landmark_selector.hpp:79-253) -----------------------------------------------------------------------------
std::set<LandmarkId> LandmarkSelector::runScheme(const LandmarkSchemeBase& scheme, const std::map<LandmarkId, Landmark::ConstPtr>& lms,
                                                 const std::map<KeyframeId, Keyframe::ConstPtr>& kfs) {
    const auto* categorizer = dynamic_cast<const LandmarkCategorizatonInterface*>(&scheme);
    if (!categorizer) return scheme.getSelection(lms, kfs);
    landmark_categories_ = categorizer->getCategorizedSelection(lms, kfs);  // one categoriser exists: the last one wins
    std::set<LandmarkId> out;
    for (const auto& el : landmark_categories_) out.insert(el.first);
    return out;
}

void LandmarkSelector::clean(TimestampNSec oldest_ts) {
    for (auto it = last_time_seen_.begin(); it != last_time_seen_.end();) {
        if (it->second < oldest_ts) { unselected_lms_.erase(it->first); it = last_time_seen_.erase(it); }
        else ++it;
    }
}

const LandmarkSparsificationSchemeVoxel* LandmarkSelector::quantitiesChainVoxel() const {
    if (rejection_schemes_.size() != 1 || sparsification_schemes_.size() != 1) return nullptr;
    if (!dynamic_cast<const LandmarkRejectionSchemeCheirality*>(rejection_schemes_[0].get())) return nullptr;
    return dynamic_cast<const LandmarkSparsificationSchemeVoxel*>(sparsification_schemes_[0].get());
}

std::set<LandmarkId> LandmarkSelector::select(const std::map<LandmarkId, Landmark::ConstPtr>& landmarks,
                                              const std::map<KeyframeId, Keyframe::ConstPtr>& kfs) {
    return selectImpl(landmarks, kfs, nullptr);
}

std::set<LandmarkId> LandmarkSelector::select(const std::map<LandmarkId, Landmark::ConstPtr>& landmarks,
                                              const std::map<KeyframeId, Keyframe::ConstPtr>& kfs, const ChainQuantities& q) {
    return selectImpl(landmarks, kfs, &q);
}

std::set<LandmarkId> LandmarkSelector::selectImpl(const std::map<LandmarkId, Landmark::ConstPtr>& landmarks,
                                                  const std::map<KeyframeId, Keyframe::ConstPtr>& kfs, const ChainQuantities* q) {
    auto pick = [](const std::map<LandmarkId, Landmark::ConstPtr>& src, const std::set<LandmarkId>& ids,
                   std::map<LandmarkId, Landmark::ConstPtr>& dst) {  // addToMap: ids a scheme names but src lacks are skipped
        for (const auto& id : ids) { auto it = src.find(id); if (it != src.cend()) dst[id] = it->second; }
    };
    std::map<LandmarkId, Landmark::ConstPtr> non_rejected = landmarks;
    for (const auto& id : outlier_ids_) non_rejected.erase(id);
    const LandmarkSparsificationSchemeVoxel* voxel = q ? quantitiesChainVoxel() : nullptr;
    if (q) {  // the cheirality scheme's verdicts
        if (!voxel) throw std::invalid_argument("LandmarkSelector::select: the chain is not cheirality + voxel (+ selection schemes)");
        const size_t n = q->candidates.size();
        if (n != non_rejected.size() || q->cheiral.size() != n || q->bin.size() != n || q->flow.size() != n || q->seen.size() != n ||
            q->near_order.size() > n)
            throw std::invalid_argument("LandmarkSelector::select: the quantities do not cover the candidates");
        size_t c = 0;
        for (auto it = non_rejected.begin(); it != non_rejected.end(); ++c) {
            if (it->first != q->candidates[c]) throw std::invalid_argument("LandmarkSelector::select: candidates differ from the landmarks");
            it = q->cheiral[c] ? std::next(it) : non_rejected.erase(it);
        }
    } else {
        for (const auto& scheme : rejection_schemes_) {
            const auto cur = runScheme(*scheme, non_rejected, kfs);
            non_rejected.clear();
            pick(landmarks, cur, non_rejected);
        }
    }
    std::map<LandmarkId, Landmark::ConstPtr> selected;
    for (const auto& scheme : selection_schemes_) pick(non_rejected, runScheme(*scheme, non_rejected, kfs), selected);
    std::map<LandmarkId, Landmark::ConstPtr> sparsified = non_rejected;
    if (q) {  // the voxel scheme's ranking over the bins the quantities describe (getCategorizedSelection's step 6)
        std::vector<LandmarkId> ids_near, ids_middle, ids_far;
        std::map<LandmarkId, double> flow;
        std::map<LandmarkId, unsigned int> seen;
        for (const int32_t c : q->near_order) {
            ids_near.push_back(q->candidates.at(c));
            if (!std::isnan(q->flow[c])) flow[q->candidates[c]] = q->flow[c];
        }
        for (size_t c = 0; c < q->candidates.size(); ++c) {
            if (q->bin[c] == 1) ids_middle.push_back(q->candidates[c]);
            if (q->bin[c] == 2) { ids_far.push_back(q->candidates[c]); seen[q->candidates[c]] = (unsigned int)q->seen[c]; }
        }
        landmark_categories_ = voxel->rankBins(ids_near, flow, ids_middle, ids_far, seen);
        sparsified.clear();
        std::set<LandmarkId> cur;
        for (const auto& el : landmark_categories_) cur.insert(el.first);
        pick(non_rejected, cur, sparsified);
    } else {
        for (const auto& scheme : sparsification_schemes_) {
            const auto cur = runScheme(*scheme, sparsified, kfs);
            sparsified.clear();
            pick(non_rejected, cur, sparsified);
        }
    }
    for (const auto& el : selected) sparsified[el.first] = el.second;
    std::set<LandmarkId> selection;
    for (const auto& el : sparsified) selection.insert(el.first);
    // age the landmarks that were not taken; the reference dereferences max_element of an empty map here (:234-237)
    TimestampNSec cur_ts = 0;
    for (const auto& kf : kfs) cur_ts = std::max(cur_ts, kf.second->timestamp_);
    for (const auto& lm : landmarks)
        if (!selection.count(lm.first)) markUnselected(lm.first, cur_ts);
    const TimestampNSec ten = convert(TimestampSec(10.));
    clean(cur_ts > ten ? cur_ts - ten : 0);  // the reference's unsigned subtraction wraps for time stamps < 10 s (test scenes)
    last_selected_lms_ = selection;
    return selection;
}

}  // namespace keyframe_bundle_adjustment
