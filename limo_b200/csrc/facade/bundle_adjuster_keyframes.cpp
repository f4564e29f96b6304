// bundle_adjuster_keyframes.cpp -- the replacement translation unit for limo's
// keyframe_bundle_adjustment/src/bundle_adjuster_keyframes.cpp (the other sources of the facade: definitions.cpp,
// keyframe.cpp, landmark_selection.cpp): window bookkeeping on the host exactly as the reference does it, the solve
// through the C ABI (kba_b200.h).
#include "keyframe_bundle_adjustment/bundle_adjuster_keyframes.hpp"

#include <algorithm>
#include <array>
#include <cmath>
#include <iterator>
#include <sstream>
#include <stdexcept>

#include "kba_b200.h"

namespace keyframe_bundle_adjustment {

// ---- triangulation ---------------------------------------------------------------------------------------------------------
Eigen::Vector3d triangulate_rays(const std::vector<std::pair<EigenPose, Eigen::Vector3d>>& poses_rays) {
    Eigen::Matrix3d sum = Eigen::Matrix3d::Zero();
    Eigen::Vector3d rhs = Eigen::Vector3d::Zero();
    for (const auto& p_r : poses_rays) {
        const Eigen::Vector3d r = p_r.first.rotation() * p_r.second;
        const Eigen::Matrix3d cur = Eigen::Matrix3d::Identity() - r * r.transpose();
        sum += cur;
        rhs += cur * p_r.first.translation();
    }
    return sum.inverse() * rhs;  // the reference solves with a Jacobi SVD; identical for >= 2 non-parallel rays
}

// ---- exceptions --------------------------------------------------------------------------------------------------------------
BundleAdjusterKeyframes::NotEnoughKeyframesException::NotEnoughKeyframesException(size_t is, size_t should)
        : num_is(is), num_should_be(should) {
    std::stringstream ss;
    ss << "Not enough keyframes available in bundle_adjuster_keyframes. Should be " << num_should_be << " is " << num_is;
    msg = ss.str();
}
BundleAdjusterKeyframes::KeyframeNotFoundException::KeyframeNotFoundException(TimestampNSec timestamp) : ts_(timestamp) {
    std::stringstream ss;
    ss << "keyframe corresponding to timestamp " << ts_ << " nano seconds not found";
    msg = ss.str();
}

// ---- the adjuster ------------------------------------------------------------------------------------------------------------
BundleAdjusterKeyframes::BundleAdjusterKeyframes() : solver_time_sec(0.2) {
    landmark_selector_ = std::make_unique<LandmarkSelector>();
    landmark_selector_->addScheme(LandmarkRejectionSchemeCheirality::create());  // cpp:116-118
}
BundleAdjusterKeyframes::~BundleAdjusterKeyframes() {
    if (track_) kba_track_destroy(track_);
    if (handle_) kba_destroy(handle_);
}

void BundleAdjusterKeyframes::push(const std::vector<Keyframe>& kfs) { for (const auto& kf : kfs) push(kf); }

void BundleAdjusterKeyframes::push(const Keyframe& kf) {  // cpp:289-329
    keyframes_[kf.timestamp_] = std::make_shared<Keyframe>(kf);
    active_keyframe_ids_.insert(kf.timestamp_);
    for (const auto& m : kf.measurements_) {
        if (landmarks_.find(m.first) == landmarks_.cend()) {
            bool has_depth = false;
            for (const auto& cam_meas : m.second) if (cam_meas.second.d >= 0) has_depth = true;  // containsDepth, cpp:37-48
            v3 p;
            const bool success = has_depth ? calculateLandmark(kf, m.first, p) : calculateLandmark(m.first, p);
            if (!success) continue;
            landmarks_.insert(std::make_pair(m.first, std::make_shared<Landmark>(p, has_depth)));
            new_landmarks_.insert(m.first);
        }
        active_landmark_ids_.insert(m.first);
    }
    // the device-resident store gets the keyframe lazily, at the next solve() (trackPush): callers may still edit the stored
    // copy before (mono_lidar.cpp sets the pose prior after push)
}

bool BundleAdjusterKeyframes::calculateLandmark(const Keyframe& kf, const LandmarkId& lId, v3& posAbs) {  // cpp:332-355
    for (const auto& m : kf.measurements_.at(lId)) {
        if (m.second.d < 0) continue;
        const auto cam = kf.cameras_.at(m.first);
        const double z = static_cast<double>(m.second.d);
        const double x = (static_cast<double>(m.second.u) - cam->principal_point[0]) * z / cam->focal_length;
        const double y = (static_cast<double>(m.second.v) - cam->principal_point[1]) * z / cam->focal_length;
        posAbs = (cam->getEigenPose() * kf.getEigenPose()).inverse() * v3(x, y, z);
        return true;
    }
    return false;
}

bool BundleAdjusterKeyframes::calculateLandmark(const LandmarkId& lId, v3& posAbs) {  // cpp:125-159, 358-382
    std::vector<std::pair<EigenPose, v3>> poses_rays;
    for (const auto& id : active_keyframe_ids_) {
        const Keyframe& kf = *keyframes_.at(id);
        for (const auto& id_cam : kf.cameras_) {
            if (!kf.hasMeasurement(lId, id_cam.first)) continue;
            const Measurement& m = kf.getMeasurement(lId, id_cam.first);
            const v3 ray = (id_cam.second->intrin_inv * v3(static_cast<double>(m.u), static_cast<double>(m.v), 1.)).normalized();
            poses_rays.emplace_back((id_cam.second->getEigenPose() * kf.getEigenPose()).inverse(), ray);
        }
    }
    if (poses_rays.size() < 2) return false;
    posAbs = triangulate_rays(poses_rays);
    return true;
}

void BundleAdjusterKeyframes::updateLabels(const Tracklets& t, double shrubbery_weight) {  // cpp:388-431
    std::set<LandmarkId> outlier_ids;
    for (const auto& id : landmark_selector_->getOutliers())
        if (active_landmark_ids_.count(id)) outlier_ids.insert(id);
    for (const auto& track : t.tracks)
        if (track.is_outlier || labels_["outliers"].count(track.label)) outlier_ids.insert(track.id);
    landmark_selector_->clearOutliers();
    landmark_selector_->setOutlier(outlier_ids);
    for (const auto& track : t.tracks) {
        if (!active_landmark_ids_.count(track.id)) continue;
        if (labels_["shrubbery"].count(track.label)) { landmarks_.at(track.id)->weight = shrubbery_weight; dirty_weights_.insert(track.id); }
        landmarks_.at(track.id)->is_ground_plane = labels_["ground"].count(track.label) > 0;
    }
}

std::map<LandmarkId, Landmark::ConstPtr> BundleAdjusterKeyframes::filterLandmarksById(const std::set<LandmarkId>& ids) const {
    std::map<LandmarkId, Landmark::ConstPtr> out;
    for (const auto& id : ids) { auto it = landmarks_.find(id); if (it != landmarks_.cend()) out[id] = it->second; }
    return out;
}
std::map<LandmarkId, Landmark::ConstPtr> BundleAdjusterKeyframes::getActiveLandmarkConstPtrs() const { return filterLandmarksById(active_landmark_ids_); }
std::map<LandmarkId, Landmark::ConstPtr> BundleAdjusterKeyframes::getSelectedLandmarkConstPtrs() const { return filterLandmarksById(selected_landmark_ids_); }
std::map<KeyframeId, Keyframe::Ptr> BundleAdjusterKeyframes::getActiveKeyframePtrs() const {
    std::map<KeyframeId, Keyframe::Ptr> out;
    for (const auto& id : active_keyframe_ids_) out[id] = keyframes_.at(id);
    return out;
}
std::map<KeyframeId, Keyframe::ConstPtr> BundleAdjusterKeyframes::getActiveKeyframeConstPtrs() const {
    std::map<KeyframeId, Keyframe::ConstPtr> out;
    for (const auto& id : active_keyframe_ids_) out[id] = keyframes_.at(id);
    return out;
}
std::vector<std::pair<KeyframeId, Keyframe::Ptr>> BundleAdjusterKeyframes::getSortedIdsWithActiveKeyframePtrs() const {
    std::vector<std::pair<KeyframeId, Keyframe::Ptr>> v;
    for (const auto& kf : getActiveKeyframePtrs()) v.push_back(kf);
    std::sort(v.begin(), v.end(), [](const auto& a, const auto& b) { return *(a.second) < *(b.second); });
    return v;
}
std::vector<Keyframe::Ptr> BundleAdjusterKeyframes::getSortedActiveKeyframePtrs() const {
    std::vector<Keyframe::Ptr> out;
    for (const auto& el : getSortedIdsWithActiveKeyframePtrs()) out.push_back(el.second);
    return out;
}

const Keyframe& BundleAdjusterKeyframes::getKeyframe(TimestampSec timestamp) const {  // cpp:989-1021
    if (keyframes_.size() == 0) throw NotEnoughKeyframesException(keyframes_.size(), 1);
    if (timestamp < 0.) {
        auto it = std::max_element(active_keyframe_ids_.cbegin(), active_keyframe_ids_.cend(), [&](const auto& a, const auto& b) {
            return keyframes_.at(a)->timestamp_ < keyframes_.at(b)->timestamp_;
        });
        return *keyframes_.at(*it);
    }
    const TimestampNSec ts_nsec = convert(timestamp);
    for (const auto& kf : keyframes_)
        if (kf.second->timestamp_ == ts_nsec) return *kf.second;
    throw KeyframeNotFoundException(ts_nsec);
}

void BundleAdjusterKeyframes::deactivateKeyframes(int min_num_connecting_landmarks, int min_size_optimization_window,
                                                  int max_size_optimization_window) {  // cpp:907-987
    auto sorted = getSortedIdsWithActiveKeyframePtrs();
    auto newest = sorted.back().second;
    int n = 0;
    for (auto it = sorted.crbegin(); it != sorted.crend(); ++it, ++n) {
        auto& cur = *it->second;
        if (n > max_size_optimization_window - 1) cur.is_active_ = false;
        else if (n < min_size_optimization_window - 1) cur.is_active_ = true;
        else {
            int common = 0;
            for (const auto& m : cur.measurements_) common += newest->measurements_.count(m.first) ? 1 : 0;
            cur.is_active_ = common > min_num_connecting_landmarks;
        }
        if (!cur.is_active_) active_keyframe_ids_.erase(it->first);
    }
    std::set<LandmarkId> new_active;
    for (const auto& id : active_keyframe_ids_)
        for (const auto& m : keyframes_.at(id)->measurements_)
            if (active_landmark_ids_.count(m.first)) new_active.insert(m.first);
    active_landmark_ids_ = new_active;
    auto rest = getSortedIdsWithActiveKeyframePtrs();
    rest[0].second->fixation_status_ = Keyframe::FixationStatus::Pose;
    rest[1].second->fixation_status_ = Keyframe::FixationStatus::Scale;
}

namespace {
// kba_options of solve() / adjustPoseOnly() (cpp:740-764, 864-869)
kba_options solve_options(const BundleAdjusterKeyframes::OutlierRejectionOptions& o, double solver_time_sec, bool motion_only,
                          size_t n_selected) {
    kba_options opt;
    kba_default_options(&opt);
    opt.depth_thres = o.depth_thres;
    opt.reprojection_thres = o.reprojection_thres;
    opt.depth_quantile = o.depth_quantile;
    opt.reprojection_quantile = o.reprojection_quantile;
    opt.num_rounds_option = o.num_iterations;
    opt.solver_time_sec = solver_time_sec;
    if (motion_only) {  // cpp:864-869
        opt.min_landmarks_for_trimming = 30;
        opt.num_trim_rounds = n_selected > 30 ? o.num_iterations : 0;
    }
    return opt;
}

// stands in for robust_optimization::Summary::FullReport (robust_solving.hpp:54-59)
std::string solve_report(const kba_result& r, const char* where) {
    static const char* term[] = {"CONVERGENCE", "NO_CONVERGENCE", "FAILURE"};
    std::stringstream ss;
    ss << "Merged summaries:\n";
    for (int i = 0; i < r.num_solves; ++i) {
        const kba_solve_summary& s = r.solves[i];
        ss << "--------------------------------------------------\nIteration No." << i << "\n"
           << "Residual blocks " << s.num_residual_blocks << ", landmarks " << s.num_landmarks << "; initial cost "
           << s.initial_cost << ", final cost " << s.final_cost << ", iterations " << s.num_iterations << " (successful "
           << s.num_successful_steps << "), termination " << term[s.termination < 3 ? s.termination : 2] << "\n";
    }
    if (r.status != KBA_OK)  // like a Ceres failure, not surfaced as an exception (reference: only text in the report)
        ss << "\nsolver did not finish (kba status " << r.status << "): the last accepted iterate was written back\n";
    ss << "\nDuration solveTrimmed=" << r.time_sec << " sec" << where << "\n";
    return ss.str();
}
}  // namespace

// SpeedRegularizationVector2 of adjustPoseOnly (cpp:835-853) on keyframe 0 of w, when the reference adds it
void BundleAdjusterKeyframes::speedPrior(const Keyframe& speed_kf, kba_window& w) const {
    if (active_keyframe_ids_.size() <= 2) return;
    auto sorted = getSortedActiveKeyframePtrs();
    const Keyframe& b0 = *sorted[sorted.size() - 1];
    const Keyframe& b1 = *sorted[sorted.size() - 2];
    const double rot_diff = calcQuaternionDiff(b0.pose_, b1.pose_);
    if (!(rot_diff < 0.03)) return;
    const double dt_cur = convert(speed_kf.timestamp_) - convert(b0.timestamp_);
    const double dt_before = convert(b0.timestamp_) - convert(b1.timestamp_);
    if (dt_cur <= 0. || dt_before <= 0.) throw std::runtime_error("In PoseRegularizationSpeed: invalid timestamps");
    const v3 v_before = (b0.getEigenPose() * b1.getEigenPose().inverse()).translation() / dt_before;
    const Pose T_ob = convert(b0.getEigenPose().inverse());
    w.speed_kf = 0; w.speed_weight = 1. * (1 - rot_diff / 0.03); w.speed_dt = dt_cur;
    for (int i = 0; i < 3; ++i) w.speed_v_before[i] = v_before[i];
    for (int i = 0; i < 7; ++i) w.speed_T_origin_before[i] = T_ob[i];
}

// Pack -> kba_solve_window -> scatter.  Replaces addActiveKeyframesToProblem / addKeyframeToProblem (cpp:498-627),
// addGroundPlaneResiduals (:517-562), the scale / plane regulariser set-up (:703-728, 769-818, 890-904) and
// robust_optimization::solveTrimmed (:765, :886).
std::string BundleAdjusterKeyframes::runWindow(const std::vector<Keyframe*>& kfs, const std::vector<LandmarkId>& lm_ids,
                                               bool motion_only, Keyframe* speed_kf) {
    ensureHandle();
    std::vector<double> kf_pose, kf_plane, cam_intr, cam_pose, lm_pos, lm_weight, gp_weight;
    std::vector<uint8_t> kf_fixed;
    std::vector<int32_t> lm_obs_ptr{0}, obs_kf, obs_cam, gp_lm, gp_kf;
    std::vector<float> obs_u, obs_v, obs_d;
    // Cameras are de-duplicated BY VALUE: the production node makes a new Camera object for every frame
    // (mono_lidar.cpp:112, mono_standalone.cpp:101), so pointer identity would give one "camera" per keyframe.
    using CamKey = std::array<double, 10>;  // focal length, principal point, pose_camera_vehicle
    auto cam_key = [](const Camera& c) {
        CamKey k{{c.focal_length, c.principal_point[0], c.principal_point[1]}};
        std::copy(c.pose_camera_vehicle.begin(), c.pose_camera_vehicle.end(), k.begin() + 3);
        return k;
    };
    std::map<CamKey, int> cam_index;
    for (const Keyframe* kf : kfs) {
        kf_pose.insert(kf_pose.end(), kf->pose_.begin(), kf->pose_.end());
        kf_fixed.push_back(!motion_only && kf->fixation_status_ == Keyframe::FixationStatus::Pose);  // cpp:198-219
        kf_plane.insert(kf_plane.end(), kf->local_ground_plane_.direction.begin(), kf->local_ground_plane_.direction.end());
        kf_plane.push_back(kf->local_ground_plane_.distance);
        for (const auto& c : kf->cameras_)
            if (cam_index.emplace(cam_key(*c.second), int(cam_index.size())).second) {
                cam_intr.insert(cam_intr.end(), {c.second->focal_length, c.second->principal_point[0], c.second->principal_point[1]});
                cam_pose.insert(cam_pose.end(), c.second->pose_camera_vehicle.begin(), c.second->pose_camera_vehicle.end());
            }
    }
    int n_depth = 0;
    for (const auto lm_id : lm_ids) {
        const Landmark& lm = *landmarks_.at(lm_id);
        lm_pos.insert(lm_pos.end(), lm.pos.begin(), lm.pos.end());
        lm_weight.push_back(lm.weight);
        for (size_t k = 0; k < kfs.size(); ++k) {
            auto it = kfs[k]->measurements_.find(lm_id);
            if (it == kfs[k]->measurements_.end()) continue;
            for (const auto& cm : it->second) {
                obs_kf.push_back(int32_t(k));
                obs_cam.push_back(cam_index.at(cam_key(*kfs[k]->cameras_.at(cm.first))));
                obs_u.push_back(cm.second.u); obs_v.push_back(cm.second.v); obs_d.push_back(cm.second.d);
                n_depth += cm.second.d > 0.0f;
            }
        }
        lm_obs_ptr.push_back(int32_t(obs_kf.size()));
    }
    kba_window w{};
    if (!motion_only) {
        for (size_t j = 0; j < lm_ids.size(); ++j) {  // addGroundPlaneResiduals(10.), cpp:517-562
            const Landmark& lm = *landmarks_.at(lm_ids[j]);
            if (!lm.is_ground_plane) continue;
            double min_dist = std::numeric_limits<double>::max();
            int best = -1;
            for (size_t k = 0; k < kfs.size(); ++k) {
                if (kfs[k]->local_ground_plane_.distance < -10.) continue;
                const double dist = (kfs[k]->getEigenPose() * v3(lm.pos.data())).norm();
                if (dist < min_dist) { min_dist = dist; best = int(k); }
            }
            if (best < 0 || !(min_dist < 25.)) continue;
            gp_lm.push_back(int32_t(j)); gp_kf.push_back(best); gp_weight.push_back(10. * (1. - min_dist / 25.));
        }
        const int n_gp = int(gp_lm.size());
        double scale_weight = 0.;  // cpp:703-716
        if (n_depth > 10 || n_gp > 10) { if (n_gp < 30) scale_weight = 1000. / (double(n_depth) + double(n_gp)); }
        else scale_weight = 1000.;
        if (scale_weight > 0 && kfs.size() > 1) {
            w.scale_kf0 = 0; w.scale_kf1 = 1; w.scale_weight = scale_weight;
            w.scale_value = (kfs[1]->getEigenPose() * kfs[0]->getEigenPose().inverse()).translation().norm();
        }
        if (n_gp > 0) w.plane_reg_weight = 10.;  // cpp:717-719
        w.plane_dist_fixed = n_depth < 10;       // cpp:722-728
    } else if (speed_kf) {
        speedPrior(*speed_kf, w);
    }
    w.landmarks_fixed = motion_only;
    w.n_kf = int(kfs.size()); w.n_cam = int(cam_index.size()); w.n_lm = int(lm_ids.size()); w.n_obs = int(obs_kf.size());
    w.n_gp = int(gp_lm.size());
    w.kf_pose = kf_pose.data(); w.kf_fixed = kf_fixed.data(); w.kf_plane = kf_plane.data();
    w.cam_intr = cam_intr.data(); w.cam_pose = cam_pose.data();
    w.lm_pos = lm_pos.data(); w.lm_weight = lm_weight.data(); w.lm_obs_ptr = lm_obs_ptr.data();
    w.obs_kf = obs_kf.data(); w.obs_cam = obs_cam.data(); w.obs_u = obs_u.data(); w.obs_v = obs_v.data(); w.obs_d = obs_d.data();
    w.gp_lm = gp_lm.data(); w.gp_kf = gp_kf.data(); w.gp_weight = gp_weight.data();

    const kba_options opt = solve_options(outlier_rejection_options_, solver_time_sec, motion_only, selected_landmark_ids_.size());
    std::vector<double> out_pose(kf_pose.size()), out_plane(kf_plane.size()), out_lm(lm_pos.size() + 3);
    kba_result r{};
    r.kf_pose = out_pose.data(); r.kf_plane = out_plane.data(); r.lm_pos = out_lm.data();
    if (kba_solve_window(handle_, &w, &opt, &r) != KBA_OK) throw std::runtime_error(std::string("kba_b200: ") + kba_last_error());
    // what the rebuild path uploads: the window's arrays as passed (kba_batch_transfer_bytes reports the same for a batch)
    last_solve_h2d_ = (long long)(kf_pose.size() + kf_plane.size() + lm_pos.size() + lm_weight.size() + cam_intr.size() + cam_pose.size()) * 8 +
                      (long long)(lm_obs_ptr.size() + 2 * obs_kf.size()) * 4 + (long long)obs_u.size() * 12 + (long long)kf_fixed.size();

    for (size_t k = 0; k < kfs.size(); ++k) {  // the reference optimises in place (cpp:554-557, 592-593)
        std::copy_n(out_pose.begin() + 7 * k, 7, kfs[k]->pose_.begin());
        if (!motion_only && w.n_gp > 0) {
            std::copy_n(out_plane.begin() + 4 * k, 3, kfs[k]->local_ground_plane_.direction.begin());
            kfs[k]->local_ground_plane_.distance = out_plane[4 * k + 3];
        }
    }
    if (!motion_only)
        for (size_t j = 0; j < lm_ids.size(); ++j) {
            std::copy_n(out_lm.begin() + 3 * j, 3, landmarks_.at(lm_ids[j])->pos.begin());
            if (track_) dirty_positions_.insert(lm_ids[j]);  // the store still holds the old position: flushLandmarks()
        }

    return solve_report(r, "");
}

namespace {
std::array<double, 10> camera_value(const Camera& c);  // below, with the other helpers of the persistent window
}  // namespace

std::string BundleAdjusterKeyframes::solve() {  // cpp:629-767
    if (keyframes_.size() < 3) throw NotEnoughKeyframesException(keyframes_.size(), 3);
    std::vector<Keyframe*> kfs;
    for (const auto& id : active_keyframe_ids_) kfs.push_back(keyframes_.at(id).get());
    last_select_h2d_ = 0;
    const bool synced = selectOnDevice(kfs);
    if (!synced) selected_landmark_ids_ = landmark_selector_->select(getActiveLandmarkConstPtrs(), getActiveKeyframeConstPtrs());
    std::vector<LandmarkId> lm_ids(selected_landmark_ids_.begin(), selected_landmark_ids_.end());
    std::string report;
    if (persistent_window_ && !track_failed_ && solveTracked(kfs, lm_ids, report, synced)) return report;
    return runWindow(kfs, lm_ids, false, nullptr);
}

// solve()'s landmark selection with the store computing the chain's per-landmark quantities (kba_track_select_landmarks) and the
// selector ranking them: the same selection as the host select(), without a host pass over the window's measurements.  Only for
// a chain the quantities stand for (LandmarkSelector::quantitiesChainVoxel), every active keyframe in the store, every candidate
// with a slot, and camera ids that map onto the store's camera indices in the same order (flow is kept per camera).  true: the
// selection is made and the store holds the active keyframes' current state; false: the caller selects on the host.
bool BundleAdjusterKeyframes::selectOnDevice(const std::vector<Keyframe*>& kfs) {
    last_select_on_device_ = false;
    if (!device_selection_ || !persistent_window_ || track_failed_ || kfs.empty()) return false;
    const LandmarkSparsificationSchemeVoxel* voxel = landmark_selector_->quantitiesChainVoxel();
    if (!voxel) return false;
    for (const Keyframe* kf : kfs)
        if (!kf->is_active_) return false;  // the host's cheirality test skips inactive keyframes
    if (!trackSync(kfs)) return false;
    std::map<CameraId, int> cam_index;
    for (const Keyframe* kf : kfs)
        for (const auto& c : kf->cameras_) {
            const int idx = int(std::find(track_cams_.begin(), track_cams_.end(), camera_value(*c.second)) - track_cams_.begin());
            const auto ins = cam_index.emplace(c.first, idx);
            if (!ins.second && ins.first->second != idx) return false;
        }
    int prev = -1;
    for (const auto& el : cam_index) {
        if (el.second <= prev) return false;
        prev = el.second;
    }
    LandmarkSelector::ChainQuantities q;
    std::vector<int32_t> kf_slots, lm_slots;
    for (const Keyframe* kf : kfs) kf_slots.push_back(kf_slot_.at(kf->timestamp_));
    const auto landmarks = getActiveLandmarkConstPtrs();
    const auto& outliers = landmark_selector_->getOutliers();
    for (const auto& el : landmarks) {
        if (outliers.count(el.first)) continue;
        const auto it = lm_slot_.find(el.first);
        if (it == lm_slot_.end()) return false;
        q.candidates.push_back(el.first);
        lm_slots.push_back(it->second);
    }
    const size_t n = q.candidates.size();
    q.cheiral.resize(n); q.bin.resize(n); q.near_order.resize(n); q.flow.resize(n); q.seen.resize(n);
    int32_t n_near = 0;
    const auto& vp = voxel->params_;
    kba_select_params p{{vp.voxel_size_xyz[0], vp.voxel_size_xyz[1], vp.voxel_size_xyz[2]}, vp.roi_far_xyz[0], vp.roi_middle_xyz[0]};
    kba_select_out o{q.cheiral.data(), q.bin.data(), q.near_order.data(), &n_near, q.flow.data(), q.seen.data()};
    if (kba_track_select_landmarks(track_, int(kf_slots.size()), kf_slots.data(), int(n), lm_slots.data(), &p, &o) != KBA_OK)
        throw std::runtime_error(std::string("kba_b200: ") + kba_last_error());
    q.near_order.resize(size_t(n_near));
    int64_t h2d = 0;
    kba_track_transfer_bytes(track_, &h2d, nullptr, nullptr);
    last_select_h2d_ = (long long)h2d;
    selected_landmark_ids_ = landmark_selector_->select(landmarks, getActiveKeyframeConstPtrs(), q);
    last_select_on_device_ = true;
    return true;
}

// ---- persistent device-resident window ---------------------------------------------------------------------------------------
bool BundleAdjusterKeyframes::ensureHandle() {
    if (!handle_ && kba_create(&handle_, 0) != KBA_OK) throw std::runtime_error(std::string("kba_b200: ") + kba_last_error());
    return true;
}

namespace {
std::array<double, 10> camera_value(const Camera& c) {
    std::array<double, 10> k{{c.focal_length, c.principal_point[0], c.principal_point[1]}};
    std::copy(c.pose_camera_vehicle.begin(), c.pose_camera_vehicle.end(), k.begin() + 3);
    return k;
}
constexpr int kTrackWinKeyframes = 30, kTrackWinLandmarks = 16384, kTrackWinObservations = 1 << 18;
}  // namespace

// the keyframe's measurements go to the device ONCE (landmark slot, camera, u, v, d in measurements_ order: landmark id, then
// camera id -- the order addKeyframeToProblem enumerates, cpp:564-627); false: this keyframe cannot live in the store
bool BundleAdjusterKeyframes::trackPush(const Keyframe& kf) {
    ensureHandle();
    if (!track_) {  // created from the cameras of the first keyframe that reaches it
        std::vector<double> intr, pose;
        for (const auto& c : kf.cameras_) {
            const auto v = camera_value(*c.second);
            if (std::find(track_cams_.begin(), track_cams_.end(), v) != track_cams_.end()) continue;
            track_cams_.push_back(v);
            intr.insert(intr.end(), v.begin(), v.begin() + 3);
            pose.insert(pose.end(), v.begin() + 3, v.end());
        }
        // ground capacity for every selected landmark: the candidate lists are 4 B per landmark.  Reduced rows for every window
        // up to kTrackWinKeyframes with plane blocks: windows beyond 184 rows (19-30 keyframes with ground points, limo's default of
        // 20 among them) take the track's large-window solver instead of the rebuild path
        kba_track_caps caps{track_keyframes_, track_landmarks_, track_measurements_, kTrackWinKeyframes, kTrackWinLandmarks, kTrackWinObservations,
                            kTrackWinLandmarks, 10 * kTrackWinKeyframes + 1};
        if (kba_track_create(handle_, &caps, int(track_cams_.size()), intr.data(), pose.data(), &track_) != KBA_OK) return false;
        for (int i = track_keyframes_ - 1; i >= 0; --i) free_kf_slots_.push_back(i);
    }
    std::map<CameraId, int> cam_of;
    for (const auto& c : kf.cameras_) {
        const auto it = std::find(track_cams_.begin(), track_cams_.end(), camera_value(*c.second));
        if (it == track_cams_.end()) return false;  // a camera the store does not know
        cam_of[c.first] = int(it - track_cams_.begin());
    }
    if (free_kf_slots_.empty()) {  // reclaim the slots of the oldest keyframes that are no longer active
        dropInactiveKeyframes(32);
        if (free_kf_slots_.empty()) return false;
    }
    // before any slot is handed to kf: kf is not in the arena yet, so a slot given to it here would count as free
    if (!reclaimLandmarkSlots(kf)) return false;
    std::vector<int32_t> lm, cam;
    std::vector<float> u, v, d;
    for (const auto& m : kf.measurements_) {
        auto it = lm_slot_.find(m.first);
        if (it == lm_slot_.end()) {
            int s = int(slot_lm_.size());  // dense from 0 until the first reclaim, then from the free list first
            if (!free_lm_slots_.empty()) {
                s = free_lm_slots_.back();
                free_lm_slots_.pop_back();
                slot_lm_[size_t(s)] = m.first;
            } else {
                if (s >= track_landmarks_) return false;
                slot_lm_.push_back(m.first);
            }
            it = lm_slot_.emplace(m.first, s).first;
            // a landmark measured again after its slot was reclaimed: its host state goes up at the flush
            if (landmarks_.count(m.first) && !new_landmarks_.count(m.first)) restore_landmarks_.insert(m.first);
        }
        for (const auto& cm : m.second) {
            lm.push_back(it->second); cam.push_back(cam_of.at(cm.first));
            u.push_back(cm.second.u); v.push_back(cm.second.v); d.push_back(cm.second.d);
        }
    }
    const int slot = free_kf_slots_.back();
    double plane[4] = {kf.local_ground_plane_.direction[0], kf.local_ground_plane_.direction[1], kf.local_ground_plane_.direction[2], kf.local_ground_plane_.distance};
    if (kba_track_push_keyframe(track_, slot, kf.pose_.data(), plane, int(lm.size()), lm.data(), cam.data(), u.data(), v.data(), d.data()) != KBA_OK) return false;
    free_kf_slots_.pop_back();
    kf_slot_[kf.timestamp_] = slot;
    return true;
}

void BundleAdjusterKeyframes::set_track_capacity(int max_keyframes, int max_landmarks, int max_measurements) {
    if (track_) throw std::logic_error("set_track_capacity: the device-resident store exists already");
    track_keyframes_ = max_keyframes; track_landmarks_ = max_landmarks; track_measurements_ = max_measurements;
}

// the stored keyframes that are no longer active leave the store, oldest first, until max_free_kf_slots keyframe slots are free
void BundleAdjusterKeyframes::dropInactiveKeyframes(size_t max_free_kf_slots) {
    for (auto it = kf_slot_.begin(); it != kf_slot_.end() && free_kf_slots_.size() < max_free_kf_slots;) {
        if (active_keyframe_ids_.count(it->first)) { ++it; continue; }
        kba_track_drop_keyframe(track_, it->second);
        free_kf_slots_.push_back(it->second);
        it = kf_slot_.erase(it);
    }
}

// Landmark slots for the landmarks of kf that have none.  When the free list and the unused capacity cannot cover them, the
// slots no stored keyframe measures (kba_track_reclaim_landmarks) go on the free list: first as the store stands, then after the
// stored keyframes that are no longer active have left it.  A landmark whose slot is reclaimed keeps its host state in landmarks_
// and gets a slot again when a keyframe that measures it is pushed (restore_landmarks_).  false: still too few slots.
bool BundleAdjusterKeyframes::reclaimLandmarkSlots(const Keyframe& kf) {
    size_t need = 0;
    for (const auto& m : kf.measurements_) need += lm_slot_.count(m.first) == 0;
    auto room = [&] { return free_lm_slots_.size() + size_t(track_landmarks_) - slot_lm_.size(); };
    for (int pass = 0; pass < 2 && need > room(); ++pass) {
        if (pass == 1) dropInactiveKeyframes(size_t(track_keyframes_));
        const int hi = int(slot_lm_.size());
        std::vector<int32_t> free_slot(size_t(hi) + 1);
        kba_reclaim_request q{0, hi};
        kba_reclaim_out o{};
        o.free_slot = free_slot.data();
        if (kba_track_reclaim_landmarks(track_, &q, &o) != KBA_OK) return false;
        for (int i = o.n_free - 1; i >= 0; --i) {  // descending onto the free list: the lowest slot is handed out first
            const int s = free_slot[size_t(i)];
            const LandmarkId id = slot_lm_[size_t(s)];
            const auto it = lm_slot_.find(id);
            if (it == lm_slot_.end() || it->second != s) continue;  // on the free list already
            if (kf.measurements_.count(id)) continue;               // kf measures it: it keeps its slot
            lm_slot_.erase(it);
            restore_landmarks_.erase(id);
            free_lm_slots_.push_back(s);
        }
    }
    return need <= room();
}

// solve() on the device-resident window: only the selection goes up.  false: not possible for this window (caller rebuilds).
// The store brought to the host's state for the active keyframes kfs: every one pushed, their poses / planes, new landmarks,
// positions and weights.  false: not possible (track_failed_ is set).
bool BundleAdjusterKeyframes::trackSync(const std::vector<Keyframe*>& kfs) {
    for (const Keyframe* kf : kfs)
        if (!kf_slot_.count(kf->timestamp_) && !trackPush(*kf)) { track_failed_ = true; return false; }
    std::vector<int32_t> kf_slots;
    std::vector<double> poses, planes;
    for (const Keyframe* kf : kfs) {
        kf_slots.push_back(kf_slot_.at(kf->timestamp_));
        poses.insert(poses.end(), kf->pose_.begin(), kf->pose_.end());
        planes.insert(planes.end(), kf->local_ground_plane_.direction.begin(), kf->local_ground_plane_.direction.end());
        planes.push_back(kf->local_ground_plane_.distance);
    }
    if (kba_track_set_keyframe_poses(track_, int(kfs.size()), kf_slots.data(), poses.data(), planes.data()) != KBA_OK) { track_failed_ = true; return false; }
    if (!flushLandmarks()) { track_failed_ = true; return false; }
    return true;
}

// the lists of a solve or evaluation of the window kfs / lm_ids on the track (sel points into q's candidate list)
struct BundleAdjusterKeyframes::TrackRequest {
    std::vector<int32_t> kf_slots, lm_slots, gp_cand;
    std::vector<uint8_t> fixed;
    kba_window sel{};
};

// false: a selected landmark was never measured by a stored keyframe (no slot)
bool BundleAdjusterKeyframes::trackRequest(const std::vector<Keyframe*>& kfs, const std::vector<LandmarkId>& lm_ids, TrackRequest& q) const {
    const int n_kf = int(kfs.size()), n_lm = int(lm_ids.size());
    for (const Keyframe* kf : kfs) {
        q.kf_slots.push_back(kf_slot_.at(kf->timestamp_));
        q.fixed.push_back(kf->fixation_status_ == Keyframe::FixationStatus::Pose);
    }
    for (const auto id : lm_ids) {
        auto it = lm_slot_.find(id);
        if (it == lm_slot_.end()) return false;
        q.lm_slots.push_back(it->second);
    }
    // addGroundPlaneResiduals (cpp:517-562) on the device: the selected ground-plane landmarks go up as candidates, the store's
    // poses, planes and positions decide which are attached to which keyframe
    for (int j = 0; j < n_lm; ++j)
        if (landmarks_.at(lm_ids[j])->is_ground_plane) q.gp_cand.push_back(j);
    kba_window& sel = q.sel;
    sel.n_kf = n_kf; sel.n_lm = n_lm;
    sel.n_gp = int(q.gp_cand.size()); sel.gp_lm = q.gp_cand.data();
    sel.plane_reg_weight = q.gp_cand.empty() ? 0. : -1.;  // -1: 10 iff a ground-plane residual is attached (cpp:717-719)
    sel.scale_kf0 = 0; sel.scale_kf1 = 1;
    sel.scale_weight = -1.;  // the reference's rule (cpp:703-716), evaluated on the device from the gathered window
    sel.scale_value = n_kf > 1 ? (kfs[1]->getEigenPose() * kfs[0]->getEigenPose().inverse()).translation().norm() : 0.;
    return true;
}

// synced: trackSync(kfs) already ran for this solve (the device-side selection needed the same state)
bool BundleAdjusterKeyframes::solveTracked(const std::vector<Keyframe*>& kfs, const std::vector<LandmarkId>& lm_ids, std::string& report,
                                           bool synced) {
    if (int(kfs.size()) > kTrackWinKeyframes || int(lm_ids.size()) > kTrackWinLandmarks) return false;
    // state the host may have changed since the last solve: poses / planes of the active keyframes, new landmarks, weights
    if (!synced && !trackSync(kfs)) return false;
    const int n_kf = int(kfs.size()), n_lm = int(lm_ids.size());
    TrackRequest q;
    if (!trackRequest(kfs, lm_ids, q)) return false;  // selected but never measured by a stored keyframe: let the rebuild path decide
    const std::vector<int32_t>& kf_slots = q.kf_slots, &lm_slots = q.lm_slots;
    const std::vector<uint8_t>& fixed = q.fixed;
    const kba_window& sel = q.sel;
    const kba_options opt = solve_options(outlier_rejection_options_, solver_time_sec, false, lm_ids.size());
    std::vector<double> out_pose(7 * size_t(n_kf)), out_plane(4 * size_t(n_kf)), out_lm(3 * size_t(n_lm) + 3);
    kba_result r{};
    r.kf_pose = out_pose.data(); r.kf_plane = out_plane.data(); r.lm_pos = out_lm.data();
    const int rc = kba_track_solve(track_, n_kf, kf_slots.data(), fixed.data(), n_lm, lm_slots.data(), &sel, &opt, &r);
    // e.g. more observations than the store's window capacity: rebuild
    if (rc == KBA_ERR_CAPACITY) return false;
    if (rc != KBA_OK) throw std::runtime_error(std::string("kba_b200: ") + kba_last_error());
    int64_t h2d = 0, d2h = 0, pushes = 0;
    kba_track_transfer_bytes(track_, &h2d, &d2h, &pushes);
    push_h2d_ = (long long)pushes;
    // the selection lists + the active keyframes' poses, and the lists of a device-side landmark selection
    last_solve_h2d_ = (long long)h2d + (long long)n_kf * (7 + 4) * 8 + last_select_h2d_;
    for (int k = 0; k < n_kf; ++k) {  // in place, as the reference (cpp:554-557); planes nothing was attached to come back unchanged
        std::copy_n(out_pose.begin() + 7 * k, 7, kfs[k]->pose_.begin());
        std::copy_n(out_plane.begin() + 4 * k, 3, kfs[k]->local_ground_plane_.direction.begin());
        kfs[k]->local_ground_plane_.distance = out_plane[4 * k + 3];
    }
    for (int j = 0; j < n_lm; ++j) std::copy_n(out_lm.begin() + 3 * j, 3, landmarks_.at(lm_ids[j])->pos.begin());
    report = solve_report(r, " (device-resident window)");
    return true;
}

void BundleAdjusterKeyframes::evaluateResiduals() {
    const char* who = "evaluateResiduals: ";
    if (!persistent_window_) throw std::runtime_error(std::string(who) + "the persistent window is off (set_persistent_window(false)); there is no host evaluation");
    if (track_failed_) throw std::runtime_error(std::string(who) + "the device-resident store failed (a keyframe or landmark it could not take)");
    if (!track_) throw std::runtime_error(std::string(who) + "no device-resident window yet: call solve() first");
    std::vector<Keyframe*> kfs;
    for (const auto& id : active_keyframe_ids_) kfs.push_back(keyframes_.at(id).get());
    std::vector<LandmarkId> lm_ids(selected_landmark_ids_.begin(), selected_landmark_ids_.end());
    if (kfs.size() < 3) throw std::runtime_error(std::string(who) + "fewer than 3 active keyframes");
    if (int(kfs.size()) > kTrackWinKeyframes || int(lm_ids.size()) > kTrackWinLandmarks)
        throw std::runtime_error(std::string(who) + "the window is larger than the device-resident store's window capacity");
    if (!trackSync(kfs)) throw std::runtime_error(std::string(who) + "the device-resident store failed while taking the current state");
    TrackRequest q;
    if (!trackRequest(kfs, lm_ids, q)) throw std::runtime_error(std::string(who) + "a selected landmark is not in the device-resident store");
    const kba_options opt = solve_options(outlier_rejection_options_, solver_time_sec, false, lm_ids.size());
    const size_t n_lm = lm_ids.size(), cap = size_t(kTrackWinObservations), n_gp = q.gp_cand.size();
    std::vector<int32_t> obs_lm(cap), obs_kf(cap), obs_cam(cap), gp_lm(n_gp + 1), gp_kf(n_gp + 1);
    std::vector<double> res(3 * cap), rho(2 * cap), trim_r(n_lm + 1), trim_d(n_lm + 1), gp_w(n_gp + 1), gp_r(n_gp + 1);
    std::vector<uint8_t> rej_r(n_lm + 1), rej_d(n_lm + 1);
    kba_evaluate_out out{};
    out.obs_capacity = int32_t(cap);
    out.obs_lm = obs_lm.data(); out.obs_kf = obs_kf.data(); out.obs_cam = obs_cam.data(); out.residual = res.data(); out.rho = rho.data();
    out.trim_repr = trim_r.data(); out.trim_depth = trim_d.data(); out.rejected_repr = rej_r.data(); out.rejected_depth = rej_d.data();
    out.gp_lm = gp_lm.data(); out.gp_kf = gp_kf.data(); out.gp_weight = gp_w.data(); out.gp_residual = gp_r.data();
    kba_track_request req{int32_t(kfs.size()), q.kf_slots.data(), q.fixed.data(), int32_t(n_lm), q.lm_slots.data(), &q.sel};
    if (kba_track_evaluate(track_, &req, &opt, &out) != KBA_OK) throw std::runtime_error(std::string(who) + "kba_b200: " + kba_last_error());
    last_evaluation_ = keyEvaluation(std::vector<const Keyframe*>(kfs.begin(), kfs.end()), lm_ids, track_cams_, out);
}

BundleAdjusterKeyframes::Evaluation keyEvaluation(const std::vector<const Keyframe*>& kfs, const std::vector<LandmarkId>& lm_ids,
                                                  const std::vector<std::array<double, 10>>& track_cams, const kba_evaluate_out& out) {
    BundleAdjusterKeyframes::Evaluation e;
    auto bad = [](const std::string& why) { throw std::runtime_error("evaluateResiduals: " + why); };
    int o = 0;
    for (size_t j = 0; j < lm_ids.size(); ++j) {
        for (size_t k = 0; k < kfs.size(); ++k) {
            const auto it = kfs[k]->measurements_.find(lm_ids[j]);
            if (it == kfs[k]->measurements_.end()) continue;
            for (const auto& cm : it->second) {
                if (o >= out.n_obs) bad("fewer observations in the window than the keyframes measure");
                const int cam = int(std::find(track_cams.begin(), track_cams.end(), camera_value(*kfs[k]->cameras_.at(cm.first))) - track_cams.begin());
                if (out.obs_lm[o] != int(j) || out.obs_kf[o] != int(k) || out.obs_cam[o] != cam)
                    bad("observation " + std::to_string(o) + " is not the one the host enumerates");
                BundleAdjusterKeyframes::Evaluation::Residual r;
                r.u = out.residual[3 * o]; r.v = out.residual[3 * o + 1]; r.depth = out.residual[3 * o + 2];
                r.rho_reprojection = out.rho[2 * o]; r.rho_depth = out.rho[2 * o + 1];
                e.residuals[std::make_tuple(lm_ids[j], KeyframeId(kfs[k]->timestamp_), cm.first)] = r;
                ++o;
            }
        }
        BundleAdjusterKeyframes::Evaluation::Trim t;
        t.reprojection = out.trim_repr[j]; t.depth = out.trim_depth[j];
        t.rejected_reprojection = out.rejected_repr[j] != 0; t.rejected_depth = out.rejected_depth[j] != 0;
        e.landmarks[lm_ids[j]] = t;
    }
    if (o != out.n_obs) bad("more observations in the window than the keyframes measure");
    for (int g = 0; g < out.n_gp; ++g) e.ground_plane[lm_ids.at(size_t(out.gp_lm[g]))] = out.gp_residual[g];
    e.cost_reprojection = out.cost[0]; e.cost_depth = out.cost[1]; e.cost_ground_plane = out.cost[2];
    e.cost_scale = out.cost[3]; e.cost_plane_chain = out.cost[4]; e.cost_total = out.cost[5];
    e.failed = out.failed != 0;
    return e;
}

// Landmark state the host changed since the store last saw it: position and weight of new landmarks (push()) and of landmarks
// that got a slot again after theirs was reclaimed, positions the rebuild path wrote (runWindow), weights set by updateLabels().
// A landmark without a slot is not in the store: its value goes up when it gets one (a new one with its keyframe, a reclaimed
// one through restore_landmarks_).  false: the store could not be written.
bool BundleAdjusterKeyframes::flushLandmarks() {
    std::vector<int32_t> slots;
    std::vector<double> pos, wgt;
    for (const auto id : restore_landmarks_) {
        auto it = lm_slot_.find(id);
        if (it == lm_slot_.end()) continue;
        const Landmark& lm = *landmarks_.at(id);
        slots.push_back(it->second); pos.insert(pos.end(), lm.pos.begin(), lm.pos.end()); wgt.push_back(lm.weight);
    }
    if (!slots.empty() && kba_track_set_landmarks(track_, int(slots.size()), slots.data(), pos.data(), wgt.data()) != KBA_OK) return false;
    restore_landmarks_.clear();
    slots.clear(); pos.clear(); wgt.clear();
    for (const auto id : new_landmarks_) {
        auto it = lm_slot_.find(id);
        if (it == lm_slot_.end()) continue;  // created, but its keyframe has not reached the store yet
        const Landmark& lm = *landmarks_.at(id);
        slots.push_back(it->second); pos.insert(pos.end(), lm.pos.begin(), lm.pos.end()); wgt.push_back(lm.weight);
    }
    if (!slots.empty() && kba_track_set_landmarks(track_, int(slots.size()), slots.data(), pos.data(), wgt.data()) != KBA_OK) return false;
    for (const auto id : std::set<LandmarkId>(new_landmarks_)) if (lm_slot_.count(id)) new_landmarks_.erase(id);
    slots.clear(); pos.clear();
    for (const auto id : dirty_positions_) {
        auto it = lm_slot_.find(id);
        if (it == lm_slot_.end()) continue;
        const Landmark& lm = *landmarks_.at(id);
        slots.push_back(it->second); pos.insert(pos.end(), lm.pos.begin(), lm.pos.end());
    }
    if (!slots.empty() && kba_track_set_landmarks(track_, int(slots.size()), slots.data(), pos.data(), nullptr) != KBA_OK) return false;
    dirty_positions_.clear();
    slots.clear(); wgt.clear();
    for (const auto id : dirty_weights_) { auto it = lm_slot_.find(id); if (it != lm_slot_.end()) { slots.push_back(it->second); wgt.push_back(landmarks_.at(id)->weight); } }
    if (!slots.empty() && kba_track_set_landmarks(track_, int(slots.size()), slots.data(), nullptr, wgt.data()) != KBA_OK) return false;
    dirty_weights_.clear();
    return true;
}

// adjustPoseOnly() against the device-resident store: only the frame goes up.  false: not possible for this frame (caller rebuilds).
bool BundleAdjusterKeyframes::adjustPoseTracked(Keyframe& kf, const std::vector<LandmarkId>& lm_ids, std::string& report) {
    if (lm_ids.empty() || int(lm_ids.size()) > kTrackWinLandmarks) return false;
    std::map<CameraId, int> cam_of;
    for (const auto& c : kf.cameras_) {
        const auto it = std::find(track_cams_.begin(), track_cams_.end(), camera_value(*c.second));
        if (it == track_cams_.end()) return false;  // a camera the store does not know
        cam_of[c.first] = int(it - track_cams_.begin());
    }
    std::vector<int32_t> lm, cam;
    std::vector<float> u, v, d;
    for (const auto id : lm_ids) {  // ascending landmark id, cameras in measurement order inside: runWindow's observation order
        auto it = lm_slot_.find(id);
        if (it == lm_slot_.end()) {
            // no stored keyframe measures it (any more): a slot from the free list, which is only filled once slots were
            // reclaimed, with its host state (flushLandmarks below); without a free slot the frame goes the rebuild path
            if (free_lm_slots_.empty()) return false;
            const int s = free_lm_slots_.back();
            free_lm_slots_.pop_back();
            slot_lm_[size_t(s)] = id;
            it = lm_slot_.emplace(id, s).first;
            restore_landmarks_.insert(id);
        }
        for (const auto& cm : kf.measurements_.at(id)) {
            lm.push_back(it->second); cam.push_back(cam_of.at(cm.first));
            u.push_back(cm.second.u); v.push_back(cm.second.v); d.push_back(cm.second.d);
        }
    }
    if (int(lm.size()) > kTrackWinObservations) return false;
    if (!flushLandmarks()) { track_failed_ = true; return false; }
    kba_window w{};  // carries the speed prior
    speedPrior(kf, w);
    kba_track_frame f{};
    f.n_meas = int(lm.size());
    f.pose7 = kf.pose_.data(); f.lm_slot = lm.data(); f.cam = cam.data(); f.u = u.data(); f.v = v.data(); f.d = d.data();
    f.speed_weight = w.speed_weight; f.speed_dt = w.speed_dt;
    std::copy_n(w.speed_v_before, 3, f.speed_v_before);
    std::copy_n(w.speed_T_origin_before, 7, f.speed_T_origin_before);
    const kba_options opt = solve_options(outlier_rejection_options_, solver_time_sec, true, selected_landmark_ids_.size());
    double out_pose[7];
    kba_result r{};
    r.kf_pose = out_pose;
    const int rc = kba_track_adjust_pose(track_, &f, &opt, &r);
    if (rc == KBA_ERR_CAPACITY) return false;
    if (rc != KBA_OK) throw std::runtime_error(std::string("kba_b200: ") + kba_last_error());
    int64_t h2d = 0;
    kba_track_transfer_bytes(track_, &h2d, nullptr, nullptr);
    last_solve_h2d_ = (long long)h2d;  // the frame upload
    std::copy_n(out_pose, 7, kf.pose_.begin());  // in place, as the reference
    report = solve_report(r, " (device-resident window)");
    return true;
}

std::string BundleAdjusterKeyframes::adjustPoseOnly(Keyframe& kf) {  // cpp:820-888
    selected_landmark_ids_ = landmark_selector_->getLastSelection();
    std::vector<LandmarkId> lm_ids;
    for (const auto& m : kf.measurements_)
        if (selected_landmark_ids_.count(m.first)) lm_ids.push_back(m.first);  // landmarks_.at() would throw like the reference
    std::string report;
    if (persistent_window_ && track_ && !track_failed_ && adjustPoseTracked(kf, lm_ids, report)) return report;
    return runWindow({&kf}, lm_ids, true, &kf);
}

}  // namespace keyframe_bundle_adjustment
