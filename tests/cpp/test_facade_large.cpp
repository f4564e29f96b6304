// limo's default mono-lidar window through the facade: test_facade_ground.cpp's drive with deactivateKeyframes(3, 4, 20) (the
// max_size_optimization_window default of the mono-lidar node) over 26 frames, so that the window grows through 18 keyframes into
// 19 and 20 with ground points attached -- more than 184 reduced rows, the track's large-window solver.  Adjuster `a` keeps the
// persistent window, its twin `b` rebuilds every window (set_persistent_window(false)).  Checks:
//   - every solve() of `a` runs on the device-resident window, and after it poses, planes and selected landmarks of both
//     adjusters are bit-identical, with the same iteration counts;
//   - windows of 19 and more keyframes with ground landmarks are solved, and ground points move planes in them;
//   - every adjustPoseOnly() of `a` runs on the store, agrees with the twin's pose to 1e-9 m and leaves both states bit-identical.
#include <cmath>
#include <cstdio>
#include <string>
#include <vector>

#include "keyframe_bundle_adjustment/bundle_adjuster_keyframes.hpp"
#include "keyframe_bundle_adjustment/landmark_selection_schemes.hpp"

using namespace keyframe_bundle_adjustment;
static int g_fail = 0;
#define CHECK(c) do { if (!(c)) { std::printf("CHECK FAILED %s:%d: %s\n", __FILE__, __LINE__, #c); ++g_fail; } } while (0)

static std::vector<int> iterations(const std::string& report) {
    std::vector<int> out;
    const std::string key = ", iterations ";
    for (size_t p = report.find(key); p != std::string::npos; p = report.find(key, p + 1)) out.push_back(std::atoi(report.c_str() + p + key.size()));
    return out;
}

// keyframes (poses and planes) and selected landmarks of the two adjusters, bit for bit
static bool same_state(const BundleAdjusterKeyframes& a, const BundleAdjusterKeyframes& b) {
    if (a.active_keyframe_ids_ != b.active_keyframe_ids_ || a.selected_landmark_ids_ != b.selected_landmark_ids_) return false;
    for (const auto& id : a.active_keyframe_ids_) {
        const Keyframe& ka = *a.keyframes_.at(id);
        const Keyframe& kb = *b.keyframes_.at(id);
        if (ka.pose_ != kb.pose_ || ka.local_ground_plane_.direction != kb.local_ground_plane_.direction ||
            ka.local_ground_plane_.distance != kb.local_ground_plane_.distance)
            return false;
    }
    for (const auto& id : a.selected_landmark_ids_)
        if (a.landmarks_.at(id)->pos != b.landmarks_.at(id)->pos) return false;
    return true;
}

int main() {
    std::setvbuf(stdout, nullptr, _IOLBF, 0);
    const int n_frames = 26, n_scene = 150, n_ground = 89;
    const double height = 1.6;
    // origin frame = first vehicle frame: x forward, z up; the ground is z = -height
    std::vector<Eigen::Vector3d> lms;
    for (int i = 0; i < n_scene; ++i)
        lms.push_back(Eigen::Vector3d(14. + 0.17 * ((i * 37) % 151), -6. + 0.09 * ((i * 53) % 131), -1. + 0.035 * ((i * 29) % 113)));
    for (int i = 0; i < n_ground; ++i)  // 12 - 30 m ahead of the first keyframe: the farthest are not attached at first
        lms.push_back(Eigen::Vector3d(12. + 0.2 * ((i * 41) % 89), -5. + 0.11 * ((i * 23) % 89), -height));
    std::vector<Eigen::Isometry3d> gt(n_frames);  // vehicle <- origin
    gt[0] = Eigen::Isometry3d::Identity();
    for (int k = 1; k < n_frames; ++k) {
        gt[k] = gt[k - 1];
        gt[k].translate(Eigen::Vector3d(-0.35, 0.01 * (k % 3), 0.));  // 8.75 m in all: every point stays ahead
        gt[k].rotate(Eigen::AngleAxisd(0.004, Eigen::Vector3d(0., 0., 1.)));
    }
    Eigen::Matrix3d rc = Eigen::Matrix3d::Zero();  // camera <- vehicle: camera z forward, x right, y down
    rc(0, 1) = -1.; rc(1, 2) = -1.; rc(2, 0) = 1.;
    Eigen::Isometry3d ext = Eigen::Isometry3d::Identity();
    ext.rotate(rc);
    const Camera proto(700., Eigen::Vector2d(600., 190.), ext);
    Tracklets ts;
    for (int k = 0; k < n_frames; ++k) ts.stamps.push_back(k);
    ts.tracks.resize(lms.size());
    for (size_t i = 0; i < lms.size(); ++i) {
        const bool ground = int(i) >= n_scene;
        ts.tracks[i].id = i;
        ts.tracks[i].label = ground ? 7 : 0;  // 7: road, one of the "ground" labels
        for (int k = 0; k < n_frames; ++k) {
            const Eigen::Vector3d lm_cam = ext * (gt[k] * lms[i]);
            Eigen::Vector3d proj = proto.getIntrinsicMatrix() * lm_cam;
            proj /= proj[2];
            const float du = 0.3f * float((int(i) * 7 + k * 3) % 5 - 2), dv = 0.3f * float((int(i) * 3 + k * 5) % 5 - 2);
            const float d = (!ground && i % 3 == 0) ? float(lm_cam[2]) : -1.f;  // lidar depth on some scene points
            ts.tracks[i].feature_points.push_back(FeaturePoint(float(proj[0]) + du, float(proj[1]) + dv, d));
        }
    }
    BundleAdjusterKeyframes a, b;
    b.set_persistent_window(false);
    for (BundleAdjusterKeyframes* adj : {&a, &b}) {
        adj->set_solver_time(20.);
        LandmarkSelectionSchemeAddDepth::Parameters p;
        auto gp_comparator = [](const Landmark::ConstPtr& lm) { return lm->is_ground_plane; };
        auto gp_sorter = [](const Measurement&, const Eigen::Vector3d& local) { return float(local.norm()); };
        for (int i = 0; i < 20; ++i) p.params_per_keyframe.push_back(std::make_tuple(i, 50, gp_comparator, gp_sorter));
        adj->landmark_selector_->addScheme(LandmarkSelectionSchemeAddDepth::create(p));
    }
    Plane plane;
    plane.distance = height;
    auto cam = [&] { return std::make_shared<Camera>(700., Eigen::Vector2d(600., 190.), ext); };
    int solves = 0, tracked_solves = 0, frames = 0, tracked_frames = 0, moved_planes = 0, large_solves = 0, large_moved = 0;
    size_t max_kf = 0;
    size_t max_ground = 0;
    long long up_a = 0, up_b = 0, fr_a = 0, fr_b = 0;
    double max_dt = 0., max_ratio = 0.;
    for (int k = 0; k < n_frames; ++k) {
        Eigen::Isometry3d start = gt[k];
        if (k >= 2) start.translate(Eigen::Vector3d(0.03, -0.02, 0.01));
        const auto fix = k == 0 ? Keyframe::FixationStatus::Pose : (k == 1 ? Keyframe::FixationStatus::Scale : Keyframe::FixationStatus::None);
        if (k >= 4) {  // track the frame before it becomes a keyframe
            Keyframe fa(k, ts, cam(), start, fix, plane), fb(k, ts, cam(), start, fix, plane);
            const std::string ra = a.adjustPoseOnly(fa), rb = b.adjustPoseOnly(fb);
            double dt = 0.;
            for (int i = 4; i < 7; ++i) dt += (fa.pose_[i] - fb.pose_[i]) * (fa.pose_[i] - fb.pose_[i]);
            dt = std::sqrt(dt);
            max_dt = std::max(max_dt, dt);
            CHECK(dt <= 1e-9);
            CHECK(!iterations(ra).empty() && iterations(ra) == iterations(rb));
            CHECK(rb.find("device-resident") == std::string::npos);
            CHECK(same_state(a, b));
            ++frames;
            if (ra.find("device-resident") != std::string::npos) {
                ++tracked_frames;
                const long long n_meas = (long long)a.selected_landmark_ids_.size();  // every landmark is seen in every frame
                CHECK(a.lastSolveUploadBytes() > 0 && a.lastSolveUploadBytes() <= 24 * n_meas + 2048);  // the frame, not a window
                fr_a += a.lastSolveUploadBytes(); fr_b += b.lastSolveUploadBytes();
            }
        }
        for (BundleAdjusterKeyframes* adj : {&a, &b}) adj->push(Keyframe(k, ts, cam(), start, fix, plane));
        if (k < 3) continue;
        for (BundleAdjusterKeyframes* adj : {&a, &b}) {
            adj->deactivateKeyframes(3, 4, 20);
            adj->updateLabels(ts, 0.9);
        }
        const std::string ra = a.solve(), rb = b.solve();
        ++solves;
        tracked_solves += ra.find("device-resident") != std::string::npos;
        CHECK(rb.find("device-resident") == std::string::npos);
        CHECK(iterations(ra) == iterations(rb));
        CHECK(same_state(a, b));
        size_t n_ground_sel = 0;
        for (const auto& id : a.selected_landmark_ids_) n_ground_sel += a.landmarks_.at(id)->is_ground_plane;
        max_ground = std::max(max_ground, n_ground_sel);
        int moved = 0;
        for (const auto& id : a.active_keyframe_ids_) moved += a.keyframes_.at(id)->local_ground_plane_.distance != height;
        moved_planes += moved;
        max_kf = std::max(max_kf, a.active_keyframe_ids_.size());
        if (a.active_keyframe_ids_.size() >= 19 && n_ground_sel > 0) {  // 10 * 19 + 1 = 191 reduced rows: the large-window solver
            ++large_solves;
            large_moved += moved;
        }
        const double ratio = double(a.lastSolveUploadBytes()) / double(b.lastSolveUploadBytes());
        max_ratio = std::max(max_ratio, ratio);
        CHECK(ratio < 0.1);
        up_a += a.lastSolveUploadBytes(); up_b += b.lastSolveUploadBytes();
    }
    CHECK(solves == n_frames - 3 && tracked_solves == solves);
    CHECK(max_ground >= 30);
    CHECK(moved_planes > 0);  // ground points were attached: the plane chain moved planes
    CHECK(max_kf == 20 && large_solves >= 3 && large_moved > 0);
    CHECK(frames == n_frames - 4 && tracked_frames == frames);
    CHECK(fr_a > 0 && fr_a < fr_b);
    std::printf("solve(): %d of %d on the device-resident window (%d of them with 19-20 keyframes and ground landmarks), up to %zu "
                "ground landmarks selected, upload %lld B per solve (rebuild path %lld B, largest ratio %.3f)\n", tracked_solves, solves,
                large_solves, max_ground, up_a / solves, up_b / solves, max_ratio);
    std::printf("adjustPoseOnly(): %d of %d frames tracked, max pose difference %.3g m, upload %lld B per frame (rebuild path %lld B)\n",
                tracked_frames, frames, max_dt, tracked_frames ? fr_a / tracked_frames : 0, tracked_frames ? fr_b / tracked_frames : 0);
    std::printf("%d failed checks\n", g_fail);
    return g_fail ? 1 : 0;
}
