// The facade past its store's landmark capacity.  Adjuster `a` has a store of 4096 landmark slots (set_track_capacity) and limo's
// mono-lidar chain (cheirality, voxel, AddDepth with the ground comparator); its twin `b` rebuilds every window
// (set_persistent_window(false)).  The drive makes 60 new landmarks per keyframe (scene points, some with a lidar depth, and road
// points labelled ground) and 5 revisited ones, seen for three keyframes and again 25 keyframes later, long after every keyframe
// of the first visit has left the window.  Both adjusters follow limo's per-frame step: adjustPoseOnly on the frame, push,
// deactivateKeyframes(3, 4, 12), updateLabels, solve.  The drive makes several times 4096 landmarks, so `a` reclaims slots
// (kba_track_reclaim_landmarks) again and again and restores revisited landmarks.  Checks:
//   - every solve() of `a` selects on the device and solves on the device-resident window: the store was never abandoned
//     (before landmark slots were reclaimed, the push that ran out of slots sent `a` to the rebuild path for good);
//   - after every solve, keyframe poses and planes and every landmark position of both adjusters are bit-identical, as are the
//     selections;
//   - every adjustPoseOnly() of `a` runs on the store, its pose agrees with the twin's to 1e-9 m with the same iteration counts
//     (one kernel against the general solver), and it leaves both adjusters' states bit-identical.
// With arguments `n_frames bench` it prints timings instead (median / p90 of solve() and adjustPoseOnly(), ms, for `a` and `b`;
// scripts/reclaim_bench.py).
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
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

static bool same_state(const BundleAdjusterKeyframes& a, const BundleAdjusterKeyframes& b) {
    if (a.active_keyframe_ids_ != b.active_keyframe_ids_ || a.selected_landmark_ids_ != b.selected_landmark_ids_) return false;
    for (const auto& el : a.keyframes_) {
        const Keyframe& ka = *el.second;
        const Keyframe& kb = *b.keyframes_.at(el.first);
        if (ka.pose_ != kb.pose_ || ka.local_ground_plane_.direction != kb.local_ground_plane_.direction ||
            ka.local_ground_plane_.distance != kb.local_ground_plane_.distance)
            return false;
    }
    if (a.landmarks_.size() != b.landmarks_.size()) return false;
    for (const auto& el : a.landmarks_)
        if (el.second->pos != b.landmarks_.at(el.first)->pos || el.second->weight != b.landmarks_.at(el.first)->weight) return false;
    return true;
}

static void add_chain(LandmarkSelector& s, int window) {  // mono_lidar.cpp:383-429 (cheirality is the adjuster's default)
    LandmarkSparsificationSchemeVoxel::Parameters pv;
    pv.voxel_size_xyz = {{0.5, 0.5, 0.3}};
    pv.roi_far_xyz = {{40., 40., 40.}};
    pv.roi_middle_xyz = {{15., 15., 15.}};
    pv.max_num_landmarks_near = pv.max_num_landmarks_middle = pv.max_num_landmarks_far = 400;
    s.addScheme(LandmarkSparsificationSchemeVoxel::create(pv));
    LandmarkSelectionSchemeAddDepth::Parameters p;
    auto gp_comparator = [](const Landmark::ConstPtr& lm) { return lm->is_ground_plane; };
    auto gp_sorter = [](const Measurement&, const Eigen::Vector3d& local) { return float(local.norm()); };
    for (int i = 0; i < window; ++i) p.params_per_keyframe.push_back(std::make_tuple(i, 50, gp_comparator, gp_sorter));
    s.addScheme(LandmarkSelectionSchemeAddDepth::create(p));
}

static double pct(std::vector<double> v, double q) {
    std::sort(v.begin(), v.end());
    return v.empty() ? 0. : v[std::min(v.size() - 1, size_t(q * double(v.size())))];
}

struct Lm {
    Eigen::Vector3d p;
    std::vector<int> frames;  // ascending
    bool ground;
};

int main(int argc, char** argv) {
    std::setvbuf(stdout, nullptr, _IOLBF, 0);
    const bool bench = argc == 3;
    const int n_frames = bench ? std::atoi(argv[1]) : 130, window = 12, cap = 4096;
    const double height = 1.6;
    std::vector<Eigen::Isometry3d> gt(n_frames);  // vehicle <- origin; origin = first vehicle frame, x forward, z up
    gt[0] = Eigen::Isometry3d::Identity();
    for (int k = 1; k < n_frames; ++k) {
        gt[k] = gt[k - 1];
        gt[k].translate(Eigen::Vector3d(-0.6, 0.01 * (k % 3), 0.));
        gt[k].rotate(Eigen::AngleAxisd(0.002 * ((k / 20) % 2 ? 1. : -1.), Eigen::Vector3d(0., 0., 1.)));
    }
    std::vector<Lm> lms;
    for (int k = 0; k < n_frames; ++k) {
        const Eigen::Vector3d at = gt[k].inverse().translation();
        for (int j = 0; j < 60; ++j) {
            const int i = int(lms.size());
            Lm l;
            l.ground = j % 4 == 3;
            l.p = l.ground ? at + Eigen::Vector3d(8. + 0.37 * ((i * 41) % 61), -6. + 0.013 * ((i * 23) % 991), 0.)
                           : at + Eigen::Vector3d(10. + 0.061 * ((i * 37) % 601), -15. + 0.047 * ((i * 53) % 641), 0.);
            l.p[2] = l.ground ? -height : -1. + 0.011 * ((i * 29) % 457);
            const int len = 3 + (i * 7) % 8;
            for (int f = k; f < std::min(n_frames, k + len); ++f) l.frames.push_back(f);
            lms.push_back(l);
        }
        for (int j = 0; j < 5; ++j) {  // revisited: three keyframes now, two keyframes 25 later
            const int i = int(lms.size());
            Lm l;
            l.ground = false;
            l.p = at + Eigen::Vector3d(45. + 0.41 * ((i * 13) % 61), -10. + 0.29 * ((i * 7) % 67), -0.5 + 0.05 * ((i * 3) % 61));
            for (const int f : {k, k + 1, k + 2, k + 25, k + 26})
                if (f < n_frames) l.frames.push_back(f);
            lms.push_back(l);
        }
    }
    Eigen::Matrix3d rc = Eigen::Matrix3d::Zero();  // camera <- vehicle: camera z forward, x right, y down
    rc(0, 1) = -1.; rc(1, 2) = -1.; rc(2, 0) = 1.;
    Eigen::Isometry3d ext = Eigen::Isometry3d::Identity();
    ext.rotate(rc);
    const Camera proto(700., Eigen::Vector2d(600., 190.), ext);
    std::vector<Tracklets> frame_ts(n_frames);  // one message per frame: the tracks it sees, one feature point each
    for (int k = 0; k < n_frames; ++k) frame_ts[k].stamps.push_back(k);
    for (size_t i = 0; i < lms.size(); ++i)
        for (const int k : lms[i].frames) {
            const Eigen::Vector3d lm_cam = ext * (gt[k] * lms[i].p);
            Eigen::Vector3d proj = proto.getIntrinsicMatrix() * lm_cam;
            proj /= proj[2];
            const float du = 0.3f * float((int(i) * 7 + k * 3) % 5 - 2), dv = 0.3f * float((int(i) * 3 + k * 5) % 5 - 2);
            const float d = (!lms[i].ground && i % 3 == 0 && k == lms[i].frames[0]) ? float(lm_cam[2]) : -1.f;
            Tracklet t = Tracklet();
            t.id = i;
            t.label = lms[i].ground ? 7 : 0;  // 7: road, one of the "ground" labels
            t.feature_points.push_back(FeaturePoint(float(proj[0]) + du, float(proj[1]) + dv, d));
            frame_ts[k].tracks.push_back(t);
        }
    BundleAdjusterKeyframes a, b;
    a.set_track_capacity(256, cap, 1 << 21);
    b.set_persistent_window(false);
    for (BundleAdjusterKeyframes* adj : {&a, &b}) {
        adj->set_solver_time(20.);
        add_chain(*adj->landmark_selector_, window);
    }
    Plane plane;
    plane.distance = height;
    auto cam = [&] { return std::make_shared<Camera>(700., Eigen::Vector2d(600., 190.), ext); };
    using clk = std::chrono::steady_clock;
    auto ms = [](clk::time_point t0) { return std::chrono::duration<double, std::milli>(clk::now() - t0).count(); };
    std::vector<double> t_solve_a, t_solve_b, t_pose_a, t_pose_b;
    int solves = 0, on_device = 0, frames = 0, tracked_frames = 0;
    double max_dt = 0.;
    for (int k = 0; k < n_frames; ++k) {
        Eigen::Isometry3d start = gt[k];
        if (k >= 2) start.translate(Eigen::Vector3d(0.03, -0.02, 0.01));
        const auto fix = k == 0 ? Keyframe::FixationStatus::Pose : (k == 1 ? Keyframe::FixationStatus::Scale : Keyframe::FixationStatus::None);
        if (k >= 4) {  // track the frame before it becomes a keyframe
            Keyframe fa(k, frame_ts[k], cam(), start, fix, plane), fb(k, frame_ts[k], cam(), start, fix, plane);
            auto t0 = clk::now();
            const std::string ra = a.adjustPoseOnly(fa);
            t_pose_a.push_back(ms(t0));
            t0 = clk::now();
            const std::string rb = b.adjustPoseOnly(fb);
            t_pose_b.push_back(ms(t0));
            double dt = 0.;
            for (int i = 4; i < 7; ++i) dt += (fa.pose_[i] - fb.pose_[i]) * (fa.pose_[i] - fb.pose_[i]);
            max_dt = std::max(max_dt, std::sqrt(dt));
            CHECK(std::sqrt(dt) <= 1e-9);
            CHECK(iterations(ra) == iterations(rb));
            CHECK(same_state(a, b));
            ++frames;
            tracked_frames += ra.find("device-resident") != std::string::npos;
        }
        for (BundleAdjusterKeyframes* adj : {&a, &b}) adj->push(Keyframe(k, frame_ts[k], cam(), start, fix, plane));
        if (k < 3) continue;
        for (BundleAdjusterKeyframes* adj : {&a, &b}) {
            adj->deactivateKeyframes(3, 4, window);
            adj->updateLabels(frame_ts[k], 0.9);
        }
        std::srand(1000 + k);
        auto t0 = clk::now();
        const std::string ra = a.solve();
        t_solve_a.push_back(ms(t0));
        std::srand(1000 + k);
        t0 = clk::now();
        const std::string rb = b.solve();
        t_solve_b.push_back(ms(t0));
        ++solves;
        const bool dev = a.lastSelectionOnDevice() && ra.find("device-resident") != std::string::npos;
        on_device += dev;
        CHECK(dev);
        CHECK(rb.find("device-resident") == std::string::npos);
        CHECK(iterations(ra) == iterations(rb));
        CHECK(same_state(a, b));
    }
    if (bench) {
        std::printf("{\"frames\": %d, \"landmarks\": %zu, \"capacity\": %d, \"solve_ms\": [%.3f, %.3f], \"solve_rebuild_ms\": [%.3f, %.3f], "
                    "\"adjust_pose_ms\": [%.3f, %.3f], \"adjust_pose_rebuild_ms\": [%.3f, %.3f], \"solves_on_device\": %d, \"solves\": %d}\n",
                    n_frames, a.landmarks_.size(), cap, pct(t_solve_a, 0.5), pct(t_solve_a, 0.9), pct(t_solve_b, 0.5), pct(t_solve_b, 0.9),
                    pct(t_pose_a, 0.5), pct(t_pose_a, 0.9), pct(t_pose_b, 0.5), pct(t_pose_b, 0.9), on_device, solves);
        return 0;
    }
    CHECK(a.landmarks_.size() > size_t(2 * cap));
    CHECK(solves == n_frames - 3 && on_device == solves);
    CHECK(frames == n_frames - 4 && tracked_frames == frames);
    std::printf("%zu landmarks through %d slots: %d of %d solves on the device-resident window with device selection, %d of %d "
                "frames tracked on the store, max pose difference %.3g m\n",
                a.landmarks_.size(), cap, on_device, solves, tracked_frames, frames, max_dt);
    std::printf("%d failed checks\n", g_fail);
    return g_fail ? 1 : 0;
}
