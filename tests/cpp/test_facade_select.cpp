// limo's mono-lidar selection chain through the facade (mono_lidar.cpp:383-429: LandmarkRejectionSchemeCheirality, then
// LandmarkSparsificationSchemeVoxel with voxels of 0.5 / 0.5 / 0.3 m, regions of 40 / 15 m and 400 landmarks per bin, then
// LandmarkSelectionSchemeAddDepth with 50 ground landmarks per keyframe) on a drive with scene and road landmarks.  Adjuster `a`
// selects with the store computing the chain's per-landmark quantities (kba_track_select_landmarks), its twin `b` selects on the
// host (set_device_selection(false)); both keep the persistent window.  std::srand is reseeded identically before each solve().
// Checks, for a 12- and a 20-keyframe window over 33 keyframes (30 solves each):
//   - every solve() of `a` selects on the device, none of `b` does;
//   - at every solve() the selections, the selector's categories and its unselected-landmark counters are equal;
//   - poses, planes and all landmarks of both adjusters are bit-identical after every solve and at the end;
//   - the chain did its work: landmarks rejected by cheirality, all three bins filled, a bin capped (the ranking decides).
// With arguments `W n_scene n_frames` it prints timings instead (median / p90 per solve, ms): the host select() of a standalone
// selector on the same state, and the facade's solve() with device and with host selection (scripts/select_bench.py).
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
        if (el.second->pos != b.landmarks_.at(el.first)->pos) return false;
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

// returns the number of solves; bench: print timings instead of checking
static int drive(int window, int n_scene, int n_frames, bool bench) {
    const int n_ground = n_scene / 4;
    const double height = 1.6;
    std::vector<Eigen::Vector3d> lms;  // origin frame = first vehicle frame: x forward, z up, the ground at z = -height
    for (int i = 0; i < n_scene; ++i)
        lms.push_back(Eigen::Vector3d(4. + 0.061 * ((i * 37) % 1201), -30. + 0.047 * ((i * 53) % 1279), -1. + 0.011 * ((i * 29) % 997)));
    for (int i = 0; i < n_ground; ++i)
        lms.push_back(Eigen::Vector3d(6. + 0.05 * ((i * 41) % 997), -6. + 0.013 * ((i * 23) % 991), -height));
    std::vector<Eigen::Isometry3d> gt(n_frames);  // vehicle <- origin
    gt[0] = Eigen::Isometry3d::Identity();
    for (int k = 1; k < n_frames; ++k) {
        gt[k] = gt[k - 1];
        gt[k].translate(Eigen::Vector3d(-0.6, 0.01 * (k % 3), 0.));
        gt[k].rotate(Eigen::AngleAxisd(0.003, Eigen::Vector3d(0., 0., 1.)));
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
        // tracks end: the later a track ends, the longer its flow; some are seen in one frame only (no flow)
        const int len = (i % 11 == 0) ? 1 : 2 + int((i * 7) % size_t(n_frames));
        for (int k = 0; k < std::min(len, n_frames); ++k) {
            const Eigen::Vector3d lm_cam = ext * (gt[k] * lms[i]);
            Eigen::Vector3d proj = proto.getIntrinsicMatrix() * lm_cam;
            proj /= proj[2];
            const float du = 0.3f * float((int(i) * 7 + k * 3) % 5 - 2), dv = 0.3f * float((int(i) * 3 + k * 5) % 5 - 2);
            const float d = (!ground && i % 3 == 0) ? float(lm_cam[2]) : -1.f;
            ts.tracks[i].feature_points.push_back(FeaturePoint(float(proj[0]) + du, float(proj[1]) + dv, d));
        }
    }
    BundleAdjusterKeyframes a, b;
    b.set_device_selection(false);
    for (BundleAdjusterKeyframes* adj : {&a, &b}) {
        adj->set_solver_time(20.);
        add_chain(*adj->landmark_selector_, window);
    }
    Plane plane;
    plane.distance = height;
    auto cam = [&] { return std::make_shared<Camera>(700., Eigen::Vector2d(600., 190.), ext); };
    int solves = 0, on_device = 0, rejected = 0, capped = 0;
    size_t bins[3] = {0, 0, 0};
    std::vector<double> t_host_select, t_solve_a, t_solve_b;
    using clk = std::chrono::steady_clock;
    auto ms = [](clk::time_point t0) { return std::chrono::duration<double, std::milli>(clk::now() - t0).count(); };
    for (int k = 0; k < n_frames; ++k) {
        Eigen::Isometry3d start = gt[k];
        if (k >= 2) start.translate(Eigen::Vector3d(0.03, -0.02, 0.01));
        const auto fix = k == 0 ? Keyframe::FixationStatus::Pose : (k == 1 ? Keyframe::FixationStatus::Scale : Keyframe::FixationStatus::None);
        for (BundleAdjusterKeyframes* adj : {&a, &b}) adj->push(Keyframe(k, ts, cam(), start, fix, plane));
        if (k < 3) continue;
        for (BundleAdjusterKeyframes* adj : {&a, &b}) {
            adj->deactivateKeyframes(3, 4, window);
            adj->updateLabels(ts, 0.9);
        }
        if (bench) {  // the host select() alone, on a standalone selector with the same chain and outliers
            LandmarkSelector s;
            s.addScheme(LandmarkRejectionSchemeCheirality::create());
            add_chain(s, window);
            s.setOutlier(a.landmark_selector_->getOutliers());
            std::srand(1000 + k);
            const auto t0 = clk::now();
            s.select(a.getActiveLandmarkConstPtrs(), a.getActiveKeyframeConstPtrs());
            t_host_select.push_back(ms(t0));
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
        on_device += a.lastSelectionOnDevice();
        CHECK(!b.lastSelectionOnDevice());
        CHECK(ra.find("device-resident") != std::string::npos && rb.find("device-resident") != std::string::npos);
        CHECK(a.selected_landmark_ids_ == b.selected_landmark_ids_);
        CHECK(a.landmark_selector_->getLandmarkCategories() == b.landmark_selector_->getLandmarkCategories());
        CHECK(a.landmark_selector_->getUnselectedLandmarks() == b.landmark_selector_->getUnselectedLandmarks());
        CHECK(same_state(a, b));
        size_t per_bin[3] = {0, 0, 0};
        for (const auto& el : a.landmark_selector_->getLandmarkCategories()) {
            ++bins[int(el.second)];
            ++per_bin[int(el.second)];
        }
        capped += per_bin[0] == 400 || per_bin[1] == 400 || per_bin[2] == 400;
        rejected += int(a.getActiveLandmarkConstPtrs().size() - a.landmark_selector_->getOutliers().size() >
                        a.selected_landmark_ids_.size());
    }
    if (bench) {
        std::printf("{\"window\": %d, \"landmarks\": %zu, \"solves\": %d, \"host_select_ms\": [%.3f, %.3f], "
                    "\"solve_device_select_ms\": [%.3f, %.3f], \"solve_host_select_ms\": [%.3f, %.3f]}\n",
                    window, a.getActiveLandmarkConstPtrs().size(), solves, pct(t_host_select, 0.5), pct(t_host_select, 0.9),
                    pct(t_solve_a, 0.5), pct(t_solve_a, 0.9), pct(t_solve_b, 0.5), pct(t_solve_b, 0.9));
        return solves;
    }
    CHECK(on_device == solves);
    CHECK(bins[0] > 0 && bins[1] > 0 && bins[2] > 0);
    CHECK(capped > 0);
    CHECK(rejected > 0);
    std::printf("window %d: %d solves, %d with device-side selection; categories near / middle / far %zu / %zu / %zu over all solves, "
                "a bin capped in %d; solve() median %.2f ms (device selection), %.2f ms (host selection)\n",
                window, solves, on_device, bins[0], bins[1], bins[2], capped, pct(t_solve_a, 0.5), pct(t_solve_b, 0.5));
    return solves;
}

int main(int argc, char** argv) {
    std::setvbuf(stdout, nullptr, _IOLBF, 0);
    if (argc == 4) {
        drive(std::atoi(argv[1]), std::atoi(argv[2]), std::atoi(argv[3]), true);
        return 0;
    }
    for (const int window : {12, 20}) CHECK(drive(window, 1400, 33, false) == 30);
    std::printf("%d failed checks\n", g_fail);
    return g_fail ? 1 : 0;
}
