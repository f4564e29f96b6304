// evaluateResiduals() of the facade on the device-resident store (kba_track_evaluate).
//   host mode (argument "host", no GPU needed): with the persistent window off, and before the first solve(), it throws
//   std::runtime_error naming the reason; keyEvaluation keys a hand-made output by (landmark id, keyframe timestamp, camera id) and
//   by landmark id, and refuses an output in another order.
//   default mode (GPU): a two-camera drive with lidar depths; after every solve(), evaluateResiduals() gives one residual per
//   measurement of a selected landmark in an active keyframe, each equal to a host computation from the facade's own state (pose,
//   camera, landmark, measurement) to 1e-9, losses whose halves sum to the reprojection and depth costs, a trimming value per
//   selected landmark equal to the largest norm of its residuals, and no change to poses, landmarks or the selection.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include "kba_b200.h"
#include "keyframe_bundle_adjustment/bundle_adjuster_keyframes.hpp"

using namespace keyframe_bundle_adjustment;
static int g_fail = 0;
#define CHECK(c) do { if (!(c)) { std::printf("CHECK FAILED %s:%d: %s\n", __FILE__, __LINE__, #c); ++g_fail; } } while (0)

static std::string thrown(BundleAdjusterKeyframes& a) {
    try { a.evaluateResiduals(); } catch (const std::runtime_error& e) { return e.what(); }
    return "";
}

// half a metre to the side of the vehicle frame
static Eigen::Isometry3d side() {
    Eigen::Isometry3d T = Eigen::Isometry3d::Identity();
    T.translate(Eigen::Vector3d(-0.5, 0., 0.));
    return T;
}

static int host_mode() {
    {   // persistent window off: no host evaluation
        BundleAdjusterKeyframes a;
        a.set_persistent_window(false);
        const std::string w = thrown(a);
        CHECK(w.find("persistent window is off") != std::string::npos);
        std::printf("persistent window off: %s\n", w.c_str());
    }
    {   // before the first solve(): no store yet
        BundleAdjusterKeyframes a;
        const std::string w = thrown(a);
        CHECK(w.find("solve() first") != std::string::npos);
        std::printf("before solve(): %s\n", w.c_str());
    }
    // keying: two keyframes, two cameras (store indices 1 and 0: the order of the store's camera list), three landmarks
    const Camera ca(600., Eigen::Vector2d(300., 200.), Eigen::Isometry3d::Identity());
    const Camera cb(500., Eigen::Vector2d(320., 240.), side());
    auto value = [](const Camera& c) {
        std::array<double, 10> v{{c.focal_length, c.principal_point[0], c.principal_point[1]}};
        std::copy(c.pose_camera_vehicle.begin(), c.pose_camera_vehicle.end(), v.begin() + 3);
        return v;
    };
    const std::vector<std::array<double, 10>> track_cams{value(cb), value(ca)};
    Tracklets t;
    t.stamps = {100, 200};
    t.tracks.resize(3);
    for (int i = 0; i < 3; ++i) {
        t.tracks[i].id = 10 + i;
        t.tracks[i].feature_points = {FeaturePoint(1.f + i, 2.f, -1.f), FeaturePoint(3.f + i, 4.f, 5.f)};
    }
    std::map<CameraId, Camera::Ptr> cams{{7, std::make_shared<Camera>(ca)}, {9, std::make_shared<Camera>(cb)}};
    std::vector<Keyframe> kfs_v;
    for (int k = 0; k < 2; ++k) {
        Tracklets tk = t;
        const std::map<LandmarkId, CameraIds> lookup{{10, {7, 9}}, {11, {7, 9}}, {12, {7, 9}}};
        kfs_v.emplace_back(TimestampNSec(100 * (k + 1)), tk, cams, lookup, Eigen::Isometry3d::Identity(), Keyframe::FixationStatus::None);
    }
    const std::vector<const Keyframe*> kfs{&kfs_v[0], &kfs_v[1]};
    const std::vector<LandmarkId> lm_ids{10, 12};  // landmark 11 is not selected
    // the window's order: landmark 10 (kf 0: cam 7, 9; kf 1: cam 7, 9), then landmark 12 (likewise)
    std::vector<int32_t> olm, okf, ocam;
    std::vector<double> res, rho;
    for (int j = 0; j < 2; ++j)
        for (int k = 0; k < 2; ++k)
            for (int c : {1, 0}) {  // camera 7 is store camera 1, camera 9 store camera 0
                olm.push_back(j); okf.push_back(k); ocam.push_back(c);
                const double o = double(olm.size());
                res.insert(res.end(), {o, -o, 0.5 * o}); rho.insert(rho.end(), {2. * o, 3. * o});
            }
    std::vector<double> trim_r{1.5, 2.5}, trim_d{-1., 0.25}, gp_w{1.}, gp_r{-0.125};
    std::vector<uint8_t> rej_r{0, 1}, rej_d{1, 0};
    std::vector<int32_t> gp_lm{1}, gp_kf{0};
    kba_evaluate_out out{};
    out.obs_capacity = int32_t(olm.size()); out.n_obs = int32_t(olm.size()); out.n_gp = 1; out.failed = 0;
    for (int i = 0; i < 6; ++i) out.cost[i] = i + 1.;
    out.obs_lm = olm.data(); out.obs_kf = okf.data(); out.obs_cam = ocam.data(); out.residual = res.data(); out.rho = rho.data();
    out.trim_repr = trim_r.data(); out.trim_depth = trim_d.data(); out.rejected_repr = rej_r.data(); out.rejected_depth = rej_d.data();
    out.gp_lm = gp_lm.data(); out.gp_kf = gp_kf.data(); out.gp_weight = gp_w.data(); out.gp_residual = gp_r.data();
    const auto e = keyEvaluation(kfs, lm_ids, track_cams, out);
    CHECK(e.residuals.size() == 8 && e.landmarks.size() == 2 && !e.landmarks.count(11));
    const auto& r = e.residuals.at(std::make_tuple(LandmarkId(12), KeyframeId(200), CameraId(9)));  // the last observation
    CHECK(r.u == 8. && r.v == -8. && r.depth == 4. && r.rho_reprojection == 16. && r.rho_depth == 24.);
    const auto& r0 = e.residuals.at(std::make_tuple(LandmarkId(10), KeyframeId(100), CameraId(7)));
    CHECK(r0.u == 1. && r0.rho_depth == 3.);
    CHECK(e.landmarks.at(12).reprojection == 2.5 && e.landmarks.at(12).rejected_reprojection && !e.landmarks.at(12).rejected_depth);
    CHECK(e.landmarks.at(10).depth == -1. && e.landmarks.at(10).rejected_depth);
    CHECK(e.ground_plane.size() == 1 && e.ground_plane.at(12) == -0.125);
    CHECK(e.cost_reprojection == 1. && e.cost_plane_chain == 5. && e.cost_total == 6. && !e.failed);
    // an output in another order is refused
    std::swap(ocam[0], ocam[1]);
    bool refused = false;
    try { keyEvaluation(kfs, lm_ids, track_cams, out); } catch (const std::runtime_error&) { refused = true; }
    CHECK(refused);
    std::swap(ocam[0], ocam[1]);
    out.n_obs -= 1;
    refused = false;
    try { keyEvaluation(kfs, lm_ids, track_cams, out); } catch (const std::runtime_error&) { refused = true; }
    CHECK(refused);
    std::printf("%d failed checks\n", g_fail);
    return g_fail ? 1 : 0;
}

int main(int argc, char** argv) {
    std::setvbuf(stdout, nullptr, _IOLBF, 0);
    if (argc > 1 && std::strcmp(argv[1], "host") == 0) return host_mode();
    const int n_kf = 10;
    std::vector<Eigen::Vector3d> lms;
    for (int i = 0; i < 160; ++i) lms.push_back(Eigen::Vector3d(-3. + 0.041 * ((i * 37) % 151), -1.5 + 0.023 * ((i * 53) % 131), 5. + 0.07 * ((i * 29) % 113)));
    std::vector<Eigen::Isometry3d> gt(n_kf);
    gt[0] = Eigen::Isometry3d::Identity();
    for (int k = 1; k < n_kf; ++k) { gt[k] = gt[k - 1]; gt[k].translate(Eigen::Vector3d(0.04 * (k % 3), 0.015, -0.3)); gt[k].rotate(Eigen::AngleAxisd(0.008, Eigen::Vector3d(0., 1., 0.))); }
    const Camera c0(600., Eigen::Vector2d(300., 200.), Eigen::Isometry3d::Identity());
    const Camera c1(600., Eigen::Vector2d(300., 200.), side());
    // camera 0 sees every landmark, camera 1 (half a metre to the side) every third one with the same feature point
    Tracklets t;
    std::map<LandmarkId, CameraIds> lookup;
    for (int k = 0; k < n_kf; ++k) t.stamps.push_back(k);
    for (size_t i = 0; i < lms.size(); ++i) {
        Tracklet tr;
        tr.id = i;
        for (int k = 0; k < n_kf; ++k) {
            const Eigen::Vector3d lm_cam = gt[k] * lms[i];
            Eigen::Vector3d proj = c0.getIntrinsicMatrix() * lm_cam;
            proj /= proj[2];
            const float du = 0.3f * float((int(i) * 7 + k * 3) % 5 - 2), dv = 0.3f * float((int(i) * 3 + k * 5) % 5 - 2);
            tr.feature_points.push_back(FeaturePoint(float(proj[0]) + du, float(proj[1]) + dv, (i % 3 == 0) ? float(lm_cam[2]) + 0.01f : -1.f));
        }
        t.tracks.push_back(tr);
        lookup[i] = i % 3 ? CameraIds{0} : CameraIds{0, 1};
    }
    BundleAdjusterKeyframes a;
    a.set_solver_time(20.);
    int evaluated = 0;
    size_t max_obs = 0;
    double max_diff = 0.;
    for (int k = 0; k < n_kf; ++k) {
        Eigen::Isometry3d start = gt[k];
        if (k >= 2) start.translate(Eigen::Vector3d(0.02, -0.015, 0.03));
        const auto fix = k == 0 ? Keyframe::FixationStatus::Pose : (k == 1 ? Keyframe::FixationStatus::Scale : Keyframe::FixationStatus::None);
        std::map<CameraId, Camera::Ptr> cams{{0, std::make_shared<Camera>(c0)}, {1, std::make_shared<Camera>(c1)}};
        a.push(Keyframe(k, t, cams, lookup, start, fix));
        if (k < 3) continue;
        a.deactivateKeyframes(3, 4, 8);
        const std::string rep = a.solve();
        if (rep.find("device-resident") == std::string::npos) continue;
        // the state before the evaluation
        std::map<KeyframeId, std::array<double, 7>> poses;
        for (const auto& id : a.active_keyframe_ids_) poses[id] = a.keyframes_.at(id)->pose_;
        const auto selected = a.selected_landmark_ids_;
        a.evaluateResiduals();
        const auto& e = a.last_evaluation_;
        ++evaluated;
        CHECK(a.selected_landmark_ids_ == selected);
        for (const auto& id : a.active_keyframe_ids_) CHECK(a.keyframes_.at(id)->pose_ == poses[id]);
        // one residual per measurement of a selected landmark in an active keyframe, each from the host's state
        size_t n = 0;
        double c_r = 0., c_d = 0.;
        const double b_r = a.outlier_rejection_options_.reprojection_thres * a.outlier_rejection_options_.reprojection_thres;
        for (const auto lm : a.selected_landmark_ids_) {
            double m_r = -1.;
            const Landmark& L = *a.landmarks_.at(lm);
            for (const auto& kid : a.active_keyframe_ids_) {
                const Keyframe& kf = *a.keyframes_.at(kid);
                const auto it = kf.measurements_.find(lm);
                if (it == kf.measurements_.end()) continue;
                for (const auto& cm : it->second) {
                    ++n;
                    const auto rit = e.residuals.find(std::make_tuple(lm, kid, cm.first));
                    CHECK(rit != e.residuals.end());
                    if (rit == e.residuals.end()) continue;
                    const Camera& cam = *kf.cameras_.at(cm.first);
                    const Eigen::Vector3d pc = convert(cam.pose_camera_vehicle) * (kf.getEigenPose() * Eigen::Vector3d(L.pos.data()));
                    const double u = cam.focal_length * pc[0] / pc[2] + cam.principal_point[0] - double(cm.second.u);
                    const double v = cam.focal_length * pc[1] / pc[2] + cam.principal_point[1] - double(cm.second.v);
                    const double d = cm.second.d > 0.f ? pc[2] - double(cm.second.d) : 0.;
                    const auto& r = rit->second;
                    const double diff = std::max({std::fabs(r.u - u), std::fabs(r.v - v), std::fabs(r.depth - d)});
                    max_diff = std::max(max_diff, diff);
                    CHECK(diff <= 1e-9);
                    const double s = r.u * r.u + r.v * r.v;
                    CHECK(std::fabs(r.rho_reprojection - L.weight * b_r * std::log1p(s / b_r)) <= 1e-9 * (1. + r.rho_reprojection));
                    c_r += 0.5 * r.rho_reprojection; c_d += 0.5 * r.rho_depth;
                    m_r = std::max(m_r, std::sqrt(s));
                }
            }
            CHECK(e.landmarks.count(lm) && std::fabs(e.landmarks.at(lm).reprojection - m_r) <= 1e-12 * (1. + m_r));
        }
        CHECK(n == e.residuals.size() && e.landmarks.size() == a.selected_landmark_ids_.size());
        CHECK(std::fabs(e.cost_reprojection - c_r) <= 1e-10 * c_r && std::fabs(e.cost_depth - c_d) <= 1e-10 * (1. + c_d));
        CHECK(!e.failed && e.cost_total > 0.);
        max_obs = std::max(max_obs, n);
    }
    CHECK(evaluated >= 5);
    // switched off: the facade refuses, naming the reason
    a.set_persistent_window(false);
    CHECK(thrown(a).find("persistent window is off") != std::string::npos);
    std::printf("evaluateResiduals: %d windows evaluated, up to %zu residuals, max difference to the host %.3g\n", evaluated, max_obs, max_diff);
    std::printf("%d failed checks\n", g_fail);
    return g_fail ? 1 : 0;
}
