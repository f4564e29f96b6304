// adjustPoseOnly() of the facade on the device-resident store (kba_track_adjust_pose) against a twin adjuster that rebuilds every
// window (set_persistent_window(false)).  A drive: every frame is tracked with adjustPoseOnly() before it becomes a keyframe, then
// pushed (with the same initial pose into both adjusters) and the window solved.  Checks:
//   - the tracked frame poses agree with the twin's to 1e-9 m, with the same iteration counts in the report;
//   - the tracked adjustPoseOnly() uploads less than the rebuild path;
//   - one solve() with the persistent window switched off and back on: the landmarks that solve wrote on the host reach the store,
//     so every later solve() stays bit-identical to the twin.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "keyframe_bundle_adjustment/bundle_adjuster_keyframes.hpp"

using namespace keyframe_bundle_adjustment;
static int g_fail = 0;
#define CHECK(c) do { if (!(c)) { std::printf("CHECK FAILED %s:%d: %s\n", __FILE__, __LINE__, #c); ++g_fail; } } while (0)

// the iteration counts of every inner solve, as the report prints them
static std::vector<int> iterations(const std::string& report) {
    std::vector<int> out;
    const std::string key = ", iterations ";
    for (size_t p = report.find(key); p != std::string::npos; p = report.find(key, p + 1)) out.push_back(std::atoi(report.c_str() + p + key.size()));
    return out;
}

int main() {
    std::setvbuf(stdout, nullptr, _IOLBF, 0);
    const int n_kf = 16, toggle = 8;
    std::vector<Eigen::Vector3d> lms;
    for (int i = 0; i < 160; ++i) lms.push_back(Eigen::Vector3d(-3. + 0.041 * ((i * 37) % 151), -1.5 + 0.023 * ((i * 53) % 131), 5. + 0.07 * ((i * 29) % 113)));
    std::vector<Eigen::Isometry3d> gt(n_kf);
    gt[0] = Eigen::Isometry3d::Identity();
    for (int k = 1; k < n_kf; ++k) { gt[k] = gt[k - 1]; gt[k].translate(Eigen::Vector3d(0.04 * (k % 3), 0.015, -0.3)); gt[k].rotate(Eigen::AngleAxisd(0.008, Eigen::Vector3d(0., 1., 0.))); }
    const Camera proto(600., Eigen::Vector2d(300., 200.), Eigen::Isometry3d::Identity());
    Tracklets ts;
    for (int k = 0; k < n_kf; ++k) ts.stamps.push_back(k);
    ts.tracks.resize(lms.size());
    for (size_t i = 0; i < lms.size(); ++i) {
        ts.tracks[i].id = i;
        for (int k = 0; k < n_kf; ++k) {
            const Eigen::Vector3d lm_cam = gt[k] * lms[i];
            Eigen::Vector3d proj = proto.getIntrinsicMatrix() * lm_cam;
            proj /= proj[2];
            const float du = 0.3f * float((int(i) * 7 + k * 3) % 5 - 2), dv = 0.3f * float((int(i) * 3 + k * 5) % 5 - 2);  // deterministic pixel noise
            ts.tracks[i].feature_points.push_back(FeaturePoint(float(proj[0]) + du, float(proj[1]) + dv, (i % 3 == 0) ? float(lm_cam[2]) : -1.f));
        }
    }
    BundleAdjusterKeyframes a, b;
    b.set_persistent_window(false);
    a.set_solver_time(20.); b.set_solver_time(20.);
    auto cam = [] { return std::make_shared<Camera>(600., Eigen::Vector2d(300., 200.), Eigen::Isometry3d::Identity()); };
    long long up_a = 0, up_b = 0;
    int tracked = 0, frames = 0;
    double max_dt = 0.;
    for (int k = 0; k < n_kf; ++k) {
        Eigen::Isometry3d start = gt[k];
        if (k >= 2) start.translate(Eigen::Vector3d(0.02, -0.015, 0.03));
        const auto fix = k == 0 ? Keyframe::FixationStatus::Pose : (k == 1 ? Keyframe::FixationStatus::Scale : Keyframe::FixationStatus::None);
        if (k >= 4) {  // track the frame before it becomes a keyframe
            Keyframe fa(k, ts, cam(), start, fix), fb(k, ts, cam(), start, fix);
            const std::string ra = a.adjustPoseOnly(fa), rb = b.adjustPoseOnly(fb);
            double dt = 0.;
            for (int i = 4; i < 7; ++i) dt += (fa.pose_[i] - fb.pose_[i]) * (fa.pose_[i] - fb.pose_[i]);
            dt = std::sqrt(dt);
            max_dt = std::max(max_dt, dt);
            CHECK(dt <= 1e-9);
            CHECK(!iterations(ra).empty() && iterations(ra) == iterations(rb));
            CHECK(rb.find("device-resident") == std::string::npos);
            ++frames;
            if (ra.find("device-resident") != std::string::npos) {
                ++tracked;
                up_a += a.lastSolveUploadBytes(); up_b += b.lastSolveUploadBytes();
            }
        }
        for (BundleAdjusterKeyframes* adj : {&a, &b}) adj->push(Keyframe(k, ts, cam(), start, fix));
        if (k < 3) continue;
        for (BundleAdjusterKeyframes* adj : {&a, &b}) adj->deactivateKeyframes(3, 4, 8);
        if (k == toggle) a.set_persistent_window(false);  // one rebuild-path solve on the persistent adjuster
        a.solve(); b.solve();
        if (k == toggle) a.set_persistent_window(true);
        bool same = true;
        for (const auto& id : a.active_keyframe_ids_) same = same && a.keyframes_.at(id)->pose_ == b.keyframes_.at(id)->pose_;
        for (const auto& id : a.selected_landmark_ids_) same = same && a.landmarks_.at(id)->pos == b.landmarks_.at(id)->pos;
        CHECK(same);
        CHECK(a.active_keyframe_ids_ == b.active_keyframe_ids_ && a.selected_landmark_ids_ == b.selected_landmark_ids_);
    }
    CHECK(frames == n_kf - 4);
    CHECK(tracked >= frames - 1);  // the frame after the toggle may see a landmark the store has no slot for yet: rebuild path
    CHECK(up_a > 0 && up_a < up_b);
    std::printf("adjustPoseOnly: %d of %d frames tracked, max pose difference %.3g m, upload %lld B per frame (rebuild path %lld B)\n",
                tracked, frames, max_dt, tracked ? up_a / tracked : 0, tracked ? up_b / tracked : 0);
    std::printf("%d failed checks\n", g_fail);
    return g_fail ? 1 : 0;
}
