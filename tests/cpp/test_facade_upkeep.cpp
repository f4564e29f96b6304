// The window upkeep of limo's keyframe step through the facade -- deactivateKeyframes(3, 4, W), updateLabels and the AddDepth
// scheme with 50 ground landmarks per keyframe (mono_lidar.cpp:413-429) -- against kba_track_deactivate_keyframes and
// kba_track_depth_costs on the device-resident store.  The drive comes from a file that tests/upkeep_drive.py writes (the format
// of tests/cpp/test_facade_create.cpp plus a line `ground N id ...`).  At every push the facade pushes the keyframe; from the
// fourth push on it deactivates keyframes, labels the created landmarks (updateLabels) and runs the AddDepth scheme over the
// active landmarks that exist and pass a stand-in for the rejection schemes (id % 13 != 5):
//   host FILE    prints after each such step `D k ids` (active keyframes), `L k ids` (active landmarks) and `S k ids` (the
//                AddDepth selection).  No GPU needed.
//   device FILE  mirrors every keyframe into a kba_track (the slot of a keyframe that left the window is dropped and reused) and
//                creates its new landmarks there (kba_track_create_landmarks); then, before the facade deactivates, the device
//                deactivation of the same lists must give the facade's new active_keyframe_ids_ / active_landmark_ids_, and
//                std::partial_sort over the device costs, as the scheme ranks, must give the scheme's selection.
//   bench FILE   prints the median / p90 time (ms) of the facade's deactivateKeyframes() and of the scheme's getSelection()
//                (scripts/upkeep_bench.py).
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <string>
#include <vector>

#include "kba_b200.h"
#include "keyframe_bundle_adjustment/bundle_adjuster_keyframes.hpp"
#include "keyframe_bundle_adjustment/landmark_selection_schemes.hpp"

using namespace keyframe_bundle_adjustment;
static int g_fail = 0;
#define CHECK(c) do { if (!(c)) { std::printf("CHECK FAILED %s:%d: %s\n", __FILE__, __LINE__, #c); ++g_fail; } } while (0)

struct Meas { int lm, cam; float u, v, d; };
struct Push { unsigned long id; Pose pose; std::vector<Meas> meas; };
struct Drive {
    std::vector<double> intr, cam_pose;  // [n_cam * 3], [n_cam * 7]
    int window = 0, n_lm = 0;
    std::vector<Push> pushes;
    std::vector<char> ground;
};

static bool read_drive(const char* path, Drive& dr) {
    std::ifstream f(path);
    std::string tok;
    auto num = [&] { f >> tok; return std::strtod(tok.c_str(), nullptr); };
    auto word = [&](const char* w) { f >> tok; return tok == w; };
    if (!word("cams")) return false;
    const int n_cam = (int)num();
    for (int c = 0; c < n_cam; ++c) {
        for (int q = 0; q < 3; ++q) dr.intr.push_back(num());
        for (int q = 0; q < 7; ++q) dr.cam_pose.push_back(num());
    }
    if (!word("window")) return false;
    dr.window = (int)num();
    if (!word("landmarks")) return false;
    dr.n_lm = (int)num();
    if (!word("pushes")) return false;
    const int n_push = (int)num();
    for (int k = 0; k < n_push; ++k) {
        Push p;
        if (!word("kf")) return false;
        p.id = (unsigned long)num();
        const int n = (int)num();
        for (int q = 0; q < 7; ++q) p.pose[q] = num();
        for (int i = 0; i < n; ++i) {
            Meas m;
            m.lm = (int)num(); m.cam = (int)num();
            m.u = (float)num(); m.v = (float)num(); m.d = (float)num();
            p.meas.push_back(m);
        }
        dr.pushes.push_back(p);
    }
    if (!word("ground")) return false;
    dr.ground.assign(dr.n_lm, 0);
    const int n_ground = (int)num();
    for (int i = 0; i < n_ground; ++i) dr.ground[(int)num()] = 1;
    return bool(f);
}

static double pct(std::vector<double> v, double q) {
    std::sort(v.begin(), v.end());
    return v.empty() ? 0. : v[std::min(v.size() - 1, size_t(q * double(v.size())))];
}

template <typename Ids> static void print_ids(char tag, unsigned long k, const Ids& ids) {
    std::printf("%c %lu", tag, k);
    for (const auto& id : ids) std::printf(" %lu", (unsigned long)id);
    std::printf("\n");
}

static int run(const Drive& dr, const std::string& mode) {
    const int n_cam = (int)dr.intr.size() / 3, W = dr.window;
    std::map<CameraId, Camera::Ptr> cams;
    for (int c = 0; c < n_cam; ++c) {
        auto cam = std::make_shared<Camera>(dr.intr[3 * c], Eigen::Vector2d(dr.intr[3 * c + 1], dr.intr[3 * c + 2]), Eigen::Isometry3d::Identity());
        for (int q = 0; q < 7; ++q) cam->pose_camera_vehicle[q] = dr.cam_pose[7 * c + q];
        cams[c] = cam;
    }
    LandmarkSelectionSchemeAddDepth::Parameters p;  // mono_lidar.cpp:413-429
    auto gp_comparator = [](const Landmark::ConstPtr& lm) { return lm->is_ground_plane; };
    auto gp_sorter = [](const Measurement&, const Eigen::Vector3d& local) { return float(local.norm()); };
    for (int i = 0; i < W; ++i) p.params_per_keyframe.push_back(std::make_tuple(i, 50, gp_comparator, gp_sorter));
    const LandmarkSelectionSchemeAddDepth add_depth(p);

    BundleAdjusterKeyframes ba;
    kba_handle* h = nullptr;
    kba_track* t = nullptr;
    const int n_slots = W + 2;
    if (mode == "device") {
        size_t total = 0;
        for (const auto& ps : dr.pushes) total += ps.meas.size();
        CHECK(kba_create(&h, 0) == KBA_OK);
        kba_track_caps caps{n_slots, dr.n_lm, (int32_t)total, std::min(W + 1, 30), 64, 64, 0, 0};
        CHECK(kba_track_create(h, &caps, n_cam, dr.intr.data(), dr.cam_pose.data(), &t) == KBA_OK);
        if (!t) { std::printf("%s\n", kba_last_error()); return 1; }
    }
    using clk = std::chrono::steady_clock;
    auto ms = [](clk::time_point t0) { return std::chrono::duration<double, std::milli>(clk::now() - t0).count(); };
    std::vector<double> t_deact, t_depth;
    size_t steps = 0, by_rule = 0, by_window = 0, n_selected = 0, n_neg = 0;
    for (size_t k = 0; k < dr.pushes.size(); ++k) {
        const Push& ps = dr.pushes[k];
        Keyframe kf;
        kf.timestamp_ = ps.id; kf.cameras_ = cams; kf.fixation_status_ = Keyframe::FixationStatus::None; kf.pose_ = ps.pose;
        kf.is_active_ = true;
        for (const Meas& m : ps.meas) kf.measurements_[m.lm][m.cam] = Measurement(m.u, m.v, m.d);
        std::vector<int32_t> fresh;
        for (const auto& el : kf.measurements_)
            if (!ba.landmarks_.count(el.first)) fresh.push_back((int32_t)el.first);
        ba.push(kf);
        auto kf_slots = [&] {
            std::vector<int32_t> s;
            for (KeyframeId id : ba.active_keyframe_ids_) s.push_back(int32_t(id % n_slots));
            return s;
        };
        if (t) {  // mirror the keyframe and create its new landmarks on the store
            if (k >= size_t(n_slots)) CHECK(kba_track_drop_keyframe(t, int(dr.pushes[k - n_slots].id % n_slots)) == KBA_OK);
            std::vector<int32_t> lm, cam;
            std::vector<float> u, v, d;
            for (const auto& el : kf.measurements_)
                for (const auto& cm : el.second) {
                    lm.push_back((int32_t)el.first); cam.push_back((int32_t)cm.first);
                    u.push_back(cm.second.u); v.push_back(cm.second.v); d.push_back(cm.second.d);
                }
            CHECK(kba_track_push_keyframe(t, int(ps.id % n_slots), ps.pose.data(), nullptr, (int32_t)lm.size(), lm.data(), cam.data(), u.data(),
                                          v.data(), d.data()) == KBA_OK);
            std::vector<int32_t> ks = kf_slots();
            std::vector<double> pos(3 * fresh.size() + 3);
            std::vector<uint8_t> flags(fresh.size() + 1);
            kba_create_request rq{(int32_t)ks.size(), (int32_t)ks.size() - 1, (int32_t)fresh.size(), 0, ks.data(), fresh.data()};
            kba_create_out o{pos.data(), flags.data()};
            CHECK(kba_track_create_landmarks(t, &rq, &o) == KBA_OK);
        }
        if (k < 3) continue;
        // ---- deactivateKeyframes(3, 4, W): the device on the lists before, the facade's own call
        const std::vector<KeyframeId> kf_before(ba.active_keyframe_ids_.begin(), ba.active_keyframe_ids_.end());
        const std::vector<LandmarkId> lm_before(ba.active_landmark_ids_.begin(), ba.active_landmark_ids_.end());
        std::vector<uint8_t> kf_active(kf_before.size()), lm_active(lm_before.size() + 1);
        std::vector<int32_t> kf_common(kf_before.size());
        if (t) {
            std::vector<int32_t> ks = kf_slots(), ls(lm_before.begin(), lm_before.end());
            kba_deactivate_request rq{(int32_t)ks.size(), (int32_t)ls.size(), 3, 4, W, 0, ks.data(), ls.data()};
            kba_deactivate_out o{kf_active.data(), kf_common.data(), lm_active.data()};
            const int rc = kba_track_deactivate_keyframes(t, &rq, &o);
            CHECK(rc == KBA_OK);
            if (rc != KBA_OK) { std::printf("%s\n", kba_last_error()); break; }
        }
        auto t0 = clk::now();
        ba.deactivateKeyframes(3, 4, W);
        t_deact.push_back(ms(t0));
        if (t) {
            for (size_t i = 0; i < kf_before.size(); ++i) {
                CHECK(kf_active[i] == ba.active_keyframe_ids_.count(kf_before[i]));
                const int age = int(kf_before.size() - 1 - i);
                by_rule += !kf_active[i] && age <= W - 1;
                by_window += !kf_active[i] && age > W - 1;
            }
            for (size_t j = 0; j < lm_before.size(); ++j) CHECK(lm_active[j] == ba.active_landmark_ids_.count(lm_before[j]));
        }
        // ---- updateLabels: the created landmarks' labels (7: road, a ground label; 0: none)
        Tracklets ts;
        for (const auto& el : ba.landmarks_) {
            Tracklet tr;
            tr.id = el.first; tr.age = 0; tr.label = dr.ground[el.first] ? 7 : 0;
            ts.tracks.push_back(tr);
        }
        ba.updateLabels(ts, 0.9);
        // ---- AddDepth over the active landmarks that exist and pass the stand-in rejection
        std::map<LandmarkId, Landmark::ConstPtr> lms;
        for (const auto& el : ba.getActiveLandmarkConstPtrs())
            if (el.first % 13 != 5) lms.insert(el);
        const auto kfs = ba.getActiveKeyframeConstPtrs();
        t0 = clk::now();
        const std::set<LandmarkId> sel = add_depth.getSelection(lms, kfs);
        t_depth.push_back(ms(t0));
        ++steps;
        n_selected += sel.size();
        if (mode == "host") {
            print_ids('D', ps.id, ba.active_keyframe_ids_);
            print_ids('L', ps.id, ba.active_landmark_ids_);
            print_ids('S', ps.id, sel);
        }
        if (t) {
            std::vector<int32_t> ks = kf_slots(), elig;
            for (const auto& el : lms)
                if (el.second->is_ground_plane) elig.push_back((int32_t)el.first);
            const int cap = int(ks.size() * elig.size());
            std::vector<int32_t> off(ks.size() + 1), cand(cap + 1);
            std::vector<double> cost(cap + 1);
            kba_depth_request rq{(int32_t)ks.size(), (int32_t)elig.size(), cap, 0, ks.data(), elig.data()};
            kba_depth_out o{off.data(), cand.data(), cost.data()};
            const int rc = kba_track_depth_costs(t, &rq, &o);
            CHECK(rc == KBA_OK);
            if (rc != KBA_OK) { std::printf("%s\n", kba_last_error()); break; }
            std::set<LandmarkId> dsel;
            for (const auto& el : p.params_per_keyframe) {  // the scheme's ranking over the device's cost vectors
                const int ind = std::get<0>(el), wanted = std::get<1>(el);
                if (ind > int(ks.size()) - 1) continue;
                std::vector<std::pair<LandmarkId, double>> c;
                for (int i = off[ind]; i < off[ind + 1]; ++i) {
                    c.emplace_back((LandmarkId)elig[cand[i]], cost[i]);
                    n_neg += cost[i] == -std::numeric_limits<double>::max();
                }
                const int n = std::min(wanted, int(c.size()));
                std::partial_sort(c.begin(), c.begin() + n, c.end(), [](const auto& a, const auto& b) { return a.second < b.second; });
                for (int i = 0; i < n; ++i) dsel.insert(c[i].first);
            }
            CHECK(dsel == sel);
        }
    }
    if (mode == "bench")
        std::printf("{\"window\": %d, \"steps\": %zu, \"facade_deactivate_ms\": [%.4f, %.4f], \"facade_add_depth_ms\": [%.4f, %.4f]}\n", W,
                    steps, pct(t_deact, 0.5), pct(t_deact, 0.9), pct(t_depth, 0.5), pct(t_depth, 0.9));
    if (t) {
        std::printf("window %d: %zu steps, keyframes deactivated by the connection rule %zu, by the window %zu; %zu selected, "
                    "%zu -DBL_MAX costs\n", W, steps, by_rule, by_window, n_selected, n_neg);
        CHECK(steps > 0 && by_rule > 0 && by_window > 0 && n_neg > 0);
        kba_track_destroy(t);
        kba_destroy(h);
    }
    return 0;
}

int main(int argc, char** argv) {
    std::setvbuf(stdout, nullptr, _IOLBF, 0);
    if (argc != 3) { std::printf("usage: %s host|device|bench DRIVE_FILE\n", argv[0]); return 2; }
    Drive dr;
    if (!read_drive(argv[2], dr)) { std::printf("cannot read %s\n", argv[2]); return 2; }
    run(dr, argv[1]);
    if (std::string(argv[1]) == "device") std::printf("%d failed checks\n", g_fail);
    return g_fail ? 1 : 0;
}
