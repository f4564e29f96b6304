// The landmark creation of BundleAdjusterKeyframes::push() (calculateLandmark(kf, id) with a depth, calculateLandmark(id) without)
// against kba_track_create_landmarks on the device-resident store.  The drive comes from a file that tests/create_drive.py writes
// (cameras, window size, then per keyframe its pose and measurements, doubles as C99 hex floats):
//   host FILE    pushes every keyframe through push() and keeps the newest `window` keyframes active (deactivateKeyframes); after
//                each push it prints, for every landmark the keyframe measures that push() had to create and for every fourth
//                landmark it measures that already existed (what the facade's calculateLandmark gives for it now: a re-creation
//                over all active keyframes), one line `push id created has_depth x y z` with the position in hex.  No GPU needed.
//   device FILE  does the same and mirrors every keyframe into a kba_track (the slot of a keyframe that left the window is dropped
//                and reused); after each push kba_track_create_landmarks for the same landmarks must return the facade's flags
//                and positions bit for bit (NaN where the facade has NaN).
//   bench FILE   prints the median / p90 time of the facade's push() (ms), which creates the keyframe's new landmarks on the host
//                (scripts/create_landmarks_bench.py).
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

using namespace keyframe_bundle_adjustment;
static int g_fail = 0;
#define CHECK(c) do { if (!(c)) { std::printf("CHECK FAILED %s:%d: %s\n", __FILE__, __LINE__, #c); ++g_fail; } } while (0)

struct Meas { int lm, cam; float u, v, d; };
struct Push { unsigned long id; Pose pose; std::vector<Meas> meas; };
struct Drive {
    std::vector<double> intr, cam_pose;  // [n_cam * 3], [n_cam * 7]
    int window = 0, n_lm = 0;
    std::vector<Push> pushes;
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
    return bool(f);
}

static uint64_t bits(double x) { uint64_t b; std::memcpy(&b, &x, 8); return b; }
static bool same(double a, double b) { return (std::isnan(a) && std::isnan(b)) || bits(a) == bits(b); }
static double pct(std::vector<double> v, double q) {
    std::sort(v.begin(), v.end());
    return v.empty() ? 0. : v[std::min(v.size() - 1, size_t(q * double(v.size())))];
}

// what push() (and, for a landmark that exists, calculateLandmark) gives for one landmark of the pushed keyframe
struct Created { int lm; bool created, has_depth; double pos[3]; };

static int run(const Drive& dr, const std::string& mode) {
    const int n_cam = (int)dr.intr.size() / 3, W = dr.window;
    std::map<CameraId, Camera::Ptr> cams;
    for (int c = 0; c < n_cam; ++c) {
        auto cam = std::make_shared<Camera>(dr.intr[3 * c], Eigen::Vector2d(dr.intr[3 * c + 1], dr.intr[3 * c + 2]), Eigen::Isometry3d::Identity());
        for (int q = 0; q < 7; ++q) cam->pose_camera_vehicle[q] = dr.cam_pose[7 * c + q];  // the drive's extrinsics, not a round trip
        cams[c] = cam;
    }
    BundleAdjusterKeyframes ba;
    kba_handle* h = nullptr;
    kba_track* t = nullptr;
    const int n_slots = W + 2;
    if (mode == "device") {
        size_t total = 0;
        for (const auto& p : dr.pushes) total += p.meas.size();
        CHECK(kba_create(&h, 0) == KBA_OK);
        kba_track_caps caps{n_slots, dr.n_lm, (int32_t)total, std::min(W + 1, 30), 64, 64, 0, 0};
        CHECK(kba_track_create(h, &caps, n_cam, dr.intr.data(), dr.cam_pose.data(), &t) == KBA_OK);
        if (!t) { std::printf("%s\n", kba_last_error()); return 1; }
    }
    using clk = std::chrono::steady_clock;
    std::vector<double> t_push;
    size_t n_checked = 0, n_created = 0, n_depth = 0, n_nan = 0;
    for (size_t k = 0; k < dr.pushes.size(); ++k) {
        const Push& p = dr.pushes[k];
        Keyframe kf;
        kf.timestamp_ = p.id; kf.cameras_ = cams; kf.fixation_status_ = Keyframe::FixationStatus::None; kf.pose_ = p.pose;
        kf.is_active_ = true;
        for (const Meas& m : p.meas) kf.measurements_[m.lm][m.cam] = Measurement(m.u, m.v, m.d);
        std::vector<int> fresh, again;  // landmarks push() must create; every fourth one that exists already
        for (const auto& el : kf.measurements_) {
            if (!ba.landmarks_.count(el.first)) fresh.push_back((int)el.first);
            else if (el.first % 4 == 0) again.push_back((int)el.first);
        }
        const auto t0 = clk::now();
        ba.push(kf);
        t_push.push_back(std::chrono::duration<double, std::milli>(clk::now() - t0).count());
        std::vector<Created> out;
        for (int id : fresh) {
            Created c{id, false, false, {NAN, NAN, NAN}};
            auto it = ba.landmarks_.find(id);
            if (it != ba.landmarks_.end()) { c.created = true; c.has_depth = it->second->has_measured_depth; std::memcpy(c.pos, it->second->pos.data(), 24); }
            out.push_back(c);
        }
        const Keyframe& stored = *ba.keyframes_.at(p.id);
        for (int id : again) {  // push()'s rule for a landmark it creates, through the public calculateLandmark overloads
            bool depth = false;
            for (const auto& cm : stored.measurements_.at(id)) depth |= cm.second.d >= 0;
            BundleAdjusterKeyframes::v3 pos;
            Created c{id, false, depth, {NAN, NAN, NAN}};
            c.created = depth ? ba.calculateLandmark(stored, id, pos) : ba.calculateLandmark(id, pos);
            if (c.created) for (int q = 0; q < 3; ++q) c.pos[q] = pos[q];
            out.push_back(c);
        }
        std::sort(out.begin(), out.end(), [](const Created& a, const Created& b) { return a.lm < b.lm; });
        if (mode == "host")
            for (const Created& c : out)
                std::printf("%lu %d %d %d %a %a %a\n", p.id, c.lm, int(c.created), int(c.has_depth), c.pos[0], c.pos[1], c.pos[2]);
        if (t) {
            // mirror the keyframe: the slot of the keyframe that left the window is dropped, measurements in (id, camera) order
            const int slot = int(p.id % n_slots);
            if (k >= size_t(W) + 1) CHECK(kba_track_drop_keyframe(t, int(dr.pushes[k - W - 1].id % n_slots)) == KBA_OK);
            std::vector<int32_t> lm, cam;
            std::vector<float> u, v, d;
            for (const auto& el : kf.measurements_)
                for (const auto& cm : el.second) {
                    lm.push_back((int32_t)el.first); cam.push_back((int32_t)cm.first);
                    u.push_back(cm.second.u); v.push_back(cm.second.v); d.push_back(cm.second.d);
                }
            CHECK(kba_track_push_keyframe(t, slot, p.pose.data(), nullptr, (int32_t)lm.size(), lm.data(), cam.data(), u.data(), v.data(), d.data()) == KBA_OK);
            std::vector<int32_t> kf_slot, lm_slot;
            for (KeyframeId id : ba.active_keyframe_ids_) kf_slot.push_back(int32_t(id % n_slots));
            for (const Created& c : out) lm_slot.push_back(c.lm);
            std::vector<double> pos(3 * out.size() + 3);
            std::vector<uint8_t> flags(out.size() + 1);
            kba_create_request rq{(int32_t)kf_slot.size(), (int32_t)kf_slot.size() - 1, (int32_t)lm_slot.size(), 0, kf_slot.data(), lm_slot.data()};
            kba_create_out o{pos.data(), flags.data()};
            const int rc = kba_track_create_landmarks(t, &rq, &o);
            CHECK(rc == KBA_OK);
            if (rc != KBA_OK) { std::printf("%s\n", kba_last_error()); break; }
            for (size_t i = 0; i < out.size(); ++i) {
                const Created& c = out[i];
                CHECK(flags[i] == ((c.created ? 1 : 0) | (c.has_depth ? 2 : 0)));
                for (int q = 0; q < 3; ++q) CHECK(same(pos[3 * i + q], c.pos[q]));
                ++n_checked; n_created += c.created; n_depth += c.has_depth; n_nan += c.created && std::isnan(c.pos[0]);
            }
        }
        if (k >= 1) ba.deactivateKeyframes(-1, W, W);  // the newest W keyframes stay active
    }
    if (mode == "bench")
        std::printf("{\"window\": %d, \"pushes\": %zu, \"facade_push_ms\": [%.4f, %.4f]}\n", W, dr.pushes.size(), pct(t_push, 0.5), pct(t_push, 0.9));
    if (t) {
        std::printf("window %d: %zu landmark requests checked over %zu pushes, %zu created (%zu from a depth, %zu NaN)\n", W, n_checked,
                    dr.pushes.size(), n_created, n_depth, n_nan);
        CHECK(n_created > 0 && n_depth > 0 && n_created < n_checked);
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
