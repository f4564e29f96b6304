// limo's keyframe selection through the facade -- KeyframeSelector with KeyframeRejectionSchemeFlow, KeyframeSelectionSchemePose
// and KeyframeSparsificationSchemeTime (mono_lidar.cpp:447-453), select({frame}, active keyframes) on every frame
// (mono_lidar.cpp:219-220) -- against kba_track_frame_flow on the device-resident store.  The drive comes from a file that
// tests/keyframe_drive.py writes; the buffer holds the last `window` selected frames.
//   reference    the reference's KeyframeSelector.process test (keyframe_bundle_adjustment.cpp:613-647), restated.
//   host FILE    prints per frame `F k n_matched flow_sum mean_flow_sq flow pose time selected`, the two doubles as the hex of
//                their bits, the quantities of the flow scheme against the newest keyframe (-1 0 0 with an empty buffer) and each
//                scheme's isUsable against the buffer.  No GPU needed.
//   device FILE  mirrors every selected frame into a kba_track (keyframe i in slot i % (window + 2)) and, at every frame,
//                checks kba_track_frame_flow against the facade's flow scheme bit for bit and the selection composed from its
//                verdict against KeyframeSelector::select.
//   bench FILE   prints the median / p90 time (ms) of the facade's select() and of the flow scheme's walk alone
//                (scripts/keyframe_flow_bench.py).
#include <algorithm>
#include <chrono>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <string>
#include <vector>

#include "kba_b200.h"
#include "keyframe_bundle_adjustment/keyframe_selector.hpp"

using namespace keyframe_bundle_adjustment;
static int g_fail = 0;
#define CHECK(c) do { if (!(c)) { std::printf("CHECK FAILED %s:%d: %s\n", __FILE__, __LINE__, #c); ++g_fail; } } while (0)

struct Meas { int lm, cam; float u, v; };
struct FrameIn { TimestampNSec ts; Pose pose; double thr; std::vector<Meas> meas; };
struct Drive {
    std::vector<double> intr, cam_pose;
    int window = 0, n_lm = 0;
    double critical = 0, time_sec = 0;
    std::vector<FrameIn> frames;
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
    if (!word("params")) return false;
    dr.window = (int)num(); dr.critical = num(); dr.time_sec = num();
    if (!word("landmarks")) return false;
    dr.n_lm = (int)num();
    if (!word("frames")) return false;
    const int n = (int)num();
    for (int k = 0; k < n; ++k) {
        FrameIn fr;
        if (!word("f")) return false;
        f >> tok; fr.ts = std::strtoull(tok.c_str(), nullptr, 10);
        const int m = (int)num();
        for (int q = 0; q < 7; ++q) fr.pose[q] = num();
        fr.thr = num();
        for (int i = 0; i < m; ++i) {
            Meas e;
            e.lm = (int)num(); e.cam = (int)num(); e.u = (float)num(); e.v = (float)num();
            fr.meas.push_back(e);
        }
        dr.frames.push_back(fr);
    }
    return bool(f);
}

static unsigned long long bits(double x) { unsigned long long b; std::memcpy(&b, &x, 8); return b; }

static double pct(std::vector<double> v, double q) {
    std::sort(v.begin(), v.end());
    return v.empty() ? 0. : v[std::min(v.size() - 1, size_t(q * double(v.size())))];
}

// The reference's KeyframeSelector.process (keyframe_bundle_adjustment.cpp:613-647): one time scheme of 0.5 s, a buffer with
// frames at 0 and 10000 ns; a frame 1 s after the newer one is kept, one 0.25 s after it is not, by the scheme and by select().
static int reference_test() {
    const double dt = 0.5;
    auto make = [](TimestampNSec ts) { return std::make_shared<Keyframe>(ts, Tracklets{}, Camera::Ptr(), Eigen::Isometry3d::Identity()); };
    std::map<KeyframeId, Keyframe::Ptr> buffer{{0, make(0)}, {1, make(10000)}};
    KeyframeSparsificationSchemeBase::ConstPtr time_scheme = std::make_shared<KeyframeSparsificationSchemeTime>(dt);
    KeyframeSelector s;
    s.addScheme(time_scheme);
    const TimestampNSec late = 10000 + convert(TimestampSec(2. * dt)), early = 10000 + convert(TimestampSec(dt / 2.));
    const Keyframe::Ptr a = make(late), b = make(early);
    CHECK(time_scheme->isUsable(a, buffer));
    CHECK(!time_scheme->isUsable(b, buffer));
    const KeyframeSelector::Keyframes kept = s.select({a, b}, buffer);
    CHECK(kept.size() == 1 && (*kept.begin())->timestamp_ == late);
    std::printf("%d failed checks\n", g_fail);
    return g_fail ? 1 : 0;
}

static int run(const Drive& dr, const std::string& mode) {
    const int n_cam = (int)dr.intr.size() / 3, W = dr.window, n_slots = W + 2;
    const auto pose_scheme = KeyframeSelectionSchemePose::createConst(dr.critical);
    const auto time_scheme = KeyframeSparsificationSchemeTime::createConst(dr.time_sec);
    std::map<KeyframeId, Keyframe::Ptr> buffer;
    std::map<KeyframeId, int> slot_of;  // selected frame -> its keyframe slot in the track
    kba_handle* h = nullptr;
    kba_track* t = nullptr;
    std::vector<char> has_slot(dr.n_lm, 0);
    if (mode == "device") {
        size_t total = 0, most = 1;
        for (const auto& fr : dr.frames) { total += fr.meas.size(); most = std::max(most, fr.meas.size()); }
        CHECK(kba_create(&h, 0) == KBA_OK);
        kba_track_caps caps{n_slots, dr.n_lm, (int32_t)total, std::min(W + 1, 30), 64, (int32_t)most, 0, 0};
        CHECK(kba_track_create(h, &caps, n_cam, dr.intr.data(), dr.cam_pose.data(), &t) == KBA_OK);
        if (!t) { std::printf("%s\n", kba_last_error()); return 1; }
    }
    using clk = std::chrono::steady_clock;
    auto ms = [](clk::time_point t0) { return std::chrono::duration<double, std::milli>(clk::now() - t0).count(); };
    std::vector<double> t_select, t_flow;
    size_t n_sel = 0, n_nan = 0, n_checked = 0;
    int n_kf = 0;
    for (size_t k = 0; k < dr.frames.size(); ++k) {
        const FrameIn& fr = dr.frames[k];
        Keyframe::Ptr f(new Keyframe());
        f->timestamp_ = fr.ts; f->pose_ = fr.pose; f->is_active_ = false; f->fixation_status_ = Keyframe::FixationStatus::None;
        for (const Meas& m : fr.meas) f->measurements_[m.lm][m.cam] = Measurement(m.u, m.v, -1.f);
        const auto flow_scheme = KeyframeRejectionSchemeFlow::createConst(fr.thr);
        KeyframeSelector selector;
        selector.addScheme(flow_scheme); selector.addScheme(pose_scheme); selector.addScheme(time_scheme);
        KeyframeRejectionSchemeFlow::Flow q;
        q.n_matched = -1;
        Keyframe::Ptr last;
        if (!buffer.empty()) {
            last = buffer.begin()->second;
            for (const auto& el : buffer)
                if (last->timestamp_ < el.second->timestamp_) last = el.second;
            auto t0 = clk::now();
            q = KeyframeRejectionSchemeFlow::flow(*f, *last);
            t_flow.push_back(ms(t0));
        }
        const bool v_flow = flow_scheme->isUsable(f, buffer), v_pose = pose_scheme->isUsable(f, buffer), v_time = time_scheme->isUsable(f, buffer);
        auto t0 = clk::now();
        const bool sel = !selector.select({f}, buffer).empty();
        t_select.push_back(ms(t0));
        if (mode == "host")
            std::printf("F %zu %d %016llx %016llx %d %d %d %d\n", k, q.n_matched, bits(q.flow_sum), bits(q.mean_flow_sq), v_flow, v_pose, v_time, sel);
        if (t && last) {  // the device's flow against the newest keyframe's slot, then limo's composition with its verdict
            std::vector<int32_t> lm, cam, match(fr.meas.size() + 1);
            std::vector<float> u, v;
            for (const Meas& m : fr.meas)
                if (has_slot[m.lm]) { lm.push_back(m.lm); cam.push_back(m.cam); u.push_back(m.u); v.push_back(m.v); }
            kba_flow_request rq{slot_of.at(last->timestamp_), (int32_t)lm.size(), lm.data(), cam.data(), u.data(), v.data(), fr.thr};
            kba_flow_out o{};
            o.match = match.data();
            const int rc = kba_track_frame_flow(t, &rq, &o);
            CHECK(rc == KBA_OK);
            if (rc != KBA_OK) { std::printf("%s\n", kba_last_error()); break; }
            CHECK(o.n_matched == q.n_matched);
            CHECK(bits(o.flow_sum) == bits(q.flow_sum));
            CHECK(bits(o.mean_flow_sq) == bits(q.mean_flow_sq));
            const bool d_flow = f->measurements_.empty() ? false : o.usable != 0;
            CHECK(d_flow == v_flow);
            // select({f}, buffer) for one frame: not rejected, and selected by the pose scheme or kept by the time scheme (both
            // also test against the empty map of frames accepted before: pose false, time true)
            CHECK((d_flow && (v_pose || v_time)) == sel);
            n_nan += o.n_matched == 0;
            ++n_checked;
        }
        if (sel) {
            ++n_sel;
            if (t) {
                const int slot = n_kf % n_slots;
                if (n_kf >= n_slots) CHECK(kba_track_drop_keyframe(t, slot) == KBA_OK);
                std::vector<int32_t> lm, cam;
                std::vector<float> u, v, d;
                for (const Meas& m : fr.meas) { lm.push_back(m.lm); cam.push_back(m.cam); u.push_back(m.u); v.push_back(m.v); d.push_back(-1.f); }
                CHECK(kba_track_push_keyframe(t, slot, fr.pose.data(), nullptr, (int32_t)lm.size(), lm.data(), cam.data(), u.data(), v.data(),
                                              d.data()) == KBA_OK);
                for (const Meas& m : fr.meas) has_slot[m.lm] = 1;
                slot_of[fr.ts] = slot;
            }
            ++n_kf;
            buffer[fr.ts] = f;
            while ((int)buffer.size() > W) buffer.erase(buffer.begin());
        }
    }
    if (mode == "bench")
        std::printf("{\"window\": %d, \"frames\": %zu, \"facade_select_ms\": [%.4f, %.4f], \"facade_flow_ms\": [%.4f, %.4f]}\n", W,
                    dr.frames.size(), pct(t_select, 0.5), pct(t_select, 0.9), pct(t_flow, 0.5), pct(t_flow, 0.9));
    if (t) {
        std::printf("window %d: %zu frames checked, %zu selected, %zu without a match\n", W, n_checked, n_sel, n_nan);
        CHECK(n_checked + 1 == dr.frames.size() && n_nan > 0);
        kba_track_destroy(t);
        kba_destroy(h);
    }
    return 0;
}

int main(int argc, char** argv) {
    std::setvbuf(stdout, nullptr, _IOLBF, 0);
    if (argc == 2 && std::string(argv[1]) == "reference") return reference_test();
    if (argc != 3) { std::printf("usage: %s reference | host|device|bench DRIVE_FILE\n", argv[0]); return 2; }
    Drive dr;
    if (!read_drive(argv[2], dr)) { std::printf("cannot read %s\n", argv[2]); return 2; }
    run(dr, argv[1]);
    if (std::string(argv[1]) == "device") std::printf("%d failed checks\n", g_fail);
    return g_fail ? 1 : 0;
}
