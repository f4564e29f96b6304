// The ranking LandmarkSelector::select applies to the chain's quantities -- the voxel scheme's rankBins (chooseNearLmIds,
// chooseMiddleLmIds with std::rand, chooseFarLmIds) and the AddDepth scheme's std::partial_sort over a keyframe's costs -- on
// cases that tests/test_track_rank.py writes, so that its Python restatement (and through it kba_track_rank_landmarks) is pinned to
// the facade and to libstdc++'s heap.
//   host FILE   for every case: std::srand(seed), rankBins, the AddDepth partial sorts as the scheme runs them, then the next
//               std::rand().  Prints `C k id:category ...` (category 0 near, 1 middle, 2 far, 3 AddDepth only, ascending id) and
//               `R k n_draws draw ...`: how many std::rand() values the ranking consumed and what they were.  No GPU needed.
//   device      limo's mono-lidar chain (cheirality, voxel 0.5 / 0.5 / 0.3 m, 40 / 15 m, 400 per bin, AddDepth 50 ground landmarks
//               per keyframe) on a 33-keyframe drive through the facade, 12- and 20-keyframe windows, mirrored into a kba_track
//               (keyframe slot = id, landmark slot = id; the facade's poses and positions go up before each step).  Before each
//               solve() std::srand is seeded identically for a standalone selector's host select() and for
//               kba_track_rank_landmarks with a std::rand draw function: the same selection, the same categories and the same
//               next std::rand() value are required.  Prints one summary line per window and the count of failed checks.
// Case format (one token stream): `case max_near max_middle max_far seed`, `near n (id flow)*`, `middle n id*`, `far n (id seen)*`,
// `depth m` and m times `entry wanted n (id cost)*`; flows and costs in any strtod spelling (hex floats, nan).
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <map>
#include <set>
#include <string>
#include <utility>
#include <vector>

#include "kba_b200.h"
#include "keyframe_bundle_adjustment/bundle_adjuster_keyframes.hpp"
#include "keyframe_bundle_adjustment/landmark_selection_schemes.hpp"

using namespace keyframe_bundle_adjustment;
static int g_fail = 0;
#define CHECK(c) do { if (!(c)) { std::printf("CHECK FAILED %s:%d: %s\n", __FILE__, __LINE__, #c); ++g_fail; } } while (0)

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

static int32_t draw_rand(void*, int32_t n, int32_t* out) {
    for (int32_t i = 0; i < n; ++i) out[i] = std::rand();
    return 0;
}

// the drive of tests/cpp/test_facade_select.cpp: scene and road landmarks, one camera, 33 keyframes
static int device_drive(kba_handle* h, int window) {
    const int n_scene = 1400, n_ground = n_scene / 4, n_frames = 33;
    const double height = 1.6;
    std::vector<Eigen::Vector3d> lms;
    for (int i = 0; i < n_scene; ++i)
        lms.push_back(Eigen::Vector3d(4. + 0.061 * ((i * 37) % 1201), -30. + 0.047 * ((i * 53) % 1279), -1. + 0.011 * ((i * 29) % 997)));
    for (int i = 0; i < n_ground; ++i)
        lms.push_back(Eigen::Vector3d(6. + 0.05 * ((i * 41) % 997), -6. + 0.013 * ((i * 23) % 991), -height));
    std::vector<Eigen::Isometry3d> gt(n_frames);
    gt[0] = Eigen::Isometry3d::Identity();
    for (int k = 1; k < n_frames; ++k) {
        gt[k] = gt[k - 1];
        gt[k].translate(Eigen::Vector3d(-0.6, 0.01 * (k % 3), 0.));
        gt[k].rotate(Eigen::AngleAxisd(0.003, Eigen::Vector3d(0., 0., 1.)));
    }
    Eigen::Matrix3d rc = Eigen::Matrix3d::Zero();
    rc(0, 1) = -1.; rc(1, 2) = -1.; rc(2, 0) = 1.;
    Eigen::Isometry3d ext = Eigen::Isometry3d::Identity();
    ext.rotate(rc);
    const Camera proto(700., Eigen::Vector2d(600., 190.), ext);
    Tracklets ts;
    for (int k = 0; k < n_frames; ++k) ts.stamps.push_back(k);
    ts.tracks.resize(lms.size());
    size_t n_meas = 0;
    for (size_t i = 0; i < lms.size(); ++i) {
        const bool ground = int(i) >= n_scene;
        ts.tracks[i].id = i;
        ts.tracks[i].label = ground ? 7 : 0;
        const int len = (i % 11 == 0) ? 1 : 2 + int((i * 7) % size_t(n_frames));
        for (int k = 0; k < std::min(len, n_frames); ++k) {
            const Eigen::Vector3d lm_cam = ext * (gt[k] * lms[i]);
            Eigen::Vector3d proj = proto.getIntrinsicMatrix() * lm_cam;
            proj /= proj[2];
            const float du = 0.3f * float((int(i) * 7 + k * 3) % 5 - 2), dv = 0.3f * float((int(i) * 3 + k * 5) % 5 - 2);
            const float d = (!ground && i % 3 == 0) ? float(lm_cam[2]) : -1.f;
            ts.tracks[i].feature_points.push_back(FeaturePoint(float(proj[0]) + du, float(proj[1]) + dv, d));
            ++n_meas;
        }
    }
    BundleAdjusterKeyframes a;
    a.set_solver_time(20.);
    add_chain(*a.landmark_selector_, window);
    Plane plane;
    plane.distance = height;
    auto cam = [&] { return std::make_shared<Camera>(700., Eigen::Vector2d(600., 190.), ext); };
    const Pose cam_pose = convert(EigenPose(ext));
    const double intr[3] = {700., 600., 190.};
    kba_track* t = nullptr;
    const int n_lm = int(lms.size());
    kba_track_caps caps{n_frames, n_lm, int32_t(n_meas), 8, 64, 64, 0, 0};
    CHECK(kba_track_create(h, &caps, 1, intr, cam_pose.data(), &t) == KBA_OK);
    if (!t) { std::printf("%s\n", kba_last_error()); return 0; }
    int steps = 0, draws_used = 0, depth_only = 0;
    size_t bins[3] = {0, 0, 0};
    for (int k = 0; k < n_frames; ++k) {
        Eigen::Isometry3d start = gt[k];
        if (k >= 2) start.translate(Eigen::Vector3d(0.03, -0.02, 0.01));
        const auto fix = k == 0 ? Keyframe::FixationStatus::Pose : (k == 1 ? Keyframe::FixationStatus::Scale : Keyframe::FixationStatus::None);
        a.push(Keyframe(k, ts, cam(), start, fix, plane));
        {  // mirror the keyframe: its measurements in landmark-id runs (one camera)
            const Keyframe& kf = *a.keyframes_.at(k);
            std::vector<int32_t> lm;
            std::vector<float> u, v, d;
            for (const auto& el : kf.measurements_)
                for (const auto& cm : el.second) { lm.push_back(int32_t(el.first)); u.push_back(cm.second.u); v.push_back(cm.second.v); d.push_back(cm.second.d); }
            CHECK(kba_track_push_keyframe(t, k, kf.pose_.data(), nullptr, int32_t(lm.size()), lm.data(), nullptr, u.data(), v.data(), d.data()) == KBA_OK);
        }
        if (k < 3) continue;
        a.deactivateKeyframes(3, 4, window);
        a.updateLabels(ts, 0.9);
        // the facade's current state into the store: every keyframe pose, every landmark position
        std::vector<int32_t> kfs, ids;
        std::vector<double> poses, pos;
        for (const auto& el : a.keyframes_) { kfs.push_back(int32_t(el.first)); poses.insert(poses.end(), el.second->pose_.begin(), el.second->pose_.end()); }
        for (const auto& el : a.landmarks_) { ids.push_back(int32_t(el.first)); pos.insert(pos.end(), el.second->pos.begin(), el.second->pos.end()); }
        CHECK(kba_track_set_keyframe_poses(t, int32_t(kfs.size()), kfs.data(), poses.data(), nullptr) == KBA_OK);
        CHECK(kba_track_set_landmarks(t, int32_t(ids.size()), ids.data(), pos.data(), nullptr) == KBA_OK);
        // host: a standalone selector with the adjuster's chain and outliers
        const auto act_lm = a.getActiveLandmarkConstPtrs();
        const auto act_kf = a.getActiveKeyframeConstPtrs();
        LandmarkSelector s;
        s.addScheme(LandmarkRejectionSchemeCheirality::create());
        add_chain(s, window);
        s.setOutlier(a.landmark_selector_->getOutliers());
        const unsigned seed = 1000u + unsigned(k);
        std::srand(seed);
        const std::set<LandmarkId> host = s.select(act_lm, act_kf);
        const int next_host = std::rand();
        // device: the same lists, a std::rand draw function
        std::vector<int32_t> kf_slot, lm_slot;
        std::vector<uint8_t> elig;
        for (const auto& el : act_kf) kf_slot.push_back(int32_t(el.first));
        for (const auto& el : act_lm)
            if (!s.getOutliers().count(el.first)) { lm_slot.push_back(int32_t(el.first)); elig.push_back(el.second->is_ground_plane ? 1 : 0); }
        std::vector<kba_depth_entry> depth;
        for (int i = 0; i < window; ++i) depth.push_back(kba_depth_entry{i, 50});
        const kba_select_params prm{{0.5, 0.5, 0.3}, 40., 15.};
        kba_rank_request rq{int32_t(kf_slot.size()), int32_t(lm_slot.size()), kf_slot.data(), lm_slot.data(), elig.data(), &prm, 400, 400, 400,
                            int32_t(depth.size()), depth.data(), draw_rand, nullptr};
        std::vector<int32_t> cand(lm_slot.size() + 1);
        std::vector<int8_t> cat(lm_slot.size() + 1);
        kba_rank_out o{0, 0, 0, 0, cand.data(), cat.data()};
        std::srand(seed);
        const int rc = kba_track_rank_landmarks(t, &rq, &o);
        CHECK(rc == KBA_OK);
        if (rc != KBA_OK) std::printf("%s\n", kba_last_error());
        const int next_device = std::rand();
        CHECK(next_device == next_host);
        std::set<LandmarkId> device;
        std::map<LandmarkId, int> device_cat, host_cat;
        for (int i = 0; i < o.n_sel; ++i) {
            device.insert(LandmarkId(lm_slot[cand[i]]));
            if (cat[i] < 3) device_cat[LandmarkId(lm_slot[cand[i]])] = cat[i];
            else ++depth_only;
        }
        for (const auto& el : s.getLandmarkCategories()) { host_cat[el.first] = int(el.second); ++bins[int(el.second)]; }
        CHECK(device == host);
        CHECK(device_cat == host_cat);
        draws_used += o.n_draws;
        ++steps;
        std::srand(seed);
        a.solve();
    }
    kba_track_destroy(t);
    CHECK(bins[0] > 0 && bins[1] > 0 && bins[2] > 0 && depth_only > 0 && draws_used > 0);
    std::printf("window %d: %d rankings equal to select(), std::rand() left where select() leaves it; near / middle / far %zu / %zu / %zu, "
                "AddDepth only %d, %d draws\n", window, steps, bins[0], bins[1], bins[2], depth_only, draws_used);
    return steps;
}

static double num(std::ifstream& in) {
    std::string s;
    in >> s;
    return std::strtod(s.c_str(), nullptr);
}

int main(int argc, char** argv) {
    if (argc == 2 && std::string(argv[1]) == "device") {
        std::setvbuf(stdout, nullptr, _IOLBF, 0);
        kba_handle* h = nullptr;
        CHECK(kba_create(&h, 0) == KBA_OK);
        if (!h) { std::printf("%s\n", kba_last_error()); return 1; }
        for (const int window : {12, 20}) CHECK(device_drive(h, window) == 30);
        kba_destroy(h);
        std::printf("%d failed checks\n", g_fail);
        return g_fail ? 1 : 0;
    }
    if (argc != 3 || std::string(argv[1]) != "host") {
        std::fprintf(stderr, "usage: %s host FILE | %s device\n", argv[0], argv[0]);
        return 2;
    }
    std::ifstream in(argv[2]);
    std::string tag;
    int k = 0;
    while (in >> tag) {
        if (tag != "case") return 3;
        LandmarkSparsificationSchemeVoxel::Parameters p;
        unsigned seed = 0;
        in >> p.max_num_landmarks_near >> p.max_num_landmarks_middle >> p.max_num_landmarks_far >> seed;
        const LandmarkSparsificationSchemeVoxel voxel(p);
        std::vector<LandmarkId> ids_near, ids_middle, ids_far;
        std::map<LandmarkId, double> flow;
        std::map<LandmarkId, unsigned int> seen;
        int n = 0;
        in >> tag >> n;
        for (int i = 0; i < n; ++i) {
            LandmarkId id;
            in >> id;
            const double f = num(in);
            ids_near.push_back(id);
            if (f == f) flow[id] = f;  // a near landmark without a flow value has no entry (calcFlow)
        }
        in >> tag >> n;
        for (int i = 0; i < n; ++i) { LandmarkId id; in >> id; ids_middle.push_back(id); }
        in >> tag >> n;
        for (int i = 0; i < n; ++i) { LandmarkId id; unsigned s; in >> id >> s; ids_far.push_back(id); seen[id] = s; }
        std::srand(seed);
        std::map<LandmarkId, int> out;
        for (const auto& el : voxel.rankBins(ids_near, flow, ids_middle, ids_far, seen)) out[el.first] = int(el.second);
        const int next = std::rand();
        int m = 0;
        in >> tag >> m;
        for (int e = 0; e < m; ++e) {  // LandmarkSelectionSchemeAddDepth::getSelection's ranking of one (ind, wanted) entry
            int wanted = 0;
            in >> tag >> wanted >> n;
            std::vector<std::pair<LandmarkId, double>> cost;
            for (int i = 0; i < n; ++i) { LandmarkId id; in >> id; cost.emplace_back(id, num(in)); }
            const int keep = std::min(wanted, int(cost.size()));
            std::partial_sort(cost.begin(), cost.begin() + keep, cost.end(), [](const auto& a, const auto& b) { return a.second < b.second; });
            for (int i = 0; i < keep; ++i) out.emplace(cost[i].first, 3);  // a landmark of a bin keeps its category
        }
        std::printf("C %d", k);
        for (const auto& el : out) std::printf(" %lu:%d", (unsigned long)el.first, el.second);
        std::printf("\n");
        // the draws the shuffle consumed: the position of `next` in the seeded sequence
        std::srand(seed);
        std::vector<int> drawn;
        for (int v = std::rand(); v != next; v = std::rand()) drawn.push_back(v);
        std::printf("R %d %zu", k, drawn.size());
        for (int v : drawn) std::printf(" %d", v);
        std::printf("\n");
        ++k;
    }
    return 0;
}
