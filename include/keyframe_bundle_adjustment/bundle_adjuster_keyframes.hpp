// bundle_adjuster_keyframes.hpp -- source-compatible facade of limo's BundleAdjusterKeyframes (reference:
// keyframe_bundle_adjustment/include/keyframe_bundle_adjustment/bundle_adjuster_keyframes.hpp:40-335) whose solve() /
// adjustPoseOnly() run on the H100 through the C ABI of kba_b200.h instead of Ceres.  Same namespace, class name, public
// members, method signatures and exceptions; the private ceres::Problem member is replaced by a kba_handle.  The types
// around it live where the reference keeps them: internal/definitions.hpp, keyframe.hpp, landmark_selector.hpp,
// landmark_selection_schemes.hpp, matches_msg_types/*.hpp.
#pragma once
#include <array>
#include <exception>
#include <map>
#include <memory>
#include <set>
#include <string>
#include <tuple>
#include <vector>

#include "internal/triangulator.hpp"
#include "keyframe.hpp"
#include "landmark_selector.hpp"

struct kba_handle;
struct kba_track;
struct kba_window;
struct kba_evaluate_out;

namespace keyframe_bundle_adjustment {

// ---- the adjuster (bundle_adjuster_keyframes.hpp:40-335) ----
class BundleAdjusterKeyframes {
public:
    using UPtr = std::unique_ptr<BundleAdjusterKeyframes>;
    using Ptr = std::shared_ptr<BundleAdjusterKeyframes>;
    using v3 = Eigen::Vector3d;

    struct NotEnoughKeyframesException : public std::exception {
        NotEnoughKeyframesException(size_t num_is, size_t num_should_be);
        const char* what() const noexcept override { return msg.c_str(); }
        size_t num_is, num_should_be;
        std::string msg;
    };
    struct KeyframeNotFoundException : public std::exception {
        explicit KeyframeNotFoundException(TimestampNSec timestamp);
        const char* what() const noexcept override { return msg.c_str(); }
        TimestampNSec ts_;
        std::string msg;
    };
    struct OutlierRejectionOptions {  // :79-89
        double depth_thres{0.16};
        double reprojection_thres{1.6};
        double depth_quantile{0.95};
        double reprojection_quantile{0.95};
        int num_iterations{1};
    };

    BundleAdjusterKeyframes();
    ~BundleAdjusterKeyframes();
    BundleAdjusterKeyframes(const BundleAdjusterKeyframes&) = delete;
    BundleAdjusterKeyframes& operator=(const BundleAdjusterKeyframes&) = delete;

    void push(const Keyframe& kf);
    void push(const std::vector<Keyframe>& kfs);
    std::string solve();
    void deactivateKeyframes(int min_num_connecting_landmarks = 3, int min_size_optimization_window = 4,
                             int max_size_optimization_window = 20);
    const Keyframe& getKeyframe(TimestampSec timestamp = -1.) const;
    std::map<KeyframeId, Keyframe::Ptr> getActiveKeyframePtrs() const;
    std::map<KeyframeId, Keyframe::ConstPtr> getActiveKeyframeConstPtrs() const;
    std::vector<Keyframe::Ptr> getSortedActiveKeyframePtrs() const;
    std::vector<std::pair<KeyframeId, Keyframe::Ptr>> getSortedIdsWithActiveKeyframePtrs() const;
    std::map<LandmarkId, Landmark::ConstPtr> getActiveLandmarkConstPtrs() const;
    std::map<LandmarkId, Landmark::ConstPtr> getSelectedLandmarkConstPtrs() const;
    std::string adjustPoseOnly(Keyframe&);
    bool calculateLandmark(const Keyframe& kf, const LandmarkId& lId, v3& posAbs);
    bool calculateLandmark(const LandmarkId& lId, v3& posAbs);
    void set_solver_time(double solver_time_sec) { this->solver_time_sec = solver_time_sec; }
    // Not in the reference: keep the pushed keyframes on the device (kba_track_*, include/kba_b200.h) so that solve() sends only
    // the lists of active keyframes / selected landmarks instead of re-packing and re-uploading the window (the reference
    // rebuilds its ceres::Problem per call, cpp:635-637).  On by default; windows the device-resident store cannot take (more than
    // 30 keyframes, ground-plane residuals, a camera that was not there at the first push) fall back to the rebuild path.
    // adjustPoseOnly() then tracks the frame against the landmarks in that store (kba_track_adjust_pose) when the store has every
    // landmark and camera of the frame, and otherwise rebuilds its one-keyframe window.
    void set_persistent_window(bool on) { persistent_window_ = on; }
    // Not in the reference: the capacities of that store (defaults 256 keyframes, 131072 landmarks, 2^21 measurements).  Landmark
    // slots that no stored keyframe measures any more are reclaimed when the store runs out (kba_track_reclaim_landmarks), so the
    // landmark capacity bounds the landmarks of the stored keyframes, not those of the whole run.  Only before the store exists
    // (the first solve()); afterwards it throws std::logic_error.
    void set_track_capacity(int max_keyframes, int max_landmarks, int max_measurements);
    // Not in the reference: with the persistent window on, solve() lets the store compute the per-landmark quantities of the
    // landmark selector's chain (kba_track_select_landmarks) when the chain is cheirality + voxel (+ selection schemes, limo's
    // mono-lidar configuration); the selector ranks them exactly as its host select() does, so the selection is the same.
    // On by default; lastSelectionOnDevice() tells whether the last solve() selected that way.
    void set_device_selection(bool on) { device_selection_ = on; }
    bool lastSelectionOnDevice() const { return last_select_on_device_; }
    // host -> device bytes of the last solve() (either path) and of all push() calls so far (persistent path)
    long long lastSolveUploadBytes() const { return last_solve_h2d_; }
    long long pushUploadBytes() const { return push_h2d_; }
    void updateLabels(const Tracklets& t, double shrubbery_weight = 1.);

    // What evaluateResiduals() finds (not in the reference, whose evaluateResiduals() only writes into its ceres::Problem).
    struct Evaluation {
        struct Residual {                  // one observation: rows before any loss or weight, and the scaled Cauchy losses
            double u{0.}, v{0.}, depth{0.};  // projection - measurement (px), z_cam - d (m; 0 without a depth); NaN if it failed
            double rho_reprojection{0.}, rho_depth{0.};
        };
        struct Trim {                      // one landmark: solveTrimmed's trimming values and TrimmerQuantile's decisions
            double reprojection{-1.}, depth{-1.};  // largest raw block norm over its observations, -1 without one
            bool rejected_reprojection{false}, rejected_depth{false};
        };
        using ObservationKey = std::tuple<LandmarkId, KeyframeId, CameraId>;  // (landmark id, keyframe timestamp, camera id)
        std::map<ObservationKey, Residual> residuals;
        std::map<LandmarkId, Trim> landmarks;
        std::map<LandmarkId, double> ground_plane;  // height residual of every attached ground-plane landmark
        // reprojection, depth, ground plane, scale regulariser, plane chain, total: 1/2 sum rho, as ceres counts the cost
        double cost_reprojection{0.}, cost_depth{0.}, cost_ground_plane{0.}, cost_scale{0.}, cost_plane_chain{0.}, cost_total{0.};
        bool failed{false};                // some observation has |z_cam| < 0.01
    };
    // The reference's evaluateResiduals() (bundle_adjuster_keyframes.hpp:171-175): the last solve()'s window (the active keyframes,
    // selected_landmark_ids_) evaluated at the current state with outlier_rejection_options_, on the device-resident store
    // (kba_track_evaluate), into last_evaluation_.  It changes no selection, outlier set, pose or landmark.  Throws
    // std::runtime_error naming the reason when the persistent window is off or failed, before the first solve(), or when the
    // window does not fit the store; there is no host fallback.
    void evaluateResiduals();
    Evaluation last_evaluation_;

    std::map<KeyframeId, Keyframe::Ptr> keyframes_;
    std::map<LandmarkId, Landmark::Ptr> landmarks_;
    std::set<KeyframeId> active_keyframe_ids_;
    std::set<LandmarkId> active_landmark_ids_;
    std::set<LandmarkId> selected_landmark_ids_;
    OutlierRejectionOptions outlier_rejection_options_;
    std::unique_ptr<LandmarkSelector> landmark_selector_;
    std::map<std::string, std::set<int>> labels_{{"outliers", {23, 24, 25, 26, 27, 28, 29, 30, 31, 32, 33}},
                                                 {"shrubbery", {21}},
                                                 {"ground", {6, 7, 8, 9, 10}}};

private:
    std::map<LandmarkId, Landmark::ConstPtr> filterLandmarksById(const std::set<LandmarkId>& ids) const;
    std::string runWindow(const std::vector<Keyframe*>& kfs, const std::vector<LandmarkId>& lm_ids, bool motion_only,
                          Keyframe* speed_prior_for);
    kba_handle* handle_{nullptr};  // replaces std::shared_ptr<ceres::Problem> problem_
    double solver_time_sec;
    // persistent device-resident window
    bool ensureHandle();
    bool trackPush(const Keyframe& kf);
    bool trackSync(const std::vector<Keyframe*>& kfs);
    bool selectOnDevice(const std::vector<Keyframe*>& kfs);
    bool solveTracked(const std::vector<Keyframe*>& kfs, const std::vector<LandmarkId>& lm_ids, std::string& report, bool synced);
    struct TrackRequest;  // a track solve's or evaluation's lists (trackRequest)
    bool trackRequest(const std::vector<Keyframe*>& kfs, const std::vector<LandmarkId>& lm_ids, TrackRequest& q) const;
    bool adjustPoseTracked(Keyframe& kf, const std::vector<LandmarkId>& lm_ids, std::string& report);
    bool flushLandmarks();  // new and dirty landmark state into the store, before any use of the track
    void dropInactiveKeyframes(size_t max_free_kf_slots);
    bool reclaimLandmarkSlots(const Keyframe& kf);
    void speedPrior(const Keyframe& speed_kf, kba_window& w) const;
    kba_track* track_{nullptr};
    bool persistent_window_{true}, track_failed_{false}, device_selection_{true}, last_select_on_device_{false};
    int track_keyframes_{256}, track_landmarks_{1 << 17}, track_measurements_{1 << 21};
    std::map<KeyframeId, int> kf_slot_;
    std::map<LandmarkId, int> lm_slot_;
    std::vector<LandmarkId> slot_lm_;  // the landmark a slot was handed to (slot -> id), for every slot handed out so far
    std::vector<int> free_kf_slots_, free_lm_slots_;
    std::vector<std::array<double, 10>> track_cams_;  // camera values (f, pp, pose_camera_vehicle) the track was created with
    std::set<LandmarkId> new_landmarks_, dirty_weights_;
    std::set<LandmarkId> restore_landmarks_;  // existing landmarks that got a slot again: position and weight go up at the flush
    std::set<LandmarkId> dirty_positions_;  // positions the rebuild path wrote on the host only
    long long last_solve_h2d_{0}, push_h2d_{0}, last_select_h2d_{0};
};

// the outputs of kba_track_evaluate for the window of keyframes kfs (ascending id) and landmarks lm_ids (ascending id), keyed as
// BundleAdjusterKeyframes::Evaluation keys them; track_cams are the store's cameras (focal length, principal point,
// pose_camera_vehicle) in index order.  The window's observations come landmark by landmark, keyframe by keyframe and, inside a
// keyframe, in Keyframe::measurements_ order; an output that does not follow that order throws std::runtime_error.
BundleAdjusterKeyframes::Evaluation keyEvaluation(const std::vector<const Keyframe*>& kfs, const std::vector<LandmarkId>& lm_ids,
                                                  const std::vector<std::array<double, 10>>& track_cams, const kba_evaluate_out& out);

}  // namespace keyframe_bundle_adjustment
