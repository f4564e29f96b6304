/*
 * kba_b200.h -- C ABI of the H100-native (sm_90a) keyframe bundle-adjustment hot path.
 *
 * This is the drop-in boundary for limo's `keyframe_bundle_adjustment` window solve.
 * The reference has no FFI: its "operator API" is the C++ class
 *   BundleAdjusterKeyframes            (keyframe_bundle_adjustment/include/keyframe_bundle_adjustment/bundle_adjuster_keyframes.hpp:40-335)
 * whose solve() / adjustPoseOnly() hand a ceres::Problem to
 *   robust_optimization::solveTrimmed  (robust_optimization/src/robust_solving.cpp:140-248).
 * Everything below the construction of that ceres::Problem -- residual/Jacobian evaluation
 * (cost_functors_ceres.hpp:53-222,224-250,355-438,507-555), robust losses, local parameterisations,
 * Schur elimination of the landmark blocks, the dense reduced solve, the Levenberg-Marquardt
 * loop and the quantile trimming -- is replaced by the entry points declared here.
 *
 * Plain C: pointers + sizes only, no torch / Eigen / ceres types.  All arrays are caller owned.
 * "host" entry points take host pointers and perform the host<->device copies themselves;
 * the kba_batch_* entry points keep a batch of windows resident in HBM.
 *
 * The library has NO CPU fallback: every entry point that computes returns KBA_ERR_CUDA if no
 * sm_90 (H100-class) device is usable.
 */
#ifndef KBA_B200_H
#define KBA_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define KBA_VERSION_MAJOR 0
#define KBA_VERSION_MINOR 5

/* ---- status codes (reference: C++ exceptions / text report, bundle_adjuster_keyframes.cpp:630-632) ---- */
enum {
    KBA_OK = 0,
    KBA_ERR_BAD_ARG = 1,       /* null pointer, negative size, index out of range */
    KBA_ERR_CUDA = 2,          /* no device / CUDA runtime error (see kba_last_error) */
    KBA_ERR_NOT_ENOUGH_KF = 3, /* fewer than 3 keyframes: NotEnoughKeyframesException, cpp:630 */
    KBA_ERR_CAPACITY = 4,      /* window larger than the limits compiled into the kernels */
    KBA_ERR_NCCL = 5,
    KBA_ERR_TIMEOUT = 6        /* kba_result.status only: the host's safety cap ended the batch before this window finished */
};

/* ---- termination of one inner solve (mirrors ceres::TerminationType as used via Summary) ---- */
enum {
    KBA_TERM_CONVERGENCE = 0,    /* function / parameter / gradient tolerance or min radius */
    KBA_TERM_NO_CONVERGENCE = 1, /* max_num_iterations reached                            */
    KBA_TERM_FAILURE = 2         /* evaluation failed at the start (|z_cam| < 0.01) or 5 invalid steps */
};

/*
 * One optimisation window = what BundleAdjusterKeyframes::solve() (cpp:629-767) assembles
 * into a ceres::Problem.  Landmark-major CSR over the observations (SURVEY.md section 8b).
 *
 * Index conventions: keyframes 0..n_kf-1 are the ACTIVE keyframes in ascending id (= timestamp)
 * order (std::set iteration order, cpp:505); landmarks 0..n_lm-1 are the SELECTED landmarks in
 * ascending id order; observations of landmark j are obs[lm_obs_ptr[j] .. lm_obs_ptr[j+1]) sorted
 * by keyframe index, then camera index.
 */
typedef struct kba_window {
    int32_t n_kf, n_cam, n_lm, n_obs, n_gp;

    /* keyframes (keyframe.hpp:172-195) */
    const double* kf_pose;    /* [n_kf*7] quaternion (w,x,y,z) + translation; p_kf = R(q) p_origin + t (definitions.hpp:75-83) */
    const uint8_t* kf_fixed;  /* [n_kf]   1 = FixationStatus::Pose -> pose and plane blocks constant (cpp:198-219) */
    const double* kf_plane;   /* [n_kf*4] ground plane direction (3) + distance (definitions.hpp:27-34); may be NULL if n_gp == 0 */

    /* cameras (definitions.hpp:93-124) */
    const double* cam_intr;   /* [n_cam*3] focal length, principal point x, y */
    const double* cam_pose;   /* [n_cam*7] camera <- vehicle extrinsics, same 7-vector convention */

    /* landmarks (definitions.hpp:42-68) */
    const double* lm_pos;     /* [n_lm*3] position in the origin frame */
    const double* lm_weight;  /* [n_lm]   ScaledLoss weight (1.0, or shrubbery weight; cpp:589-591,616-618) */
    const int32_t* lm_obs_ptr;/* [n_lm+1] CSR row pointers */

    /* observations = FeaturePoint{u,v,d} (matches_msg_types/feature_point.hpp:24-26) */
    const int32_t* obs_kf;    /* [n_obs] keyframe index */
    const int32_t* obs_cam;   /* [n_obs] camera index, or NULL (all camera 0) */
    const float* obs_u;       /* [n_obs] */
    const float* obs_v;       /* [n_obs] */
    const float* obs_d;       /* [n_obs] lidar depth; a depth residual exists iff d > 0 (cpp:578) */

    /* ground-plane height residuals, already attached to their nearest keyframe and weighted by the
     * host exactly as addGroundPlaneResiduals does at problem-build time (cpp:517-562) */
    const int32_t* gp_lm;     /* [n_gp] landmark index */
    const int32_t* gp_kf;     /* [n_gp] keyframe index */
    const double* gp_weight;  /* [n_gp] ScaledLoss weight = 10 * (1 - dist/25) */

    /* scale regulariser PoseRegularization (cost_functors_ceres.hpp:224-250, cpp:890-904):
     * residual |(T_kf1 * T_kf0^-1).t| - scale_value, TrivialLoss scaled by scale_weight. */
    int32_t scale_kf0, scale_kf1;
    double scale_weight;      /* <= 0: no scale regulariser */
    double scale_value;

    /* ground-plane regularisation chain (cpp:769-818): weight > 0 adds, for consecutive keyframes,
     * normal difference (3w), distance difference (w), motion-in-plane (2w) and, for every keyframe,
     * the (0,0,1) normal prior (w).  The reference passes w = 10 and only if n_gp > 0 (cpp:717-719). */
    double plane_reg_weight;
    uint8_t plane_dist_fixed; /* 1: all plane distances constant (fewer than 10 depth residuals, cpp:722-728) */
    uint8_t landmarks_fixed;  /* 1: every landmark block constant = motion-only problem of adjustPoseOnly (cpp:862, 221-270) */
    uint8_t reserved_[6];

    /* SpeedRegularizationVector2 prior of adjustPoseOnly (cost_functors_ceres.hpp:300-353, cpp:835-853) on keyframe
     * speed_kf: residual(3) = (T_kf * speed_T_origin_before).t / speed_dt - speed_v_before, TrivialLoss * speed_weight. */
    int32_t speed_kf;         /* keyframe index the prior acts on */
    int32_t reserved2_;
    double speed_weight;      /* <= 0: none */
    double speed_dt;
    double speed_v_before[3];
    double speed_T_origin_before[7]; /* inverse of the newest window keyframe pose, frozen (7-vector convention) */
} kba_window;

/* Options = OutlierRejectionOptions (bundle_adjuster_keyframes.hpp:79-89) + the ceres / solveTrimmed
 * settings reachable from solve() (robust_solving.hpp:93-108, cpp:740-764). Fill with kba_default_options. */
typedef struct kba_options {
    double depth_thres;            /* 0.16  Cauchy scale of the depth residual            */
    double reprojection_thres;     /* 1.6   Cauchy scale of the reprojection residual     */
    double depth_quantile;         /* 0.95                                                 */
    double reprojection_quantile;  /* 0.95                                                 */
    double gp_quantile;            /* 1.0   (cpp:758)                                      */
    double gp_huber;               /* 0.1   Huber scale of the ground-plane residual (cpp:549) */
    int32_t num_trim_rounds;       /* entries of number_iterations (cpp:740-745); -1 = reference rule:
                                      num_iterations(1) rounds iff n_lm > min_landmarks_for_trimming */
    int32_t trim_solver_iterations;/* 2     max_num_iterations per trimming round (cpp:743)  */
    int32_t final_solver_iterations;/*100   max_num_iterations of the final solve (robust_solving.hpp:100) */
    int32_t min_landmarks_for_trimming; /* 100 for solve() (cpp:741), 30 for adjustPoseOnly (cpp:865) */
    int32_t min_residual_groups;   /* 30    (cpp:762, robust_solving.cpp:109)               */
    int32_t num_rounds_option;     /* outlier_rejection_options_.num_iterations, default 1  */
    double solver_time_sec;        /* max_solver_time_in_seconds of EVERY inner ceres::Solve (robust_solving.cpp:233-238), checked on
                                      the device between iterations: the solve ends NO_CONVERGENCE with its accepted iterate and
                                      solveTrimmed continues, so the final solve always runs.  <= 0: none; ignored by sharded
                                      solves (collective).  Parity runs use 20 s as the reference tests do
                                      (test/keyframe_bundle_adjustment.cpp:486) */
    /* ceres defaults, never overridden by the reference (robust_solving.hpp:101-103 are commented out) */
    double function_tolerance;     /* 1e-6  */
    double gradient_tolerance;     /* 1e-10 */
    double parameter_tolerance;    /* 1e-8  */
    double initial_trust_region_radius; /* 1e4 */
    double max_trust_region_radius;     /* 1e16 */
    double min_trust_region_radius;     /* 1e-32 */
    double min_relative_decrease;       /* 1e-3 */
    double min_lm_diagonal;             /* 1e-6 */
    double max_lm_diagonal;             /* 1e32 */
    int32_t max_consecutive_invalid_steps; /* 5 */
    int32_t precision;             /* 0: FP64 kernels; 1: FP32 Jacobian kernels with FP64 accumulation */
} kba_options;

/* One LM iteration record (subset of ceres::IterationSummary that the report prints). */
typedef struct kba_iteration {
    double cost;               /* cost at the END of the iteration (candidate cost if rejected) */
    double cost_change;
    double gradient_max_norm;
    double step_norm;
    double relative_decrease;
    double trust_region_radius;
    int32_t iteration;
    int32_t solve_index;       /* which inner ceres::Solve of solveTrimmed */
    int32_t step_is_valid, step_is_successful;
} kba_iteration;

#define KBA_MAX_SOLVES 8

/* Summary of one inner ceres::Solve call. */
typedef struct kba_solve_summary {
    double initial_cost, final_cost;
    int32_t num_iterations;    /* iterations attempted, excluding iteration 0 */
    int32_t num_successful_steps;
    int32_t termination;       /* KBA_TERM_* */
    int32_t num_landmarks;     /* landmark blocks in the program */
    int32_t num_residual_blocks;
    int32_t reserved_;
} kba_solve_summary;

/* Result of kba_solve_window = what the caller of solve() reads back from Keyframe::pose_,
 * Landmark::pos, Plane (mono_lidar.cpp:204,263-265,283) + robust_optimization::Summary. */
typedef struct kba_result {
    /* outputs, caller-allocated; any may be NULL */
    double* kf_pose;           /* [n_kf*7] */
    double* kf_plane;          /* [n_kf*4] */
    double* lm_pos;            /* [n_lm*3] */
    uint8_t* lm_rejected;      /* [n_lm] 1 if the trimming removed the landmark's residuals */
    kba_iteration* iterations; /* [iterations_capacity] optional per-iteration log */
    int32_t iterations_capacity;
    /* filled by the library */
    int32_t num_iteration_records;
    int32_t num_solves;
    int32_t status;            /* KBA_OK or error of this window */
    kba_solve_summary solves[KBA_MAX_SOLVES];
    double initial_cost;       /* Summary::initial_cost = first solve (robust_solving.hpp:71) */
    double final_cost;         /* Summary::final_cost  = last solve  (robust_solving.hpp:72) */
    double time_sec;           /* device time of the whole window solve (batch: of the whole batch) */
} kba_result;

/* What kba_eval materialises (parity / inspection entry point; evaluates at the window's input state). */
typedef struct kba_eval_out {
    double* residual;  /* [3*n_obs] rows (u, v, depth), robustified (sqrt(rho') applied); row 2 = 0 if no depth */
    double* jac_pose;  /* [18*n_obs] 3x6 row-major, d r~ / d (delta_rot, delta_trans); zeros for fixed keyframes */
    double* jac_lm;    /* [9*n_obs]  3x3 row-major, d r~ / d landmark; precision 1 on the fused path: formed in FP64 from the
                          FP32 jac_pose as the solver forms it (translation columns times the keyframe's rotation) */
    double* cost;      /* [1] 0.5 * sum rho over reprojection + depth blocks */
    int32_t* failed;   /* [1] 1 if any |z_cam| < 0.01 (evaluation failure, cost_functors_ceres.hpp:78-83) */
} kba_eval_out;

typedef struct kba_handle kba_handle;  /* one per host thread / GPU; not thread-safe */
typedef struct kba_batch kba_batch;    /* windows resident in HBM */

/* --- lifecycle --- */
int kba_version(void);                                   /* major*100 + minor */
const char* kba_last_error(void);                        /* message of the last failing call on this thread */
void kba_default_options(kba_options* opt);
int kba_create(kba_handle** out, int device);            /* replaces `new ceres::Problem` + thread pool */
void kba_destroy(kba_handle* h);
int kba_set_stream(kba_handle* h, void* cuda_stream);    /* cudaStream_t; NULL = default stream */

/* --- host-buffer entry points (the reference-facing calls) --- */
/* replaces robust_optimization::solveTrimmed(...) as called from solve() (cpp:765); up to 128 keyframes per window, ground-plane
 * blocks included (kba_batch_create's limits) */
int kba_solve_window(kba_handle* h, const kba_window* w, const kba_options* opt, kba_result* res);
/* many independent windows in one call ("BA windows/s") */
int kba_solve_batch(kba_handle* h, int32_t n_windows, const kba_window* w, const kba_options* opt, kba_result* res);
/* kba_solve_batch with opts[n_windows]: window i is solved with opts[i] exactly as kba_solve_batch solves it with that one set
 * (a parameter sweep over one recording in one launch).  Checked before anything is uploaded: an entry that kba_batch_solve
 * refuses, or entries whose precision differs (it selects the kernel variants of the whole batch), fail the call with its code,
 * and kba_last_error names the window index. */
int kba_solve_batch_opts(kba_handle* h, int32_t n_windows, const kba_window* w, const kba_options* opts, kba_result* res);
/* residuals + Jacobian blocks of the reprojection / depth residuals at the input state
 * (what ceres::Problem::Evaluate would return for those blocks, cf. robust_solving.cpp:44) */
int kba_eval(kba_handle* h, const kba_window* w, const kba_options* opt, kba_eval_out* out);

/* --- device-resident batch (inputs stay in HBM between solves) --- */
/* A window has at most 128 keyframes (KBA_ERR_CAPACITY): a reduced system of up to 1281 rows with ground-plane blocks, allocated
 * as 1344 (about 14.5 MB per window for A plus as much per CTA its Schur sum is split over).  Above 640 rows the factorisation
 * is always spread over the GPU.  The same limits hold for kba_solve_window / kba_solve_batch, which create such a batch. */
int kba_batch_create(kba_handle* h, int32_t n_windows, const kba_window* w, kba_batch** out);
int kba_batch_upload(kba_batch* b, int32_t n_windows, const kba_window* w); /* re-upload state, same shapes */
/* resets to the uploaded state and solves; returns when every window is done.  Issued as ONE CUDA graph launch (the
 * Levenberg-Marquardt pass is the body of a conditional WHILE node, the device decides when the batch is done) unless the
 * handle runs on the legacy default stream, which cannot be captured: give the handle a stream of its own (kba_create does,
 * kba_set_stream with a created stream keeps it).  INTEGRATION.md lists the switches (KBA_GRAPH, ...). */
int kba_batch_solve(kba_batch* b, const kba_options* opt);
/* kba_batch_solve with one kba_options per window, opts[n_windows]: window i runs with opts[i] (thresholds, quantiles, trimming,
 * iteration counts, tolerances, time limit) and its results equal those of kba_batch_solve(b, &opts[i]) for that window bit for
 * bit.  precision must be the same in every entry (KBA_ERR_BAD_ARG otherwise); each entry is checked as kba_batch_solve checks
 * its one, before anything is uploaded, and kba_last_error names the window index.  The pass cap follows the largest iteration
 * counts; the host safety cap the largest solver_time_sec (none if some window has none).  The options live on the device and go
 * up only when they differ from the last solve's of the batch: a resident re-solve with the same options copies nothing more,
 * and changing only the options does not rebuild the solve's CUDA graph. */
int kba_batch_solve_opts(kba_batch* b, const kba_options* opts);
int kba_batch_download(kba_batch* b, kba_result* res);
int kba_batch_transfer_bytes(kba_batch* b, int64_t* h2d_bytes, int64_t* d2h_bytes); /* of the last upload / download */
int kba_batch_jacobian_pass(kba_batch* b, const kba_options* opt, int32_t repeats, float* ms_out); /* residual/Jacobian kernel only */
void kba_batch_destroy(kba_batch* b);
/* counters for bench.py: kernels launched / device ms per kernel family since the last reset */
typedef struct kba_counters {
    int64_t launches_total;
    int64_t launches_jacobian, launches_prep, launches_schur, launches_solve, launches_backsub, launches_cost, launches_update, launches_trim;
    double ms_jacobian;  /* CUDA-event time of the residual/Jacobian kernel launches when timing is enabled */
    int64_t jacobian_obs;/* observations processed by those launches */
} kba_counters;
int kba_get_counters(kba_handle* h, kba_counters* out, int reset);
int kba_enable_kernel_timing(kba_handle* h, int on);

/* ---- ONE large window sharded over several GPUs by landmark blocks (BASELINE config 5) --------------------------------
 * Every rank (one process per GPU) holds ALL keyframes and a block of the landmarks with their observations and ground-plane
 * residuals (limo_b200/parallel.py::shard_window shows the partition: a ground-plane residual belongs to the rank owning its
 * landmark).  Per linearisation the ranks exchange, in ONE sum all-reduce, the reduced system [S | rhs] their landmarks
 * contribute to, the per-keyframe J^T J blocks, for a window with ground-plane residuals the per-keyframe 10 x 10
 * (pose | normal | distance) blocks and the ground-plane cost, and the cost partials; per LM iteration the model-decrease,
 * step and candidate-cost scalars.  The reduced solve and the LM controller then run replicated and bit-identically on every
 * rank (the all-reduce delivers the same bits everywhere).  Trimming quantiles are taken over all ranks' landmarks.  There is
 * no reference counterpart (the reference is single-process); north_star asks for it.
 * Two kinds of communicator: NCCL (kba_shard_comm_create, one process per GPU) and in process (kba_shard_comm_create_local:
 * W handles of one process on one device, each rank's kba_batch_solve called from its own host thread; its all-reduce adds the
 * ranks' buffers in rank order).  Sharded solves on the in-process kind always run kernel by kernel on the stream (no graph). */
typedef struct kba_shard_comm kba_shard_comm;
#define KBA_SHARD_ID_BYTES 128
int kba_shard_unique_id(void* id_out);  /* KBA_SHARD_ID_BYTES; rank 0 creates it, the host broadcasts it to all ranks */
int kba_shard_comm_create(kba_handle* h, int32_t rank, int32_t world, const void* id, kba_shard_comm** out); /* collective */
/* world communicators out[0..world-1] of one process, rank r driving handles[r]; 1 <= world <= 16, distinct handles on one
 * device.  If one rank's kba_batch_set_shard or kba_batch_solve fails, the ranks waiting for it in an exchange return
 * KBA_ERR_NCCL instead of blocking, and so does every later exchange of the group: create a new one.  Destroy each out[r]. */
int kba_shard_comm_create_local(kba_handle* const* handles, int32_t world, kba_shard_comm** out);
void kba_shard_comm_destroy(kba_shard_comm* c);
/* b holds this rank's shard; lm_begin = index of its first landmark in the whole window, lm_total = landmarks of the
 * whole window.  Collective: every rank calls it, and afterwards kba_batch_solve is a collective call that every rank must make.
 * Restrictions: one window per batch (KBA_ERR_BAD_ARG; up to 128 keyframes, as kba_batch_create takes), every free keyframe is
 * in the program, and every shard must size the
 * same reduced system (KBA_ERR_BAD_ARG otherwise): with plane_reg_weight = 0 a shard has plane rows only if it holds
 * ground-plane residuals, so then every shard must hold some, or none.  The window's scalars -- scale regulariser,
 * plane_reg_weight, plane_dist_fixed, speed prior -- are given to every shard with the same values (shard_window copies them).
 * Which keyframes' plane blocks are variable is decided for the whole window: kba_batch_solve first gathers the keyframe of
 * every rank's ground-plane residuals (one all-reduce of lm_total doubles), and every rank applies the window-wide trimming
 * decisions to that list, so a rank without ground-plane residuals takes the same layout as the plain solve of the window. */
int kba_batch_set_shard(kba_batch* b, kba_shard_comm* comm, int32_t lm_begin, int32_t lm_total);

/* ---- persistent, device-resident sliding window (SURVEY 8(f) row 3) ------------------------------------------------------------
 * The reference rebuilds the whole ceres::Problem for every solve() (bundle_adjuster_keyframes.cpp:635-637) and kba_solve_window
 * re-packs and re-uploads the whole window likewise.  A kba_track keeps what push() has seen on the device instead:
 *   - every pushed keyframe's pose, plane and measurements (landmark slot, camera, u, v, d) in one arena, uploaded ONCE at push;
 *   - landmark positions / weights by caller-assigned dense slot (the caller keeps LandmarkId -> slot), updated in place by solves.
 * kba_track_solve() then takes only the small per-solve lists (which keyframe slots are active, in ascending id order, with their
 * fixation; which landmark slots are selected, in ascending id order; the ground-plane attachments; the regulariser scalars),
 * gathers the window's CSR ON THE DEVICE (k_track_* in kba_pack.cu), packs and solves it exactly like kba_solve_window, writes
 * poses / planes / landmarks back into the store and returns them.  The window it builds is, array for array, the one the caller
 * would have passed to kba_solve_window, so the results are bit-identical (tests/test_track.py).
 * Capacities are fixed at creation; a window beyond `win_*` must go through kba_solve_window.  Not thread-safe (one handle). */
typedef struct kba_track kba_track;
typedef struct kba_track_caps {
    int32_t max_keyframes;     /* keyframe slots in the store (active or not)        */
    int32_t max_landmarks;     /* landmark slots                                      */
    int32_t max_measurements;  /* arena entries over all stored keyframes             */
    int32_t win_keyframes;     /* largest window: keyframes (win_rows = 0: <= 30, and a solve with ground-plane blocks takes <= 18) */
    int32_t win_landmarks;     /*                 selected landmarks                  */
    int32_t win_observations;  /*                 observations                        */
    int32_t win_ground;        /*                 ground-plane residuals, or candidates of a device attachment (<= win_landmarks) */
    int32_t win_rows;          /*                 reduced-system rows: 6 per keyframe, 10 with plane blocks, plus one.  0: the fused
                                                  path's limits above; else 6 * win_keyframes + 1 .. 640 (the track's own
                                                  limit; kba_batch_create takes more), see kba_track_solve */
} kba_track_caps;
int kba_track_create(kba_handle* h, const kba_track_caps* caps, int32_t n_cam, const double* cam_intr, const double* cam_pose,
                     kba_track** out);
void kba_track_destroy(kba_track* t);
/* push(): keyframe `kf_slot` (re-usable after kba_track_drop_keyframe) with pose, plane (4, may be NULL) and its measurements */
int kba_track_push_keyframe(kba_track* t, int32_t kf_slot, const double* pose7, const double* plane4, int32_t n_meas,
                            const int32_t* lm_slot, const int32_t* cam, const float* u, const float* v, const float* d);
int kba_track_drop_keyframe(kba_track* t, int32_t kf_slot);  /* its arena space is reclaimed by compaction when needed */
/* landmark state the host changes outside a solve: initial positions of new landmarks (push(), cpp:318-319), weights and
 * positions touched by the caller; any of pos / weight may be NULL */
int kba_track_set_landmarks(kba_track* t, int32_t n, const int32_t* lm_slot, const double* pos3, const double* weight);
int kba_track_set_keyframe_pose(kba_track* t, int32_t kf_slot, const double* pose7, const double* plane4);
/* the same for n keyframes with ONE copy (pose7s [n*7], plane4s [n*4] or NULL): what solve() sends for its active keyframes */
int kba_track_set_keyframe_poses(kba_track* t, int32_t n, const int32_t* kf_slot, const double* pose7s, const double* plane4s);
/* one solve() on the stored window; `sel` carries sizes, the scalar members and the ground-plane lists of kba_window (gp_lm =
 * index into lm_slot), its keyframe / landmark / observation arrays are ignored; scale_weight < 0 asks for the reference's own rule
 * (cpp:703-716: 1000, or 1000 / (depth + ground-plane residuals) beyond ten of them; plane_dist_fixed by cpp:722-728), evaluated
 * on the device from the gathered window so that the host need not visit a single observation.  Results: res->kf_pose / kf_plane [n_kf],
 * res->lm_pos / lm_rejected [n_lm] in selection order.
 * Ground-plane residuals come in one of two ways:
 *   - host lists: gp_lm, gp_kf and gp_weight, attached and weighted by the caller as kba_window describes them;
 *   - device attachment: n_gp > 0, gp_lm lists CANDIDATE ground landmarks (indices into lm_slot, strictly ascending) and gp_kf,
 *     gp_weight are both NULL.  Each candidate is attached on the device exactly as addGroundPlaneResiduals (cpp:517-562) does it,
 *     from the store's current poses, planes and landmark positions: keyframes in window order, a keyframe whose plane distance is
 *     < -10 skipped, distance |R(q) p + t| (first strict minimum wins, a NaN is never a minimum), kept iff the distance is < 25
 *     with weight 10 (1 - d / 25); kept residuals in candidate order.  The arithmetic is that of the reference's host code without
 *     FMA contraction, so the lists equal those a host computes from the same state bit for bit.  The caller sends 4 B per
 *     candidate instead of 16 B per residual, and need not keep landmark positions on the host.
 * plane_reg_weight < 0 asks for the reference's rule (cpp:717-719): 10 iff at least one ground-plane residual is in the window
 * (with either kind of lists).  Errors, all before anything is uploaded: only one of gp_kf / gp_weight NULL, candidates not
 * strictly ascending or out of range: KBA_ERR_BAD_ARG; more residuals or candidates than win_ground: KBA_ERR_CAPACITY.
 * Window size: a request has rows = (planes ? 10 : 6) * n_kf + 1 reduced rows, where planes = n_gp > 0 or plane_reg_weight > 0.
 *   - caps.win_rows = 0: a request that can carry plane blocks (ground-plane lists of either kind, or plane_reg_weight != 0) with
 *     10 * n_kf + 1 > 184 (more than 18 keyframes) is KBA_ERR_CAPACITY -- the rule by which kba_batch_create keeps a window on the
 *     fused path, so that the track and kba_solve_window run the same solver.
 *   - caps.win_rows > 0: a request with rows > win_rows is KBA_ERR_CAPACITY.  A track with win_rows > 184 owns a second solver,
 *     sized for win_keyframes and win_rows, on the large-window path (k_schur_syrk and the row-major or split factorisation),
 *     packed on the device like the fused one.  Each solve goes to the solver kba_batch_create would choose for the window: the
 *     fused one iff rows <= 184 (so windows that fit the fused path keep its results bit for bit), the large one otherwise.  The
 *     Schur split, the factorisation and each window's system size follow the solved window, as kba_batch_create derives them.
 * solves[].num_residual_blocks counts the attached residuals; with nothing attached, kf_plane comes back bit-equal to the stored
 * planes, so a caller may always copy planes back.  One exception to bit-equality with kba_solve_window: the solver path and the
 * Schur kernel variant are chosen before the attachment, counting plane rows whenever candidates are given.  With nothing attached
 *   - an 18-free-keyframe window runs the seven-slot fused kernel where kba_solve_window runs the six-slot one;
 *   - a window of 19 to 30 keyframes runs the large-window path where kba_solve_window, seeing a plane-free window, runs the fused
 *     one.
 * Such results agree with kba_solve_window to the solver's tolerances (translations to 1e-6 m, the cost to 1e-8 relative), not
 * bit for bit. */
int kba_track_solve(kba_track* t, int32_t n_kf, const int32_t* kf_slot, const uint8_t* kf_fixed, int32_t n_lm, const int32_t* lm_slot,
                    const kba_window* sel, const kba_options* opt, kba_result* res);
int kba_track_transfer_bytes(kba_track* t, int64_t* h2d_last_solve, int64_t* d2h_last_solve, int64_t* h2d_pushes_total);

/* ---- landmark selection on the stored window (SURVEY row A17) ---------------------------------------------------------
 * The per-landmark quantities of limo's selection chain (landmark_selector.hpp:118-253 with LandmarkRejectionSchemeCheirality and
 * LandmarkSparsificationSchemeVoxel, as facade/landmark_selection.cpp states them), computed from what the store holds: keyframe
 * poses, the measurement arena, landmark positions by slot, the cameras.  A caller that ranks them as LandmarkSelector::select
 * does (the partial sorts, the std::rand shuffle of the middle bin, the bin caps) gets its selection bit for bit;
 * kba_track_rank_landmarks (below) does that ranking on the device instead.  A request:
 *   - kf_slot [n_kf]: the active keyframes in ascending timestamp (= id) order, every one pushed; the last one is the newest;
 *   - lm_slot [n_cand]: the candidates, i.e. the active landmarks minus the outliers, in ascending id order (<= max_landmarks).
 * Per candidate c:
 *   - cheiral[c] = 1 iff z of cam * (kf * pos) is not below 0 for every arena entry of a listed keyframe that measures it;
 *   - among the cheirality survivors (labelled in candidate order), the voxel scheme's steps 1-5: the position in the newest
 *     keyframe's frame rounded to float, PassThrough z in [-20, 100], distance (double) to the path of the listed keyframes'
 *     positions; far bin iff it is not below roi_far; the others on the float voxel grid of voxel_size (one point per voxel,
 *     the centroid, labelled by the voxel's first candidate); middle bin iff the centroid's distance is not below roi_middle.
 *     bin[c] = 0 near-bin voxel representative, 1 middle-bin representative, 2 far, -1 dropped (not cheiral, PassThrough,
 *     not the first candidate of its voxel);
 *   - near_order[0..*n_near): the near representatives' candidate indices in ascending voxel index (the scheme's ids_near);
 *   - flow[c] (near representatives): calcFlow(use_mean = false), per camera index the sum of the pixel distances between
 *     consecutive observations in keyframe order, the maximum over the cameras; NaN for a landmark no camera saw twice, and for
 *     every other candidate.  Camera indices stand for the caller's camera ids: they must be in the same order;
 *   - seen[c] (every candidate): how many listed keyframes measure it (chooseFarLmIds).
 * Every float operation is the host code's, in its order, without contraction: the quantities equal the host's bit for bit.
 * One upload (the lists), one launch sequence, one download; the first call allocates the buffers for the track's capacities,
 * later calls allocate nothing.  kba_track_transfer_bytes then reports this call's upload and download: 4 * (n_kf + n_cand)
 * and 18 * n_cand + 16 bytes.  kba_track_group_select_landmarks (below) selects for every track of a group at once.
 * Errors, before anything is uploaded: a null pointer, n_kf < 1, a slot out of range or listed twice, a keyframe slot not pushed,
 * a voxel size that is not finite and positive: KBA_ERR_BAD_ARG; more keyframes or candidates than the track has slots:
 * KBA_ERR_CAPACITY. */
typedef struct kba_select_params {
    double voxel_size[3];      /* LandmarkSparsificationSchemeVoxel::Parameters::voxel_size_xyz                    */
    double roi_far, roi_middle; /* roi_far_xyz[0], roi_middle_xyz[0]: distances to the keyframe path              */
} kba_select_params;
typedef struct kba_select_out {  /* caller-owned arrays of n_cand entries */
    uint8_t* cheiral;
    int8_t* bin;
    int32_t* near_order;
    int32_t* n_near;          /* one value */
    double* flow;
    int32_t* seen;
} kba_select_out;
int kba_track_select_landmarks(kba_track* t, int32_t n_kf, const int32_t* kf_slot, int32_t n_cand, const int32_t* lm_slot,
                               const kba_select_params* p, kba_select_out* out);

/* ---- many persistent windows in one launch: track groups -----------------------------------------------------------------
 * kba_track_solve solves one window per call, which leaves the GPU mostly idle.  A group solves one window of each of its tracks
 * as ONE batch (one kba_batch_solve: one CUDA graph launch), with the persistent store of every track: per solve only the
 * selection lists travel, for all tracks together in one copy.  For several vehicles, offline reprocessing of many sequences or
 * parameter sweeps over one recording.
 *   - Membership: every track belongs to `h` (same device and stream) and appears once; an empty group, a duplicate or a track
 *     of another handle is KBA_ERR_BAD_ARG.  Destroy a group before its tracks (as a batch before its handle).  A track of a
 *     group may still be solved alone with kba_track_solve; between calls its store is the single source of truth.
 *   - Memory: the group owns one capacity-shaped window per track, a copy of the allocations of the track's own batch (about
 *     10 MB for a track sized like config 2, 30 keyframes / 3k landmarks / 40k observations).
 *   - Validation: every request with n_kf != 0 is checked exactly as kba_track_solve checks its arguments.  If one fails, the
 *     call returns that request's code before anything is uploaded or launched, kba_last_error names the track index, and no
 *     store changes.
 *   - Results: window i is the window kba_track_solve would build for track i; its results go to res[i] and into track i's
 *     store exactly as for a single solve.  One kba_options applies to the whole group, or one per track with the _opts
 *     forms (kba_track_group_solve_opts, kba_track_group_solve_ranked_opts, kba_track_group_adjust_pose_opts: a parameter
 *     sweep over one recording, each track a grid point).  precision is the same for every track.  solver_time_sec is checked
 *     on the group's shared passes: each window's inner solves are timed on the device while the passes of the whole group run, so
 *     a window's budget includes the time its group's other windows take.
 *   - Launch configuration, decided per solve from the windows that are solved: the largest rig rank, the seven-slot Schur
 *     kernel if any window needs more than 176 reduced rows, and from these the fused-linearisation switch, as kba_batch_solve
 *     decides for any batch.  The whole group takes the large-window path when one of its requests has more than 184 rows
 *     (kba_track_solve), so the group owns a second solver iff one of its tracks has win_rows > 184.  A window in a mixed group can therefore run a different kernel variant than alone (e.g. a
 *     multi-camera rig turns the fused linearisation off for every window) and round differently in the last bits.
 *   - Skipping: a request with n_kf == 0 sits the solve out: its store is untouched, res[i] gets status KBA_OK and
 *     num_solves 0, its output arrays are not written.  A call in which every track sits out returns at once. */
typedef struct kba_track_group kba_track_group;
typedef struct kba_track_request {
    int32_t n_kf;               /* 0: this track sits this solve out (store untouched, result status KBA_OK, num_solves 0) */
    const int32_t* kf_slot;     /* the fields mean exactly what the arguments of kba_track_solve mean */
    const uint8_t* kf_fixed;
    int32_t n_lm;
    const int32_t* lm_slot;
    const kba_window* sel;      /* sizes, scalars and ground-plane lists or candidates, as for kba_track_solve; a group may mix
                                   device-attached, host-list and plane-free requests */
} kba_track_request;
int kba_track_group_create(kba_handle* h, int32_t n_tracks, kba_track* const* tracks, kba_track_group** out);
void kba_track_group_destroy(kba_track_group* g);
/* req[n_tracks], res[n_tracks] */
int kba_track_group_solve(kba_track_group* g, const kba_track_request* req, const kba_options* opt, kba_result* res);
/* kba_track_group_solve with opts[n_tracks]: track i's window runs with opts[i], and its results and store equal those of
 * kba_track_solve with opts[i] bit for bit.  The entries of the tracks that solve are checked as kba_batch_solve_opts checks
 * them, before anything is uploaded, and kba_last_error names the track index; a track that sits the solve out (n_kf == 0) does
 * not read its entry.  The options travel in the lists' copy, and only when they differ from the group's last solve's. */
int kba_track_group_solve_opts(kba_track_group* g, const kba_track_request* req, const kba_options* opts, kba_result* res);
/* upload / download of the last group solve, pose-only call, selection, creation, upkeep, flow or reclaim call or store write,
 * counted as kba_track_transfer_bytes counts them */
int kba_track_group_transfer_bytes(kba_track_group* g, int64_t* h2d_last_solve, int64_t* d2h_last_solve);

/* ---- evaluation of the stored window: residuals, costs and trimming decisions at the store's state --------------------------
 * How well the stored window fits its measurements, without solving it: for threshold tuning, outlier labelling, checking a
 * track after kba_track_load or monitoring a long drive.  A request is a kba_track_request exactly as for kba_track_solve (host
 * ground-plane lists or device-attached candidates, scale_weight < 0 and plane_reg_weight < 0 resolved by the same rules), and the
 * window evaluated is the one kba_track_solve would build for it, array for array, at the store's current poses, planes and
 * landmark positions.  Every value comes from the solver's own device code, so the total cost equals the initial_cost of
 * solves[0] of kba_track_solve on the same request to the last bits of its summation order.
 * The observation order is the window's own: landmarks in lm_slot order, then keyframes in kf_slot order, then cameras ascending.
 *   - n_obs: the window's observation count, always written;
 *   - obs_lm, obs_kf, obs_cam [n_obs]: index into lm_slot, index into kf_slot, the store's camera;
 *   - residual [3 n_obs]: the rows (u, v, depth) of the observation's residual before any loss or weight: projection minus
 *     measurement in pixels, z_cam - d in metres (0 without a depth, d <= 0);
 *   - rho [2 n_obs]: the scaled Cauchy loss w b log(1 + s / b) of the reprojection block (s = u^2 + v^2, b = reprojection_thres^2)
 *     and of the depth block (s = depth^2, b = depth_thres^2; 0 without a depth), w the landmark's weight; the cost is half
 *     their sum.  An observation with |z_cam| < 0.01 gets NaN rows and losses and sets `failed`;
 *   - trim_repr, trim_depth [n_lm]: the trimming values of solveTrimmed at this state: per landmark the largest raw block norm
 *     (|(u, v)|, |depth|) over its observations, -1 without one;
 *   - rejected_repr, rejected_depth [n_lm]: 1 where TrimmerQuantile at opt's reprojection / depth quantile over those values
 *     rejects the landmark (min_residual_groups applies; ties broken by landmark index), the selection code of the solver;
 *   - n_gp, gp_lm, gp_kf, gp_weight, gp_residual [n_gp]: the attached ground-plane residuals (the request's host lists, or what the
 *     device attachment kept, as kba_track_solve attaches them) with their height residual n . (R p + t) + dist; the caller
 *     allocates win_ground entries;
 *   - cost[6]: reprojection, depth, ground plane (HuberLoss(gp_huber) scaled by the weights), scale regulariser, plane chain and
 *     their total, each 1/2 sum rho as ceres counts it;
 *   - failed: 1 if some observation has |z_cam| < 0.01.
 * Any output array may be NULL.  Per-observation arrays hold obs_capacity entries: if the window has more observations, the call
 * returns KBA_ERR_CAPACITY after writing n_obs (and nothing else), and the caller retries with larger arrays.
 * Errors, before anything is uploaded: those of kba_track_solve, and opt->precision != 0 (FP64 only): KBA_ERR_BAD_ARG.
 * The store is never modified: a later solve gives the results it would give without the evaluation, bit for bit, and a ranking
 * stays valid.  One upload (the lists, and a record per window), one launch sequence (the gather of kba_track_solve and two
 * kernels), one download and one synchronisation; the first call allocates the track's (group's) output staging for its
 * capacities.  kba_track_transfer_bytes (kba_track_group_transfer_bytes) then report this call's upload and download.
 * The group forms evaluate one request per track in one launch sequence: out[i] is bit for bit what kba_track_evaluate gives
 * track i for req[i]; a request with n_kf == 0 sits the call out (out[i] is not written); every request is checked first and a
 * failing one returns its code with kba_last_error naming its track; the _opts form takes one kba_options per track. */
typedef struct kba_evaluate_out {  /* caller-owned arrays, any of them may be NULL */
    int32_t obs_capacity;       /* entries of obs_lm, obs_kf, obs_cam (residual: 3 per entry, rho: 2 per entry)             */
    int32_t n_obs;              /* written by the library                                                                   */
    int32_t n_gp;
    int32_t failed;
    double cost[6];             /* reprojection, depth, ground plane, scale regulariser, plane chain, total                 */
    int32_t* obs_lm;            /* [n_obs] */
    int32_t* obs_kf;
    int32_t* obs_cam;
    double* residual;           /* [3 n_obs] */
    double* rho;                /* [2 n_obs] */
    double* trim_repr;          /* [n_lm] */
    double* trim_depth;
    uint8_t* rejected_repr;     /* [n_lm] */
    uint8_t* rejected_depth;
    int32_t* gp_lm;             /* [win_ground] */
    int32_t* gp_kf;
    double* gp_weight;
    double* gp_residual;
} kba_evaluate_out;
int kba_track_evaluate(kba_track* t, const kba_track_request* req, const kba_options* opt, kba_evaluate_out* out);
/* req[n_tracks], out[n_tracks] */
int kba_track_group_evaluate(kba_track_group* g, const kba_track_request* req, const kba_options* opt, kba_evaluate_out* out);
/* opts[n_tracks]: track i is evaluated with opts[i] (its thresholds and quantiles); a track that sits out does not read its entry */
int kba_track_group_evaluate_opts(kba_track_group* g, const kba_track_request* req, const kba_options* opts, kba_evaluate_out* out);

/* ---- landmark selection for every track of a group in one launch sequence -------------------------------------------------
 * kba_track_select_landmarks for one request per track, each on its own track's store, as one window each of one launch sequence.
 *   - Results: out[i] holds exactly what kba_track_select_landmarks(tracks[i], ...) writes for the same request, bit for bit:
 *     cheiral, bin, near_order, *n_near, flow (NaN in the same places) and seen.  A single call is a one-request group call of
 *     the same host code and kernels.
 *   - Sitting out: a request with n_kf == 0 leaves out[i]'s arrays unwritten and sets *out[i].n_near = 0 (n_near must not be
 *     NULL).  A call in which every request sits out returns at once: no upload, no launch.
 *   - Validation: every other request is checked as kba_track_select_landmarks checks its arguments (n_kf < 0 is KBA_ERR_BAD_ARG)
 *     before anything is uploaded.  If one fails, the call returns that request's code, kba_last_error names the track index,
 *     and no out[i] is written.
 *   - Transfers: one upload (every request's lists and the argument records of the windows), one launch sequence, one download
 *     and one synchronisation per call.  Over the W requests that do not sit out, kba_track_group_transfer_bytes then reports
 *         h2d = 4 * sum(n_kf + n_cand) + R * (W - 1)
 *         d2h = 18 * sum(n_cand) + 16 * W
 *     where R is the size of one window's argument record, a constant of the library build that the header does not fix
 *     (the first window's record travels in the launch parameters).  With W = 1 these are kba_track_transfer_bytes' counts
 *     after a single selection, and 0 / 0 when every request sits out.
 *   - Memory: each member track's selection scratch (allocated at the first selection of that track by either entry point,
 *     for the track's capacities) is used by both entry points, and the staging of kba_track_select_landmarks is allocated at
 *     the track's first single call only; calls are serial on the handle's stream, so a track may
 *     still be selected alone between group calls.  The group adds only its staging for the lists, the argument records and
 *     the outputs (pinned and device, sized for its tracks' capacities), allocated at its first call in which some request
 *     does not sit out. */
typedef struct kba_select_request {
    int32_t n_kf;                     /* 0: this track sits the call out; < 0: KBA_ERR_BAD_ARG                         */
    int32_t n_cand;
    const int32_t* kf_slot;           /* [n_kf]   as for kba_track_select_landmarks                                  */
    const int32_t* lm_slot;           /* [n_cand] as for kba_track_select_landmarks                                  */
    const kba_select_params* params;  /* per request, so that a sweep can vary the voxel size and ROIs per track       */
} kba_select_request;
/* req[n_tracks], out[n_tracks] */
int kba_track_group_select_landmarks(kba_track_group* g, const kba_select_request* req, kba_select_out* out);

/* ---- landmark creation of push() on the stored window (SURVEY row A18) ------------------------------------------------
 * What BundleAdjusterKeyframes::push() does for every landmark a pushed keyframe measures for the first time
 * (bundle_adjuster_keyframes.cpp:289-382, facade/bundle_adjuster_keyframes.cpp), computed from what the store holds: keyframe
 * poses, the measurement arena, the cameras.  The caller pushes the keyframe (kba_track_push_keyframe), then asks for its new
 * landmarks here instead of keeping a host copy of the window to triangulate from.  A request:
 *   - kf_slot [n_kf]: the active keyframes in ascending timestamp (= id) order, every one pushed, the new keyframe among them;
 *   - kf_new: the index in kf_slot of the keyframe just pushed;
 *   - lm_slot [n_new]: the landmarks it measures that do not exist yet (the caller keeps LandmarkId -> slot).
 * Per requested landmark c, in request order:
 *   - has depth (flags bit 1) iff an arena entry of kf_new for it has d >= 0 (containsDepth; a NaN depth is no depth).  Then the
 *     first entry of kf_new for it in arena order that calculateLandmark(kf, id) does not skip (it skips d < 0 only, so a NaN
 *     depth before the valid one is taken and the position is NaN, as on the host) is back-projected: x = (u - cx) z / f,
 *     y = (v - cy) z / f, z = d, and pos = (cam * kf).inverse() * (x, y, z);
 *   - else its rays, over the listed keyframes in list order and a keyframe's entries for it in arena order: each is
 *     normalized(intrin_inv * (u, v, 1)) with pose (cam * kf).inverse(), intrin_inv the cofactor inverse of K.  With fewer than
 *     two rays it is not created; else pos = triangulate_rays of the facade: sum (I - r r^T) inverted, times sum (I - r r^T) t.
 *     Arena order within a keyframe must be the caller's camera-id order (Keyframe::cameras_), as for the select call's flow;
 *   - created (flags bit 0): pos goes into the store's slot with weight 1 (Landmark::weight's default) and to out.pos[3c..3c+3);
 *     a landmark that is not created leaves its store slot untouched and gets NaN in out.pos.
 * Every double operation is the facade's host code's, in its order, without contraction: the positions equal the host push()'s
 * bit for bit, and a degenerate triangulation (parallel rays) gives the host's inf or NaN.
 * One upload (the lists), one launch sequence, one download; the first call allocates the buffers for the track's capacities,
 * later calls allocate nothing.  kba_track_transfer_bytes then reports this call's upload and download: 4 * (n_kf + n_new) and
 * 25 * n_new bytes.
 * Errors, before anything is uploaded or written: a null pointer, n_kf < 1, n_new < 0, kf_new outside [0, n_kf), a slot out of
 * range or listed twice, a keyframe slot not pushed: KBA_ERR_BAD_ARG; more keyframes or landmarks than the track has slots:
 * KBA_ERR_CAPACITY.
 * kba_track_group_create_landmarks does this for one request per track of a group in one launch sequence (window = request):
 *   - out[i] and track i's store get exactly what kba_track_create_landmarks(tracks[i], &req[i], &out[i]) writes, bit for bit;
 *   - a request with n_kf == 0 sits the call out: out[i] is not written, its store is untouched; a call in which every request
 *     sits out returns at once (no upload, no launch);
 *   - every other request is checked as the single call checks it before anything is uploaded; if one fails, the call returns
 *     its code, kba_last_error names the track index, and no output or store is written;
 *   - over the W requests that do not sit out, kba_track_group_transfer_bytes then reports
 *         h2d = 4 * sum(n_kf + n_new) + R * (W - 1),   d2h = 25 * sum(n_new)
 *     where R is the size of one window's argument record, a constant of the library build (the first window's record travels
 *     in the launch parameters);
 *   - memory: each track's creation scratch is shared by both entry points; the group adds its own staging, sized for its
 *     tracks' capacities and allocated at its first call in which some request does not sit out. */
typedef struct kba_create_request {
    int32_t n_kf;               /* 0 (group call): this track sits the call out                                        */
    int32_t kf_new;             /* index into kf_slot of the keyframe just pushed                                      */
    int32_t n_new;
    int32_t reserved_;
    const int32_t* kf_slot;     /* [n_kf]  the active keyframes in ascending id order, every one pushed                */
    const int32_t* lm_slot;     /* [n_new] the landmarks kf_new measures that do not exist yet                         */
} kba_create_request;
typedef struct kba_create_out {  /* caller-owned arrays */
    double* pos;                /* [3 * n_new] created positions, NaN where not created                                */
    uint8_t* flags;             /* [n_new] bit 0 created, bit 1 has depth                                              */
} kba_create_out;
int kba_track_create_landmarks(kba_track* t, const kba_create_request* req, kba_create_out* out);
/* req[n_tracks], out[n_tracks] */
int kba_track_group_create_landmarks(kba_track_group* g, const kba_create_request* req, kba_create_out* out);

/* ---- window upkeep on the stored window: deactivateKeyframes and the AddDepth scheme's costs ------------------------------
 * The two steps of limo's keyframe step that read every active keyframe's measurements, computed from what the store holds, so
 * that a track (group) user keeps no host copy of the window's measurements.  Both take the slot contract of the select and
 * create calls: a keyframe's arena entries come in landmark-id order (one run per landmark), so the distinct landmarks of a
 * keyframe are the first entries of its runs; the caller keeps LandmarkId -> slot.  Everything else is as for the create call:
 *   - one upload (the lists), one launch sequence, one download, one synchronisation per call; the first call of a track by
 *     either entry point allocates its upkeep scratch, its first single call its staging, later calls allocate nothing;
 *   - every request is checked before anything is uploaded or written; null pointers, n_kf < 1, a negative size, a keyframe
 *     slot not pushed or listed twice, a landmark slot out of range or listed twice: KBA_ERR_BAD_ARG; more keyframes or
 *     landmarks than the track has slots: KBA_ERR_CAPACITY;
 *   - the group forms serve one request per track in one launch sequence (window = request): out[i] is bit for bit what the
 *     single call writes for req[i]; a request with n_kf == 0 sits the call out (out[i] not written; a call in which every
 *     request sits out returns at once); a failing request returns its code, kba_last_error names its track, nothing is written;
 *   - memory: a track's upkeep scratch is shared by both entry points; a group adds its own staging, sized for its tracks'
 *     capacities and allocated at its first call in which some request does not sit out.
 *
 * kba_track_deactivate_keyframes: BundleAdjusterKeyframes::deactivateKeyframes(min_connecting, min_window, max_window)
 * (bundle_adjuster_keyframes.cpp:907-987).  A request:
 *   - kf_slot [n_kf]: the active keyframes in ascending id order, every one pushed; the last one is the newest;
 *   - lm_slot [n_lm]: the active landmarks (active_landmark_ids_; a slot never created is allowed), any order.
 * Outputs, all integer arithmetic, so exactly the facade's:
 *   - kf_common[k]: the number of distinct landmark slots of keyframe k's arena entries that the newest keyframe's entries
 *     also name (getCommonLandmarkIds: all of its measurements, not only active landmarks), for every k;
 *   - kf_active[k] with n = n_kf - 1 - k: 0 if n > max_window - 1, else 1 if n < min_window - 1, else kf_common[k] > min_connecting;
 *   - lm_active[j]: 1 iff landmark j is measured by some keyframe with kf_active = 1 (the new active_landmark_ids_).
 * The caller still fixes the two oldest survivors.  Transfers (kba_track_transfer_bytes; over the W requests that do not sit out
 * for kba_track_group_transfer_bytes, R the size of one window's argument record, a constant of the library build):
 *         h2d = 4 * sum(n_kf + n_lm) + R * (W - 1),   d2h = sum(5 * n_kf + n_lm)
 *
 * kba_track_depth_costs: the quantities of LandmarkSelectionSchemeAddDepth::getSelection (landmark_selection_scheme_add_depth.cpp:
 * 16-75) with limo's sorter (mono_lidar.cpp:418-429: float(local.norm())).  A request:
 *   - kf_slot [n_kf]: the active keyframes in ascending id order (the scheme's FrameIndex i is kf_slot[i], 0 the oldest);
 *   - lm_slot [n_elig]: the eligible landmarks in ascending id order (non_rejected ∩ comparator; for limo is_ground_plane);
 *   - cap: the capacity of out.cand / out.cost; below B = sum over k of min(n_elig, arena entries of kf_slot[k]): KBA_ERR_CAPACITY.
 * Outputs: for every keyframe k, the pairs (cand, cost) of the eligible landmarks k measures at off[k] .. off[k + 1), in arena
 * order (ascending id: the order of the host's cost vector); cand is the index into lm_slot, cost the host's value bit for bit:
 * worst = -DBL_MAX folded by std::max(worst, double(float(|kf * pos|))) over the keyframe's entries of that landmark -- a NaN
 * norm (a landmark created from a NaN depth has a NaN position) leaves -DBL_MAX.  The caller then runs the facade's
 * std::partial_sort over each off[ind] .. off[ind + 1) for its (ind, wanted) entries and gets the scheme's selection bit for
 * bit, ties and -DBL_MAX included.  Transfers (as above, B_w the bound of request w):
 *         h2d = 4 * sum(n_kf + n_elig) + R * (W - 1),   d2h = sum(4 * n_kf + 12 * B_w) */
typedef struct kba_deactivate_request {
    int32_t n_kf;               /* 0 (group call): this track sits the call out                                        */
    int32_t n_lm;
    int32_t min_connecting, min_window, max_window;
    int32_t reserved_;
    const int32_t* kf_slot;     /* [n_kf] the active keyframes in ascending id order; the last one is the newest         */
    const int32_t* lm_slot;     /* [n_lm] the active landmarks                                                          */
} kba_deactivate_request;
typedef struct kba_deactivate_out {  /* caller-owned arrays */
    uint8_t* kf_active;         /* [n_kf] */
    int32_t* kf_common;         /* [n_kf] */
    uint8_t* lm_active;         /* [n_lm] */
} kba_deactivate_out;
int kba_track_deactivate_keyframes(kba_track* t, const kba_deactivate_request* req, kba_deactivate_out* out);
/* req[n_tracks], out[n_tracks] */
int kba_track_group_deactivate_keyframes(kba_track_group* g, const kba_deactivate_request* req, kba_deactivate_out* out);

typedef struct kba_depth_request {
    int32_t n_kf;               /* 0 (group call): this track sits the call out                                        */
    int32_t n_elig;
    int32_t cap;                /* entries of out.cand / out.cost                                                        */
    int32_t reserved_;
    const int32_t* kf_slot;     /* [n_kf] the active keyframes in ascending id order                                    */
    const int32_t* lm_slot;     /* [n_elig] the eligible landmarks in ascending id order                                */
} kba_depth_request;
typedef struct kba_depth_out {  /* caller-owned arrays */
    int32_t* off;               /* [n_kf + 1] keyframe k's pairs are off[k] .. off[k + 1)                                */
    int32_t* cand;              /* [cap] index into lm_slot                                                             */
    double* cost;               /* [cap] */
} kba_depth_out;
int kba_track_depth_costs(kba_track* t, const kba_depth_request* req, kba_depth_out* out);
/* req[n_tracks], out[n_tracks] */
int kba_track_group_depth_costs(kba_track_group* g, const kba_depth_request* req, kba_depth_out* out);

/* ---- keyframe selection on the stored window: the flow scheme's quantity ------------------------------------------------
 * KeyframeRejectionSchemeFlow::isUsable (keyframe_rejection_scheme_flow.cpp:17-74), the one scheme of limo's KeyframeSelector
 * (mono_lidar.cpp:447-453, mono_standalone.cpp:327-333) that reads stored measurements: the new frame's pixel positions against
 * those of the newest active keyframe, which the store already holds.  The rotation angle of KeyframeSelectionSchemePose, the
 * time rule of KeyframeSparsificationSchemeTime and the composition of the verdicts (KeyframeSelector::select) stay with the
 * caller.  A request:
 *   - kf_last: the slot of the newest active keyframe (the one with the largest time stamp among the caller's last_frames);
 *     it must be pushed.  In a group call kf_last < 0 sits the track out; in the single call it is KBA_ERR_BAD_ARG;
 *   - lm_slot, cam (or NULL: camera 0), u, v [n_meas]: the new frame's measurements whose landmark has a slot, in
 *     Keyframe::measurements_ order: one run per landmark, runs in ascending landmark id, cameras ascending inside a run (the run
 *     contract of kba_track_frame).  A measurement whose landmark has no slot cannot match (every landmark a pushed keyframe
 *     measures has one): the caller leaves it out.  n_meas == 0 is a valid request with no match;
 *   - min_median_flow: the scheme's parameter.
 * Outputs, every double operation the facade's, in its order, without FMA contraction, so bit for bit its flow scheme, NaN
 * included:
 *   - n_matched: the (landmark, camera) pairs of the frame that the newest keyframe also measures (hasMeasurement(lm, cam));
 *   - flow_sum: the sum, in request order, of sqrt(dx * dx + dy * dy) over the matched pairs, dx = double(u) - double(u_last),
 *     dy likewise;
 *   - mean_flow_sq: s = flow_sum; s /= n_matched; s * s (0 / 0 = NaN without a match);
 *   - usable: mean_flow_sq > min_median_flow * min_median_flow (0 for NaN): isUsable for a non-empty last_frames and a frame
 *     with measurements.  The two early returns stay with the caller: an empty last_frames is usable, a frame without
 *     measurements is not;
 *   - match [n_meas] (optional, NULL: not written): the index, among kf_last's measurements as pushed, of the matched entry, or -1.
 * As for the upkeep calls:
 *   - one upload, one launch sequence, one download, one synchronisation per call; the first call of a track by either entry
 *     point allocates the upkeep scratch (shared with the upkeep calls) if it is not there yet, its first single call its flow
 *     staging (sized for win_observations), later calls allocate nothing;
 *   - every request is checked before anything is uploaded or written: null pointers, n_meas < 0, kf_last not pushed, a slot or
 *     camera out of range, a slot that reappears after its run has ended, a camera not ascending inside a run: KBA_ERR_BAD_ARG;
 *     n_meas > win_observations: KBA_ERR_CAPACITY;
 *   - the group form serves one request per track in one launch sequence (window = request): out[i] is bit for bit what the
 *     single call writes for req[i]; a request with kf_last < 0 sits the call out (out[i] not written; a call in which every
 *     request sits out returns at once); a failing request returns its code, kba_last_error names its track, nothing is written.
 * Transfers (kba_track_transfer_bytes; over the W requests that do not sit out for kba_track_group_transfer_bytes, R the size of
 * one window's argument record, a constant of the library build; the cameras are uploaded also when cam is NULL, the match
 * indices downloaded also when match is NULL):
 *         h2d = 16 * sum(n_meas) + R * (W - 1),   d2h = sum(4 * n_meas + 24) */
typedef struct kba_flow_request {
    int32_t kf_last;            /* slot of the newest active keyframe; < 0 (group call): this track sits the call out          */
    int32_t n_meas;
    const int32_t* lm_slot;     /* [n_meas] runs as kba_track_frame's                                                          */
    const int32_t* cam;         /* [n_meas] or NULL (all camera 0)                                                              */
    const float* u, *v;         /* [n_meas] */
    double min_median_flow;
} kba_flow_request;
typedef struct kba_flow_out {   /* caller-owned */
    int32_t n_matched;
    uint8_t usable;
    uint8_t reserved_[3];
    double flow_sum;
    double mean_flow_sq;
    int32_t* match;             /* [n_meas] or NULL */
} kba_flow_out;
int kba_track_frame_flow(kba_track* t, const kba_flow_request* req, kba_flow_out* out);
/* req[n_tracks], out[n_tracks] */
int kba_track_group_frame_flow(kba_track_group* g, const kba_flow_request* req, kba_flow_out* out);

/* ---- free landmark slots of the stored window: recycle slots as keyframe slots are recycled --------------------------------
 * A keyframe slot is free again after kba_track_drop_keyframe; a landmark slot is free once no live keyframe (pushed and not
 * dropped) measures it, which only the store can tell a caller that keeps no host copy of the measurements.  A request names a
 * slot range [lo, hi), 0 <= lo <= hi <= max_landmarks (a caller with dense slots from 0 asks for [0, slots handed out)).
 * Outputs:
 *   - n_free and free_slot [0 .. n_free): the slots of the range that no arena entry of a live keyframe names, ascending;
 *   - pos [3 * n_free] and weight [n_free], each optional (NULL: not written): the store's current values of those slots, bit
 *     for bit.  A caller that evicts a landmark keeps them, and restores the landmark with kba_track_set_landmarks when its id is
 *     measured again (push() never re-creates a landmark that exists).
 * The caller allocates free_slot (and pos, weight) for the whole range, hi - lo entries.  Liveness is the caller's: the live
 * keyframe slots go up with the request (a dropped keyframe's entries stay in the arena until the next compaction).  The call
 * does not write the store: a slot handed out again must be written (kba_track_create_landmarks or kba_track_set_landmarks)
 * before any call reads it.  Integer work only, so the result is deterministic.  As for the upkeep calls:
 *   - one upload, one launch sequence, one download, one synchronisation per call; the first call of a track by either entry
 *     point allocates its upkeep scratch (shared with the upkeep and flow calls) if it is not there yet, its first single call
 *     its reclaim staging (sized for every keyframe slot and a range of max_landmarks), later calls allocate nothing.  An empty
 *     range (hi == lo) in the single call gives n_free = 0 without an upload or a launch;
 *   - every request is checked before anything is uploaded or written: a null pointer (free_slot may be NULL only for an empty
 *     range), a range outside [0, max_landmarks] or with hi < lo: KBA_ERR_BAD_ARG;
 *   - the group form serves one request per track in one launch sequence (window = request): out[i] is bit for bit what the
 *     single call writes for req[i]; a request with hi == lo sits the call out (out[i] not written; a call in which every
 *     request sits out returns at once); a failing request returns its code, kba_last_error names its track, nothing is written.
 * Transfers (kba_track_transfer_bytes; over the W requests that do not sit out for kba_track_group_transfer_bytes, R the size of
 * one window's argument record, a constant of the library build; n_w = hi - lo, L_w the live keyframes of request w's track;
 * the slots are downloaded for the whole range):
 *         h2d = 4 * sum(L_w) + R * (W - 1),   d2h = sum(4 + 4 * n_w + (pos ? 24 * n_w : 0) + (weight ? 8 * n_w : 0)) */
typedef struct kba_reclaim_request {
    int32_t lo, hi;             /* slot range [lo, hi); hi == lo (group call): this track sits the call out                  */
} kba_reclaim_request;
typedef struct kba_reclaim_out {  /* caller-owned */
    int32_t n_free;
    int32_t reserved_;
    int32_t* free_slot;         /* [hi - lo]; the first n_free are written                                                   */
    double* pos;                /* [3 * (hi - lo)] or NULL                                                                   */
    double* weight;             /* [hi - lo] or NULL                                                                         */
} kba_reclaim_out;
int kba_track_reclaim_landmarks(kba_track* t, const kba_reclaim_request* req, kba_reclaim_out* out);
/* req[n_tracks], out[n_tracks] */
int kba_track_group_reclaim_landmarks(kba_track_group* g, const kba_reclaim_request* req, kba_reclaim_out* out);

/* ---- store writes for every track of a group: push, drop, landmark values and keyframe poses in one call each -----------------
 * The group forms of kba_track_push_keyframe, kba_track_drop_keyframe, kba_track_set_landmarks and kba_track_set_keyframe_poses,
 * one request per track (req[n_tracks]); each single call is the one-track form of the same host code and kernels.
 *   - Sitting out: a push or drop with kf_slot < 0, a landmark or pose write with n == 0.  A call in which every request sits out
 *     returns at once.
 *   - Validation: every other request gets the checks of its single call, with the same error codes, before anything is uploaded:
 *     a null array, a negative size, a slot or camera out of range, a push into a slot in use: KBA_ERR_BAD_ARG; a push whose
 *     measurements do not fit max_measurements next to the track's live (pushed, not dropped) keyframes' measurements:
 *     KBA_ERR_CAPACITY, decided from the host's mirror of the arena, so nothing is compacted.  If one request fails, the call returns
 *     its code, kba_last_error names the track index, and no store changes.
 *   - Results: each track's store afterwards equals, bit for bit, what the single calls in track order leave: arena contents at the
 *     same offsets, poses, planes, positions and weights.  A slot listed twice in one write is written in an unspecified order.
 *   - A push appends the keyframe's measurements to the track's arena.  A track whose arena has no room left at its end first
 *     compacts: its live keyframes, in slot order, are copied into the track's second arena (k_arena_compact), then the keyframe is
 *     appended there (k_store_append, which also writes the keyframe's arena offset, count, pose and plane).  plane4 NULL stores
 *     (0, 0, 1, 0); cam NULL stores camera 0 for every measurement.
 *   - Transfers: one upload (the rows of every request and a fixed record per track, plus a record per live keyframe of a track
 *     that compacts), one launch sequence and one synchronisation per call; more only when the rows exceed the staging, which holds
 *     min(max_measurements, 65536) pushed rows or max(win_landmarks, 64) landmark / pose rows per track, allocated for the set's
 *     capacities at the first call of each kind (a drop shares the push's).  A drop moves nothing.
 *     kba_track_group_transfer_bytes (kba_track_transfer_bytes for a single call) reports the call's upload and 0 bytes down.
 *     Each track's h2d_pushes_total counts its own rows: 20 bytes per pushed measurement plus 88 per keyframe, and 4 + 24 (pos)
 *     + 8 (weight) bytes per landmark row.
 *   - Each track that a request changed (every request that does not sit out) makes its ranking stale; the others keep theirs. */
typedef struct kba_push_request {  /* one keyframe into track i's store */
    int32_t kf_slot;            /* < 0: this track sits the call out                                                           */
    int32_t n_meas;             /* >= 0                                                                                        */
    const double* pose7;
    const double* plane4;       /* NULL: (0, 0, 1, 0)                                                                          */
    const int32_t* lm_slot;     /* [n_meas] */
    const int32_t* cam;         /* [n_meas] or NULL (every measurement camera 0)                                               */
    const float* u;             /* [n_meas] */
    const float* v;
    const float* d;
} kba_push_request;
int kba_track_group_push_keyframes(kba_track_group* g, const kba_push_request* req);
/* kf_slot[n_tracks]; < 0 sits out */
int kba_track_group_drop_keyframes(kba_track_group* g, const int32_t* kf_slot);
typedef struct kba_landmark_write {
    int32_t n;                  /* 0: this track sits the call out                                                             */
    int32_t reserved_;
    const int32_t* lm_slot;     /* [n] */
    const double* pos3;         /* [3 * n] or NULL */
    const double* weight;       /* [n] or NULL */
} kba_landmark_write;
int kba_track_group_set_landmarks(kba_track_group* g, const kba_landmark_write* req);
typedef struct kba_pose_write {
    int32_t n;                  /* 0: this track sits the call out                                                             */
    int32_t reserved_;
    const int32_t* kf_slot;     /* [n] */
    const double* pose7s;       /* [7 * n] */
    const double* plane4s;      /* [4 * n] or NULL (planes unchanged) */
} kba_pose_write;
int kba_track_group_set_keyframe_poses(kba_track_group* g, const kba_pose_write* req);

/* ---- snapshots of the stored window: save, load and clone a track, save every track of a group -------------------------------
 * A track's store is the only copy of its state (landmarks created on the device, poses and positions written back by solves).
 * A snapshot is that state as a little-endian byte buffer, to move a track to another handle or device, to resume after the
 * process ended, to fork a track, or to read the whole map (limo's dumpMap).  Format (version KBA_SNAPSHOT_VERSION):
 *   - a kba_snapshot_header at offset 0, then four sections, each at an 8-byte aligned offset, each a list of arrays in
 *     structure-of-arrays form, every array starting 8-byte aligned (4-byte arrays padded with zero bytes to a multiple of 8):
 *       cameras       cam_intr double [3 * n_cam], cam_pose double [7 * n_cam]
 *       keyframes     the live keyframes (pushed, not dropped) in ascending slot order: slot int32 [K], count int32 [K] (arena
 *                     entries), pose7 double [7 * K], plane4 double [4 * K]
 *       measurements  the live keyframes' arena runs concatenated in that order: lm int32 [M], cam int32 [M], u, v, d float [M]
 *       landmarks     pos double [3 * lm_cap], weight double [lm_cap], every slot
 *     K = n_keyframes, M = n_entries = sum(count), lm_cap = caps.max_landmarks; the sections follow each other in this order
 *     from offset sizeof(kba_snapshot_header) without gaps, so every offset and size follows from n_cam, K, M and lm_cap.
 *   - Canonical: stores with the same cameras, caps, live keyframes (slots, poses, planes, measurements) and landmark values give
 *     the same bytes, whatever their arena history (which arena is current, compactions, dropped keyframes' entries still in
 *     the arena).  Nothing else of the track is saved: not its rankings, generation, solvers, staging or cached options.  A slot
 *     never written holds 0 (kba_track_create zero-fills positions and weights).
 * kba_track_save writes the snapshot of t into buf (bytes = its capacity; kba_track_snapshot_size gives the size): a smaller
 *   buffer is KBA_ERR_CAPACITY and nothing is written.  One upload of the keyframe lists, one launch sequence, one download,
 *   one synchronisation.  The store does not change: a ranking made before a save can be solved after it.
 * kba_track_load creates a track on h (any device) whose store gives the same snapshot back, byte for byte.  caps NULL takes the
 *   saved caps; other caps get kba_track_create's checks and must hold the content: max_keyframes above every live slot,
 *   max_landmarks >= lm_cap, max_measurements >= n_entries, else KBA_ERR_CAPACITY (larger window caps grow a track).  Slots
 *   beyond the saved lm_cap hold 0.  The buffer comes from outside the program, so before anything is allocated every
 *   structural field is checked: magic, format version, reserved_ 0, counts, every offset and size against the counts and
 *   bytes, slots strictly ascending in [0, caps.max_keyframes), counts >= 0 summing to n_entries, every entry's landmark slot in
 *   [0, lm_cap) and camera in [0, n_cam); a failure is KBA_ERR_BAD_ARG, and kba_last_error names the field.  Floating-point
 *   values are taken as they are.  The loaded arena is compact from offset 0, the track starts without a ranking.  One
 *   upload, one launch sequence, one synchronisation.
 * kba_track_clone gives the store kba_track_load(h, save(src), caps) gives.  On src's device the copy goes from store to store
 *   without a host round trip; on another device it is a save and a load.  The copy reads src after src's earlier calls on
 *   its handle's stream (an event orders h's stream after it).
 * kba_track_group_save saves every track whose bufs[i] is not NULL (bytes[i] its capacity); a NULL buffer sits the call out.
 *   Buffer i gets exactly what kba_track_save writes for track i.  Every request is checked first: a failure returns its code,
 *   kba_last_error names the track, and no buffer is written.  One launch sequence, one download and one synchronisation for
 *   the whole group.  To load a group, load each track and call kba_track_group_create.
 * Staging: the first save of a track or group allocates a device image and a pinned host copy of it for the snapshots of its
 * tracks at their capacities (every keyframe slot live, a full arena), a loaded or cloned track its own at creation.
 * kba_track_transfer_bytes / kba_track_group_transfer_bytes then report the last save's upload and download (d2h = the
 * snapshots' bytes), a load's upload. */
#define KBA_SNAPSHOT_MAGIC 0x504E534Bu   /* the bytes "KSNP" */
#define KBA_SNAPSHOT_VERSION 1
typedef struct kba_snapshot_header {
    uint32_t magic;             /* KBA_SNAPSHOT_MAGIC                                                                          */
    uint32_t format_version;    /* KBA_SNAPSHOT_VERSION                                                                        */
    int32_t writer_version;     /* kba_version() of the library that wrote it                                                  */
    int32_t n_cam;
    kba_track_caps caps;        /* the track's                                                                                 */
    int32_t n_keyframes;        /* live keyframes                                                                              */
    int32_t n_entries;          /* their arena entries                                                                         */
    int32_t lm_cap;             /* landmark slots saved: caps.max_landmarks                                                    */
    int32_t reserved_;          /* 0                                                                                           */
    int64_t cam_offset, cam_bytes;       /* sections: byte offset from the start of the buffer, and size                       */
    int64_t kf_offset, kf_bytes;
    int64_t meas_offset, meas_bytes;
    int64_t lm_offset, lm_bytes;         /* lm_offset + lm_bytes: the snapshot's size                                          */
} kba_snapshot_header;
int kba_track_snapshot_size(const kba_track* t, int64_t* bytes);
int kba_track_save(kba_track* t, void* buf, int64_t bytes);
int kba_track_load(kba_handle* h, const void* buf, int64_t bytes, const kba_track_caps* caps, kba_track** out);
int kba_track_clone(kba_track* src, kba_handle* h, const kba_track_caps* caps, kba_track** out);
/* bytes[n_tracks]: each track's kba_track_snapshot_size */
int kba_track_group_snapshot_sizes(kba_track_group* g, int64_t* bytes);
/* bufs[n_tracks] (NULL: the track sits out), bytes[n_tracks] */
int kba_track_group_save(kba_track_group* g, void* const* bufs, const int64_t* bytes);

/* ---- ranked landmark selection on the stored window, and the solve of that ranking (SURVEY row A17) ------------------------
 * kba_track_select_landmarks leaves the ranking of its quantities to the host; kba_track_rank_landmarks ranks them on the
 * device as LandmarkSelector::select (facade/landmark_selection.cpp) does for limo's chain -- cheirality, voxel, AddDepth with
 * limo's sorter -- and keeps the ranked selection on the track, where kba_track_solve_ranked reads it.  A request:
 *   - kf_slot [n_kf], lm_slot [n_cand], params: exactly as for kba_track_select_landmarks (n_cand <= 57344);
 *   - elig [n_cand] or NULL (none): the AddDepth comparator's verdict per candidate (limo: is_ground_plane);
 *   - max_near, max_middle, max_far: the voxel scheme's caps (max_num_landmarks_{near,middle,far});
 *   - depth [n_depth] (n_depth <= 1024): the AddDepth scheme's (FrameIndex, NumberLandmarks) entries; an entry with
 *     ind >= n_kf is skipped, as the scheme skips it;
 *   - draw, draw_ctx: the random source of the middle bin's shuffle (below).
 * The ranking, bit for bit the facade's from the same store state, ties included:
 *   - near: the near representatives with a flow, in near order, std::partial_sort_copy by flow descending, capped;
 *   - middle: the middle representatives in candidate order, libstdc++'s random_shuffle (for i = 1 .. n - 1: j = draw % (i + 1),
 *     swap), the first max_middle kept;
 *   - far: the far candidates in candidate order, std::partial_sort_copy by seen descending, capped;
 *   - AddDepth, per entry (ind, wanted): the cheirality survivors with elig set that keyframe kf_slot[ind] measures, in its arena
 *     order, with kba_track_depth_costs' cost; std::partial_sort ascending, the first min(wanted, n) kept.
 * Each partial sort replays libstdc++'s heap (make_heap, __adjust_heap), so the tied elements it keeps are the host's.
 * The selection is the union of the bins and the AddDepth picks in ascending candidate order.  Outputs:
 *   - n_sel, and cand [n_sel] (candidate indices, ascending) with category [n_sel]: 0 near, 1 middle, 2 far, 3 AddDepth only;
 *     the caller allocates both for n_cand entries;
 *   - n_ground: the selected candidates with elig set, which kba_track_solve_ranked can attach on the device;
 *   - n_draws: the draws the shuffle used, max(n_middle - 1, 0).
 * Draws: the shuffle needs exactly max(n_middle - 1, 0) of them, which is known on the device only.  The call therefore
 * synchronises once in its middle: after the chain's quantities it downloads 4 bytes per window (the middle bin's size), calls
 * draw(draw_ctx, n, out) once for a request that needs n > 0 draws (requests in order, before any ranking kernel runs) and
 * uploads the draws.  A draw function returning nonzero, or a NULL one where draws are needed, fails the call with
 * KBA_ERR_BAD_ARG after that synchronisation: no output is written and the track keeps no ranking.  A caller whose draw function
 * fills out[] with std::rand() gets the facade's selection and leaves std::rand's sequence where the facade's select() leaves it.
 * The track keeps the ranked slots, the ground candidates and the keyframe list until its next ranking.  The ranking goes stale
 * at any call that changes the store: push, drop, set_landmarks, set_keyframe_pose(s), create_landmarks, reclaim_landmarks and
 * every solve (alone or in a group, ranked or not).
 * Transfers (kba_track_transfer_bytes; over the W requests that do not sit out for kba_track_group_transfer_bytes, R the size of
 * one window's argument records, a constant of the library build; D_w = max(n_middle_w - 1, 0) the draws of request w;
 * B_w = min(n_cand, min(max_near, n_cand) + min(max_middle, n_middle) + min(max_far, n_cand) + sum of min(wanted, n_cand)),
 * the bound of its selection; elig bytes travel also when elig is NULL):
 *         h2d = sum(4 * (n_kf + n_cand) + n_cand + 8 * n_depth) + R * (W - 1) + 8 * W + 4 * sum(D_w)
 *         d2h = 4 * W + sum(8 + 5 * B_w)
 * Two uploads (the lists; then the output offsets and the draws), one launch sequence in two parts, two downloads (the middle
 * bin's sizes; then the outputs), two synchronisations.  The first call of a track by either entry point allocates its ranking
 * buffers (and its selection scratch, if no selection allocated it), the first single call its staging; later calls allocate
 * nothing.
 * Errors, before anything is uploaded or written: those of kba_track_select_landmarks, a null out.cand / out.category with
 * n_cand > 0, a negative cap, n_depth < 0, depth NULL with n_depth > 0, an entry with ind < 0 or wanted < 0: KBA_ERR_BAD_ARG;
 * n_cand > 57344, n_depth > 1024, or an entry with min(wanted, arena entries of kf_slot[ind]) > 57344: KBA_ERR_CAPACITY.
 * kba_track_group_rank_landmarks ranks one request per track of a group in one launch sequence (window = request): out[i] and
 * track i's ranking are bit for bit what kba_track_rank_landmarks(tracks[i], &req[i], &out[i]) gives, draws included (each
 * request's draw function is called with its own count); a request with n_kf == 0 sits the call out (out[i] not written, its
 * ranking kept); every other request is checked before anything is uploaded; a failing one returns its code and
 * kba_last_error names its track. */
typedef struct kba_depth_entry {
    int32_t ind;                /* FrameIndex: kf_slot[ind] (0 the oldest listed keyframe)                                    */
    int32_t wanted;             /* NumberLandmarks                                                                            */
} kba_depth_entry;
typedef struct kba_rank_request {
    int32_t n_kf;               /* 0 (group call): this track sits the call out                                              */
    int32_t n_cand;
    const int32_t* kf_slot;     /* [n_kf]   as for kba_track_select_landmarks                                               */
    const int32_t* lm_slot;     /* [n_cand] as for kba_track_select_landmarks                                               */
    const uint8_t* elig;        /* [n_cand] or NULL (no candidate is eligible)                                               */
    const kba_select_params* params;
    int32_t max_near, max_middle, max_far;
    int32_t n_depth;
    const kba_depth_entry* depth;  /* [n_depth] */
    int32_t (*draw)(void* ctx, int32_t n, int32_t* out);  /* fills out[0 .. n); 0 = success */
    void* draw_ctx;
} kba_rank_request;
typedef struct kba_rank_out {   /* caller-owned */
    int32_t n_sel;
    int32_t n_ground;
    int32_t n_draws;
    int32_t reserved_;
    int32_t* cand;              /* [n_cand]; the first n_sel are written                                                     */
    int8_t* category;           /* [n_cand]; the first n_sel are written                                                     */
} kba_rank_out;
int kba_track_rank_landmarks(kba_track* t, const kba_rank_request* req, kba_rank_out* out);
/* req[n_tracks], out[n_tracks] */
int kba_track_group_rank_landmarks(kba_track_group* g, const kba_rank_request* req, kba_rank_out* out);
/* kba_track_solve on the track's last ranking: lm_slot is the ranked selection (n_lm = n_sel), in ranked order, and the results'
 * landmark arrays follow it.  sel as for kba_track_solve, except that gp_lm, gp_kf and gp_weight all NULL with n_gp > 0 attach
 * the ranking's ground candidates on the device (none: no ground-plane residuals, as kba_track_solve with n_gp = 0); host lists
 * and caller candidates index the ranked selection.  Nothing about the selection is uploaded.  Errors, before anything is
 * uploaded: no ranking, a stale one, or kf_slot different from the ranking's keyframe list: KBA_ERR_BAD_ARG; then those of
 * kba_track_solve.  The results equal kba_track_solve's on the same lists bit for bit, and the solve makes the ranking stale. */
int kba_track_solve_ranked(kba_track* t, int32_t n_kf, const int32_t* kf_slot, const uint8_t* kf_fixed, const kba_window* sel,
                           const kba_options* opt, kba_result* res);
typedef struct kba_ranked_request {
    int32_t n_kf;               /* 0: this track sits this solve out (as for kba_track_group_solve)                           */
    int32_t reserved_;
    const int32_t* kf_slot;
    const uint8_t* kf_fixed;
    const kba_window* sel;
} kba_ranked_request;
/* kba_track_group_solve on every track's last ranking; each request is checked as kba_track_solve_ranked checks it.
 * req[n_tracks], res[n_tracks] */
int kba_track_group_solve_ranked(kba_track_group* g, const kba_ranked_request* req, const kba_options* opt, kba_result* res);
/* kba_track_group_solve_ranked with opts[n_tracks], one per track, as kba_track_group_solve_opts takes them */
int kba_track_group_solve_ranked_opts(kba_track_group* g, const kba_ranked_request* req, const kba_options* opts, kba_result* res);

/* ---- limo's solve block as one call: deactivateKeyframes, updateLabels and the ranked solve ---------------------------------
 * What limo runs once it decides to solve (mono_lidar.cpp:249-255, mono_standalone.cpp:171-183):
 *     deactivateKeyframes(min_connecting, min_window, max_window); updateLabels(tracklets, shrubbery_weight); solve();
 * on the stored window, with its results equal, bit for bit, to those of the chain of store calls a caller runs today:
 *   1. kba_track_deactivate_keyframes on kf_slot / lm_slot (the request's first six fields mean what kba_deactivate_request's do);
 *   2. the post-deactivation lists: the keyframes with kf_active = 1 and the landmarks with lm_active = 1, order kept; the oldest
 *      kept keyframe gets FixationStatus::Pose (bundle_adjuster_keyframes.cpp:980; Scale has no effect on the solve, cpp:736),
 *      every other one is free;
 *   3. updateLabels (cpp:388-431, facade/bundle_adjuster_keyframes.cpp) over the tracklets, each (landmark slot, label,
 *      is_outlier), slot -1 for an id without one, and the class table (label, classes) of labels_ (an unlisted label has none):
 *        - the new outlier set: the caller's outliers (outlier_slot) that are still active, plus every tracklet with is_outlier
 *          set or a label of class KBA_LABEL_OUTLIER;
 *        - a tracklet whose landmark is still active: a shrubbery label writes shrubbery_weight into the store's weight of its
 *          slot; its ground flag becomes (label of class KBA_LABEL_GROUND), the last tracklet of a slot deciding.  The other
 *          listed landmarks keep the flag the caller gives in lm_ground (NULL: none is ground);
 *   4. kba_track_rank_landmarks on the post-deactivation keyframes and the candidates -- the still-active landmarks that are not
 *      in the new outlier set, in lm_slot order -- with elig = the candidates' ground flags (limo's AddDepth comparator,
 *      is_ground_plane), and params, the caps, the AddDepth entries and the draw function as kba_rank_request takes them;
 *   5. kba_track_solve_ranked on the post-deactivation keyframes and their fixation with `sel` (its scalars and ground mode, as
 *      that call takes them; scale_kf0 / scale_kf1 index the post-deactivation keyframes; n_kf / n_lm are not read).
 * Outputs (caller-owned; cand / category and the result's landmark arrays sized for n_lm, its keyframe arrays for n_kf):
 *   - kf_active, kf_common [n_kf], lm_active [n_lm]: as the deactivation writes them;
 *   - lm_outlier [n_lm], trk_outlier [n_trk]: the new outlier set over the listed landmarks and over the tracklets (a tracklet is
 *     flagged iff its landmark is in the set); lm_ground [n_lm]: the listed landmarks' ground flags after the labels;
 *   - rank: n_sel, cand (indices into the candidates of step 4), category, n_ground, n_draws, as the ranking writes them;
 *   - res: the ranked solve's kba_result (keyframe arrays in post-deactivation order, landmark arrays in ranked order).
 * With these a caller keeps its bookkeeping (active_keyframe_ids_, the outlier set, selected_landmark_ids_) as after the chain.
 * On the device: one upload (the lists, the tracklets' classes, the AddDepth entries and every window's argument records) and ONE
 * launch sequence run the deactivation (k_up_*), updateLabels and the post-deactivation lists (k_kfs_labels, which also writes
 * the ranking records' sizes) and the ranking's first part (k_sel_*, k_rk_prep, k_rk_depth), then one download brings back the
 * deactivation's and the labels' outputs, the kept keyframes and the middle bins' sizes.  The host then checks the ranking and
 * the solve on the kept keyframes, calls the draw functions, uploads the draws and runs the ranking's second part (k_rk_heap,
 * k_rk_union; one download), and launches k_kfs_weights (the shrubbery weights) ahead of the ranked solve.
 * Checks: every check that needs only the request runs before anything is uploaded: those of the deactivation, the tracklets'
 * slots in [-1, max_landmarks), the outlier slots in range, the ranking's parameters, caps and AddDepth entries, n_lm <= 57344
 * (the ranking's candidate bound: the candidates are a subset of the listed landmarks), the options.  The checks on the kept
 * keyframes (none kept: KBA_ERR_BAD_ARG; those of kba_track_solve; an AddDepth heap over 57344) and a failing or missing draw
 * function refuse the call after the first download, the ranked solve's checks after the second, all with the codes and
 * messages of the underlying calls and before the store is written: a refused call writes no output and leaves every store's
 * content (its snapshot) as it was.  Its rankings do not survive it: a call refused before the ranking's second part leaves the
 * tracks it ran for without a ranking (kba_track_solve_ranked refuses to solve), one refused by the ranked solve's checks
 * leaves them this call's ranking.  The shrubbery weights go into the store after the ranking (which does not read weights, so
 * it stays valid) and before the solve.
 * Transfers (kba_track_transfer_bytes / kba_track_group_transfer_bytes), over the W requests that do not sit out, R the size of
 * one window's argument records (a constant of the library build), D_w the draws and B_w the selection bound of request w as
 * kba_track_rank_landmarks states them, each request's arrays padded to 8-byte boundaries:
 *         h2d = R * W + sum(8 n_depth + 4 (n_kf + n_lm + n_outlier + n_trk) + n_lm + n_trk) + 8 W + 4 sum(D_w) + the solve's
 *         d2h = 4 W + sum(8 + 9 n_kf + 3 n_lm + n_trk) + 8 W + 5 sum(B_w) + the solve's
 * where the solve's are kba_track_solve_ranked's (kba_track_group_solve_ranked's).  Allocations: each track's label scratch
 * (8 bytes per landmark slot) and the scratch of the selection, ranking and upkeep calls at their first use by any entry point;
 * the call's staging grows to its largest call: a call no larger than an earlier one allocates nothing on the device.
 * The group forms serve one request per track (req[n_tracks], out[n_tracks], res[n_tracks]), each step for all tracks at once as
 * the step's group call does it: a request with n_kf == 0 sits the call out (its outputs are not written, res[i] is idle as for
 * kba_track_group_solve); a failing request returns its code and kba_last_error names its track; _opts takes one kba_options per
 * track.  A single call is the group call's one-track case. */
#define KBA_LABEL_OUTLIER 1
#define KBA_LABEL_SHRUBBERY 2
#define KBA_LABEL_GROUND 4
typedef struct kba_label_class {
    int32_t label;
    int32_t classes;            /* KBA_LABEL_* bits                                                                           */
} kba_label_class;
typedef struct kba_tracklet {
    int32_t lm_slot;            /* -1: the landmark id has no slot                                                             */
    int32_t label;
    uint8_t is_outlier;
    uint8_t reserved_[3];
} kba_tracklet;
typedef struct kba_kfsolve_request {
    int32_t n_kf;               /* 0 (group call): this track sits the call out                                               */
    int32_t n_lm;
    int32_t min_connecting, min_window, max_window;
    int32_t n_trk;
    const int32_t* kf_slot;     /* [n_kf] the active keyframes in ascending id order; the last one is the newest             */
    const int32_t* lm_slot;     /* [n_lm] the active landmarks in ascending id order                                          */
    const uint8_t* lm_ground;   /* [n_lm] is_ground_plane of the listed landmarks before the call, or NULL (none)             */
    const kba_tracklet* trk;    /* [n_trk] the current frame's tracklets                                                      */
    const kba_label_class* classes;  /* [n_class] */
    int32_t n_class;
    int32_t n_outlier;
    const int32_t* outlier_slot;     /* [n_outlier] the caller's current outlier set (landmark_selector_->getOutliers())       */
    double shrubbery_weight;
    const kba_select_params* params; /* the ranking, as kba_rank_request                                                       */
    int32_t max_near, max_middle, max_far;
    int32_t n_depth;
    const kba_depth_entry* depth;
    int32_t (*draw)(void* ctx, int32_t n, int32_t* out);
    void* draw_ctx;
    const kba_window* sel;      /* the solve's scalars and ground mode, as kba_track_solve_ranked takes them                    */
} kba_kfsolve_request;
typedef struct kba_kfsolve_out {  /* caller-owned */
    uint8_t* kf_active;         /* [n_kf] */
    int32_t* kf_common;         /* [n_kf] */
    uint8_t* lm_active;         /* [n_lm] */
    uint8_t* lm_outlier;        /* [n_lm] */
    uint8_t* lm_ground;         /* [n_lm] */
    uint8_t* trk_outlier;       /* [n_trk] */
    kba_rank_out rank;          /* cand, category: [n_lm] */
} kba_kfsolve_out;
int kba_track_keyframe_solve(kba_track* t, const kba_kfsolve_request* req, const kba_options* opt, kba_kfsolve_out* out,
                             kba_result* res);
/* req[n_tracks], out[n_tracks], res[n_tracks] */
int kba_track_group_keyframe_solve(kba_track_group* g, const kba_kfsolve_request* req, const kba_options* opt, kba_kfsolve_out* out,
                                   kba_result* res);
/* opts[n_tracks]: track i's solve runs with opts[i]; a track that sits out does not read its entry */
int kba_track_group_keyframe_solve_opts(kba_track_group* g, const kba_kfsolve_request* req, const kba_options* opts,
                                        kba_kfsolve_out* out, kba_result* res);

/* ---- adjustPoseOnly against the persistent store: one frame's pose per call, or one frame of each track of a group -------
 * What limo calls on every frame (bundle_adjuster_keyframes.cpp:820-888): one free pose against constant landmarks, the optional
 * SpeedRegularizationVector2 prior and the trimming rounds.  The result is that of kba_solve_window on the equivalent window: one
 * keyframe (kf_fixed 0) at pose7, the frame's measurements as its observations in the caller's landmark order, landmark positions
 * and weights read from the store by slot, landmarks_fixed = 1, no ground plane, no scale or plane regulariser.
 *   - The frame is solved by ONE kernel (one CTA, the whole trimmed solve): a call makes one upload, one launch, one download
 *     and one synchronisation, and allocates nothing after the first call of its track (group), which allocates the buffers for
 *     the track's (group's) win_landmarks / win_observations.
 *   - Validation, before anything is uploaded: null pointers, negative sizes, a slot or camera out of range, a slot that
 *     reappears after its run has ended: KBA_ERR_BAD_ARG; more than win_observations measurements or more than win_landmarks
 *     runs: KBA_ERR_CAPACITY; kba_options.precision != 0: KBA_ERR_BAD_ARG (FP64 only).  As for kba_solve_window: a speed prior
 *     with speed_dt <= 0 is KBA_ERR_BAD_ARG, more than 6 trimming rounds (num_trim_rounds, or num_rounds_option when it is -1)
 *     KBA_ERR_CAPACITY.  A group checks every frame first and
 *     returns the failing frame's code, kba_last_error names its track index.
 *   - Results: res->kf_pose [7], res->lm_rejected [number of runs, in run order], the summaries, the iteration log and
 *     time_sec (the kernel's device time).  lm_pos and kf_plane are not written: the store is never modified, the frame is not
 *     a keyframe.  kba_track_transfer_bytes (kba_track_group_transfer_bytes) then report this call's upload and download.
 *   - Trimming: opt->num_trim_rounds as given; -1 = the reference rule on the frame's landmark count against
 *     min_landmarks_for_trimming (30 for adjustPoseOnly, cpp:865).  solver_time_sec is applied per inner solve on the device.
 *   - n_meas == 0: the frame sits the call out (res status KBA_OK, num_solves 0, nothing written). */
typedef struct kba_track_frame {
    int32_t n_meas;             /* 0: this frame sits the call out (res status KBA_OK, num_solves 0, nothing written) */
    int32_t reserved_;
    const double* pose7;        /* initial pose of the frame, 7-vector convention */
    const int32_t* lm_slot;     /* [n_meas] store slots; one contiguous run per landmark, runs in the caller's landmark order
                                   (ascending id, as selected_landmark_ids_ ∩ measurements_), cameras ascending inside a run */
    const int32_t* cam;         /* [n_meas] or NULL (all camera 0) */
    const float* u, *v, *d;     /* [n_meas] FeaturePoint; depth residual iff d > 0 */
    double speed_weight;        /* SpeedRegularizationVector2 exactly as kba_window's speed_* fields; <= 0: none */
    double speed_dt;
    double speed_v_before[3];
    double speed_T_origin_before[7];
} kba_track_frame;
int kba_track_adjust_pose(kba_track* t, const kba_track_frame* f, const kba_options* opt, kba_result* res);
/* f[n_tracks], res[n_tracks]: frame i is tracked against track i's store, all frames in one launch */
int kba_track_group_adjust_pose(kba_track_group* g, const kba_track_frame* f, const kba_options* opt, kba_result* res);
/* kba_track_group_adjust_pose with opts[n_tracks]: frame i is tracked with opts[i], exactly as kba_track_adjust_pose with opts[i].
 * The entries of the frames that are tracked are checked before anything is uploaded (kba_last_error names the track index); a
 * frame with n_meas == 0 does not read its entry. */
int kba_track_group_adjust_pose_opts(kba_track_group* g, const kba_track_frame* f, const kba_options* opts, kba_result* res);

/* ---- limo's frame step as one call: adjustPoseOnly, keyframe selection and the push with its new landmarks ----------------------
 * What limo runs on every camera frame (mono_lidar.cpp:200-232, mono_standalone.cpp:134-168):
 *     adjustPoseOnly(*cur_frame); kfs = keyframe_selector_.select({cur_frame}, active keyframes); if (!kfs.empty()) push(*kf);
 * on the stored window, with its results equal, bit for bit, to those of the chain of store calls a caller runs today:
 *   1. kba_track_adjust_pose on the measurements of the runs with run_sel set (landmark_selector_->getLastSelection(),
 *      bundle_adjuster_keyframes.cpp:828), in request order, with pose7 and the speed_* fields (those of kba_track_frame).  With
 *      adjust == 0 (mono_lidar's external prior, mono_lidar.cpp:200) or no run selected, no solve runs and the frame's pose is
 *      pose7; res is then idle (status KBA_OK, num_solves 0, nothing written), as kba_track_adjust_pose leaves a frame without
 *      measurements;
 *   2. kba_track_frame_flow over all measurements against kf_last = kf_slot[n_kf - 1] with min_median_flow;
 *   3. the verdict of KeyframeSelector::select({frame}, active keyframes) with limo's three schemes, composed on the host (one
 *      frame, a non-empty buffer: flow and (pose or time)):
 *        - flow: n_meas > 0 and mean_flow_sq > min_median_flow^2 (the flow call's usable);
 *        - pose: angle > critical_quaternion_diff, angle = calcQuaternionDiff(frame pose, kf_last's stored pose) in the facade's
 *          operation order (limo_b200/keyframe_selector.py; it goes through atan2, which stays on the host);
 *        - time: (stamp - stamp_last) mod 2^64 > time_difference_ns;
 *   4. if selected, kba_track_push_keyframe(kf_new, frame pose, plane4, the frame's measurements) -- compacting the arena first
 *      when its end has no room, exactly as the push does;
 *   5. if selected, kba_track_create_landmarks over kf_slot followed by kf_new (kf_new last) for the landmarks new_slot names.
 * The request's measurements follow the run contract of kba_track_frame and kba_flow_request: one run per landmark, runs in
 * ascending landmark id, cameras ascending inside a run.  Every run's landmark has a slot: a landmark the frame measures for the
 * first time carries the slot the caller assigns it, and new_slot lists those to create.  A frame that is not selected leaves
 * the store untouched (its ranking stays valid); a selected one writes it, and its ranking is stale.
 * Outputs: the flow call's (n_matched, flow_sum, mean_flow_sq, match), angle, the three scheme verdicts and selected, always;
 * pos and flags (kba_create_out's) only when the frame is selected.  res is the adjustment's kba_result as kba_track_adjust_pose
 * writes it (kf_pose [7], lm_rejected [selected runs, in run order]).
 * On the device: ONE upload (the frame's five columns, 20 bytes per measurement, the run flags, the keyframe and new-landmark
 * lists and every window's argument records) and one launch sequence run k_fs_gather (the selected runs gathered into the
 * pose-only kernel's input by a block-wide ballot scan, kf_last's stored pose copied out), k_adjust_pose and the flow kernels,
 * which read the staged columns in place; ONE download brings back the adjustment's results, the flow's and kf_last's pose.
 * The host composes the verdicts.  Only if some frame is selected: one upload of the push's and the creation's argument
 * records, k_arena_compact (tracks that compact), k_store_append -- which copies the staged columns and takes the adjusted pose
 * from the adjustment's output in device memory -- and the creation's kernels, then one download of the creations' outputs.
 * Two synchronisations per call, one when no frame is selected.
 * Checks: every check runs before anything is uploaded: null pointers, n_kf < 1 (single call), negative sizes; the keyframe
 * list as the create call checks it (pushed, listed once, n_kf + 1 keyframe slots); kf_new out of range or in use
 * (KBA_ERR_BAD_ARG); the run contract, landmark slots and cameras in range (KBA_ERR_BAD_ARG); new_slot in range and listed once
 * (KBA_ERR_BAD_ARG); n_meas > win_observations, more selected runs than win_landmarks, and measurements that would not fit
 * max_measurements next to the live keyframes' were the frame selected (from the host's mirror of the arena): KBA_ERR_CAPACITY;
 * with adjust set, the options as kba_track_adjust_pose checks them (precision != 0: KBA_ERR_BAD_ARG) and a speed prior with
 * speed_dt <= 0.  A refused call writes no output and changes no store; nothing refuses after the first download.
 * Transfers (kba_track_transfer_bytes / kba_track_group_transfer_bytes), over the W requests that do not sit out, A of them
 * adjusted (adjust set and a run selected), S selected, C of those compacting with P keyframe slots holding measurements in
 * all, R_1, R_a, R_2, R_c and R_p sizes of argument records (constants of the library build), L the iteration records the
 * results take (min(iterations_capacity, 160) of the adjusted frames' largest, 0 without iterations arrays):
 *         h2d = R_1 W + R_a A + sum(20 n_meas + 4 (n_kf + 1 + n_new) + n_runs) + (S ? R_2 S + R_c C + R_p P : 0)
 *         d2h = R_f A + R_i A L + sum over adjusted frames of their selected runs + sum(4 n_meas + 80) + 25 sum over selected of n_new
 * with R_f, R_i the sizes of a frame's result and iteration records; each term of h2d and of d2h is one region of the staging.
 * Allocations: the call uses each track's motion (pose-only), upkeep, flow and creation scratch, allocated at their first use
 * by any entry point; its staging grows to its largest call: a call no larger than an earlier one allocates nothing.
 * The group forms serve one request per track (req[n_tracks], out[n_tracks], res[n_tracks]), each phase one launch sequence
 * over every track that takes part: a request with n_kf == 0 sits the call out (out[i] not written, res[i] idle); a failing
 * request returns its code and kba_last_error names its track; _opts takes one kba_options per track (a track that sits out
 * or is not adjusted does not read its entry).  If no track is selected the call ends after the first download.  A single
 * call is the group call's one-track case. */
typedef struct kba_frame_step_request {
    int32_t n_kf;               /* 0 (group call): this track sits the call out                                              */
    int32_t n_meas;
    const int32_t* kf_slot;     /* [n_kf] the active keyframes in ascending id order; the last one is the newest (kf_last)   */
    const int32_t* lm_slot;     /* [n_meas] every measurement of the frame, runs as kba_track_frame's                         */
    const int32_t* cam;         /* [n_meas] or NULL (all camera 0)                                                            */
    const float* u, *v, *d;     /* [n_meas] FeaturePoint; d < 0: no depth                                                     */
    const uint8_t* run_sel;     /* [runs of lm_slot] 1: the run's landmark is in the last selection (adjustPoseOnly's)        */
    int32_t n_new;
    int32_t kf_new;             /* the slot the frame is pushed into if selected: free when the call starts                  */
    const int32_t* new_slot;    /* [n_new] the landmarks to create if selected (kba_create_request's lm_slot)                 */
    const double* pose7;        /* the frame's initial pose (the prior)                                                        */
    const double* plane4;       /* the pushed keyframe's plane; NULL: (0, 0, 1, 0)                                             */
    double speed_weight;        /* the speed prior, as kba_track_frame's speed_* fields; <= 0: none                           */
    double speed_dt;
    double speed_v_before[3];
    double speed_T_origin_before[7];
    double min_median_flow;     /* KeyframeRejectionSchemeFlow                                                                */
    double critical_quaternion_diff;  /* KeyframeSelectionSchemePose, radians                                                 */
    uint64_t time_difference_ns;      /* KeyframeSparsificationSchemeTime::time_difference_nano_sec_                          */
    uint64_t stamp;             /* the frame's time stamp, ns                                                                 */
    uint64_t stamp_last;        /* kf_last's time stamp, ns                                                                   */
    uint8_t adjust;             /* 0: the pose is taken as given, no solve runs                                               */
    uint8_t reserved_[7];
} kba_frame_step_request;
typedef struct kba_frame_step_out {  /* caller-owned */
    int32_t n_matched;          /* the flow call's outputs                                                                    */
    uint8_t usable_flow, usable_pose, usable_time, selected;  /* the three schemes' verdicts and the selector's                */
    double flow_sum;
    double mean_flow_sq;
    double angle;               /* calcQuaternionDiff(frame pose, kf_last's stored pose)                                      */
    int32_t* match;             /* [n_meas] or NULL                                                                           */
    double* pos;                /* [3 * n_new] written only when selected; NaN where not created                              */
    uint8_t* flags;             /* [n_new] written only when selected: bit 0 created, bit 1 has depth                         */
} kba_frame_step_out;
int kba_track_frame_step(kba_track* t, const kba_frame_step_request* req, const kba_options* opt, kba_frame_step_out* out,
                         kba_result* res);
/* req[n_tracks], out[n_tracks], res[n_tracks] */
int kba_track_group_frame_step(kba_track_group* g, const kba_frame_step_request* req, const kba_options* opt,
                               kba_frame_step_out* out, kba_result* res);
/* opts[n_tracks]: track i's adjustment runs with opts[i] */
int kba_track_group_frame_step_opts(kba_track_group* g, const kba_frame_step_request* req, const kba_options* opts,
                                    kba_frame_step_out* out, kba_result* res);

/* ---- landmark initialisation of push() for a whole window (SURVEY 8(f) row 2) ------------------------------------------
 * Replaces, for all landmarks of `w` at once, what BundleAdjusterKeyframes::push() does per new landmark on the host:
 * the first observation with a lidar depth (d >= 0) is back-projected (bundle_adjuster_keyframes.cpp:332-355); without
 * one, the point closest to all viewing rays is taken when there are at least two (cpp:125-159,358-382,
 * internal/triangulator.hpp:51-75); then the cheirality test of the landmark selector
 * (landmark_selection_scheme_cheirality.cpp:22-60).  Batch semantics: "first observation" is CSR order (keyframe, then
 * camera), where the incremental reference looks at the keyframe being pushed.  w->lm_pos is not read.
 * flags_out[j]: bit 0 = a position was computed, bit 1 = it lies in front of every observing camera. */
int kba_init_landmarks(kba_handle* h, const kba_window* w, double* lm_pos_out, uint8_t* flags_out, float* device_ms);

/* ---- lidar depth extraction (BASELINE config 4) --------------------------------------------------------------------
 * Replaces the un-vendored mono_lidar_depth::DepthEstimator call the limo front end makes per frame (install_repos.sh:9;
 * in-tree only its parameter file demo_keyframe_bundle_adjustment_meta/res/mono_lidar_fusion_parameters.yaml, whose
 * keys the fields below carry, defaults = the YAML values).  Per feature: lidar points projected into the pixel
 * rectangle around it -> depth-histogram segmentation (nearest local maximum) -> plane through the largest triangle
 * -> intersection with the view ray; -1 when any gate fails.  No reference code or tests exist for it (SURVEY 8c):
 * the CPU restatement in oracle/ follows this specification, parity is "unpinned". */
typedef struct kba_lidar_options {
    int32_t image_width, image_height;  /* 1242 x 375 */
    double rect_width, rect_height;     /* pixelarea_search_witdh 6, pixelarea_search_height 9 (yaml:11-13) */
    double rect_offset_x, rect_offset_y;/* yaml:15-18 */
    double hist_bin_width;              /* histogram_segmentation_bin_witdh 0.3 m (yaml:58-61) */
    int32_t hist_min_count;             /* histogram_segmentation_min_pointcount 1 (yaml:63) */
    int32_t min_points;                 /* points needed for a plane: 3 */
    double depth_min, depth_max;        /* treshold_depth_min/max 0 / 100 (yaml:97-104) */
    double local_rel_tolerance;         /* treshold_depth_local_value 0.5, relative (yaml:106-114); < 0 disables */
    double triangle_crossnorm_min;      /* triangleplanar_crossnorm_treshold 0.1 (yaml:172-175) */
    double viewray_plane_min;           /* viewray_plane_orthoganality_treshold 0.1 (yaml:177-178) */
} kba_lidar_options;
void kba_lidar_default_options(kba_lidar_options* opt);
/* cloud: n_points x point_stride floats, xyz first (KITTI .bin layout x,y,z,intensity: apps/main_program/utility.h:28-39);
 * T_cam_lidar: 7-vector camera <- lidar; intr: f, cx, cy; features: n_features x 2 floats (u, v); depth_out: n_features floats. */
int kba_lidar_depth(kba_handle* h, const float* cloud, int32_t n_points, int32_t point_stride, const double* T_cam_lidar,
                    const double* intr, const float* features_uv, int32_t n_features, const kba_lidar_options* opt,
                    float* depth_out, float* device_ms);

/* ---- lidar depth for many clouds and cameras in one call -------------------------------------------------------------
 * The per-frame DepthEstimator call for many frames, and for the cameras of a rig, at once.  A view is one camera looking at
 * one cloud with one feature list; kba_lidar_depth is the batch of one view of one cloud.
 *   - Results: views[i].depth_out equals, bit for bit, kba_lidar_depth on clouds[views[i].cloud] with that view's pose,
 *     intrinsics, features and options.
 *   - Shared clouds: several views may name the same cloud; it is uploaded once per call.
 *   - Sitting out: a view with n_features == 0 is skipped and none of its other fields is read (depth_out may be NULL).  A
 *     cloud that no remaining view names is neither read, uploaded nor projected.  A call in which every view sits out returns
 *     KBA_OK at once with *device_ms = 0.
 *   - Validation, before anything is uploaded: a null pointer where data is needed (clouds or views with a positive count,
 *     the options when a view works, a working view's T_cam_lidar, intr, features_uv or depth_out, a named cloud's points
 *     when n_points > 0), a negative count, stride < 3 or a cloud index out of range: KBA_ERR_BAD_ARG.  More than INT32_MAX
 *     (view, point) pairs, cells (sum over views of ceil(w/16) * ceil(h/16) + 1) or 2 * features: KBA_ERR_CAPACITY.
 *     kba_last_error names the failing cloud or view index, and no depth_out is written.  Options are not checked.
 *   - Cost of a call: one launch sequence (memset, count, scan, fill, feature kernels) whatever the number of views; one
 *     copy per used cloud from the caller's memory; one packed upload of the features and per-view parameters; one download
 *     of all depths; one synchronisation.  The handle's grow-only device workspace takes 24 B of sorted point record per
 *     (view, point) pair, plus the used clouds, 12 B per cell, and 12 B per feature: no allocation once it is large enough.
 *   - device_ms: the kernels of the whole call, between events as in kba_lidar_depth. */
typedef struct kba_lidar_cloud {
    const float* points;        /* n_points x stride floats, xyz first (as kba_lidar_depth's cloud) */
    int32_t n_points;
    int32_t stride;             /* >= 3 */
} kba_lidar_cloud;
typedef struct kba_lidar_view {
    int32_t cloud;              /* index into clouds[] */
    int32_t n_features;         /* 0: the view sits out, depth_out is not written (may be NULL) */
    const double* T_cam_lidar;  /* 7-vector, camera <- lidar */
    const double* intr;         /* f, cx, cy */
    const float* features_uv;   /* n_features x 2 */
    float* depth_out;           /* n_features, -1 = no depth */
} kba_lidar_view;
int kba_lidar_depth_batch(kba_handle* h, int32_t n_clouds, const kba_lidar_cloud* clouds, int32_t n_views,
                          const kba_lidar_view* views, const kba_lidar_options* opt, float* device_ms);
/* opts[n_views]: view i runs with opts[i] (a rig whose cameras differ in image size, or a parameter sweep); a view that sits
 * out does not read its entry */
int kba_lidar_depth_batch_opts(kba_handle* h, int32_t n_clouds, const kba_lidar_cloud* clouds, int32_t n_views,
                               const kba_lidar_view* views, const kba_lidar_options* opts, float* device_ms);

/* ---- limo's mono-lidar frame step as one store call: the frame's depths from its lidar cloud ---------------------------
 * kba_track_frame_step with the DepthEstimator call of the front end folded in: the frame's measurements get their depths
 * from the frame's cloud on the device, and the frame step runs on those depths without a round trip through the host.
 *   - Contract: a request's d column is not read (it may be NULL).  Measurement m of camera c gets, bit for bit, the depth
 *     kba_lidar_depth_batch_opts gives it for the view with lid's cloud, pose T_cam_lidar + 7 c, the track's camera c
 *     intrinsics as created, options opt[c] and camera c's measurements (u, v) in request order as its features; a camera
 *     with no measurements is no view.  Everything after that -- res, every field of out, the store afterwards -- is exactly
 *     kba_track_frame_step on those depths.  depth_out, when set, receives the depth each measurement got (-1: none).
 *   - Checks, all before anything is uploaded, and a refused call writes no output and changes no store: the frame step's own
 *     (except for d); a null lid, T_cam_lidar or opt; a null points with n_points > 0; n_points < 0 or stride < 3
 *     (KBA_ERR_BAD_ARG); the lidar batch's 32-bit totals over the call's views (KBA_ERR_CAPACITY).  kba_last_error names
 *     the track.  Options are not checked.
 *   - Cost: the frame step's shape.  One copy of each cloud a view reads, from the caller's memory into the handle's lidar
 *     workspace (as kba_lidar_depth_batch copies it); one upload of the staging, in which the lidar views' parameters and one
 *     feature index per measurement replace the d column; one launch sequence: the lidar kernels (memset, count, scan, fill,
 *     feature), whose feature pass writes the staged d column, then k_fs_gather, k_adjust_pose and the flow kernels; one
 *     download; two synchronisations, one when no frame is selected.  The push's k_store_append and the creation read the
 *     extracted depths from the staged d column.
 *   - Transfers (kba_track_transfer_bytes / kba_track_group_transfer_bytes), with the terms of kba_track_frame_step's formulas,
 *     V the views (cameras with measurements over the W requests), R_v the size of a view's parameter record (a constant of
 *     the library build), R the run flags sum(n_runs), the clouds summed over the requests with n_meas > 0:
 *         h2d = R_1 W + R_a A + R_v V + 8 (V + 1) + sum(20 n_meas + 4 (n_kf + 1 + n_new)) + 4 ceil(R / 4)
 *               + sum(4 n_points stride) + (S ? R_2 S + R_c C + R_p P : 0)
 *         d2h = kba_track_frame_step's d2h + 4 sum over requests with depth_out of n_meas
 *     (20 bytes per measurement: the columns lm, cam, u, v and the feature index; no d column goes up).
 *   - Allocations: the frame step's, plus the handle's lidar workspace (grow-only, shared with kba_lidar_depth_batch).
 * The group forms take lid[n_tracks] next to req[n_tracks]: each request brings its own cloud; a request that sits out
 * (n_kf == 0) does not read its entry.  _opts takes one kba_options per track, as kba_track_group_frame_step_opts. */
typedef struct kba_frame_lidar {
    const float* points;                 /* the frame's cloud, n_points x stride floats, xyz first (as kba_lidar_cloud)      */
    int32_t n_points, stride;            /* n_points may be 0: every depth is -1                                               */
    const double* T_cam_lidar;           /* [7 * n_cam]: camera c <- lidar, for every camera of the track                      */
    const kba_lidar_options* opt;        /* [n_cam]: camera c's extraction options (rigs whose cameras differ in image size)   */
    float* depth_out;                    /* [n_meas] or NULL: the depth each measurement got, -1 = none                        */
} kba_frame_lidar;
int kba_track_frame_step_lidar(kba_track* t, const kba_frame_step_request* req, const kba_frame_lidar* lid, const kba_options* opt,
                               kba_frame_step_out* out, kba_result* res);
/* req[n_tracks], lid[n_tracks], out[n_tracks], res[n_tracks] */
int kba_track_group_frame_step_lidar(kba_track_group* g, const kba_frame_step_request* req, const kba_frame_lidar* lid,
                                     const kba_options* opt, kba_frame_step_out* out, kba_result* res);
/* opts[n_tracks]: track i's adjustment runs with opts[i] */
int kba_track_group_frame_step_lidar_opts(kba_track_group* g, const kba_frame_step_request* req, const kba_frame_lidar* lid,
                                          const kba_options* opts, kba_frame_step_out* out, kba_result* res);

/* ---- limo's camera callback as one store call: the frame step and, when it is due, the solve block -----------------------
 * What limo's camera callback runs on the stored window (mono_lidar.cpp:88-372, mono_standalone.cpp:134-183), minus the motion
 * prior (the caller passes pose7): the frame step, then -- when it is due (more than two keyframes and enough time since the last
 * solve, mono_lidar.cpp:243-244) -- the solve block on the landmarks the push leaves active.  Every output, both results and every
 * store afterwards equal, bit for bit, what this chain of store calls gives:
 *   1. kba_track_frame_step on req->step (with lid: kba_track_frame_step_lidar on req->step and lid), with opt_adjust;
 *   2. the solve rule: KBA_STEP_SOLVE_ALWAYS solves, KBA_STEP_SOLVE_IF_SELECTED solves iff the frame was selected (a caller whose
 *      keyframe count reaches 3 only with this frame), KBA_STEP_SOLVE_NEVER does not; the caller evaluates limo's time rule;
 *   3. the solve block's lists after the push (bundle_adjuster_keyframes.cpp:289-330): the keyframes step.kf_slot, followed by
 *      step.kf_new if the frame was selected; the landmarks, in candidate order, the candidates lm_slot[j] whose tag lm_new[j] is
 *        -2 (active before the frame): always;  -1 (an existing landmark the frame measures): iff the frame was selected;
 *        k >= 0 (step.new_slot[k], lm_slot[j] == new_slot[k]): iff the frame was selected and the creation set bit 0 of flags[k];
 *      with lm_ground[j] (NULL: none is ground) as the listed landmarks' is_ground_plane;
 *   4. if it is due, kba_track_keyframe_solve on those lists with the request's other fields (as kba_kfsolve_request takes them)
 *      and opt_solve.
 * Outputs (caller-owned): step, as the frame step writes it; solved (the solve block ran); n_lm, the list's length, and
 * lm_index [n_cand], each candidate's position in the list or -1 (both written only when solved); solve, as
 * kba_track_keyframe_solve writes it, its landmark arrays indexed by the compacted list (kf_active, kf_common sized for
 * step.n_kf + 1, the landmark arrays and rank.cand / category for n_cand); res_adjust as the frame step's res; res_solve as the
 * solve block's res (idle when it does not run).
 * On the device: the first upload stages everything the frame step stages and, for each request that may solve, the solve block's
 * lists, tags, tracklets, classes, outliers and AddDepth entries; its launch sequence and download are the frame step's.  The host
 * composes the verdicts and decides which tracks solve.  Then one upload of the push's, the creation's and the solve block's
 * argument records, and one launch sequence: k_arena_compact, k_store_append, the creation's kernels, k_cs_lists (the post-push
 * landmark list, compacted by tag, verdict and creation flag into the solve block's staged list; its length stays in device
 * memory, where the deactivation and k_kfs_labels read it) and the solve block's first part (k_up_*, k_kfs_labels, k_sel_*,
 * k_rk_prep, k_rk_depth); one download brings back the creation's and the solve block's first outputs.  From there the sequence is
 * kba_track_keyframe_solve's.  A selected, solving frame synchronises three times (the chain: four) before the solve's own.
 * Checks: every check that needs only the request runs before anything is uploaded, and a refusal there writes no output and
 * changes no store: the frame step's own; an unknown solve policy; for requests that may solve, the solve block's request checks
 * on the candidate bound n_cand (the keyframe list step.kf_slot), a null lm_slot, lm_new or lm_index with n_cand > 0, a tag below
 * -2 or at least n_new, and a k >= 0 tag named twice or not at new_slot[k] (KBA_ERR_BAD_ARG).  The solve block's late refusals
 * stay late: no keyframe kept, the solve's checks on the kept keyframes, a failing or missing draw function, the ranked solve's
 * checks.  After one, the frame step is done: out.step and res_adjust are written, every store holds the frame step's writes,
 * solved = 0 and the call returns the solve block's code -- what the chain leaves behind (all-or-nothing over the solving tracks).
 * Transfers (kba_track_transfer_bytes / kba_track_group_transfer_bytes), P the requests that may solve (solve != NEVER), each
 * with K = step.n_kf + 1 and L = n_cand, D of them solving, R_s the size of one window's argument records (a constant of the
 * library build, k_cs_lists' record included), D_w and B_w the draws and the selection bound of a solving request as
 * kba_track_keyframe_solve states them, each request's arrays padded as in kba_track_keyframe_solve:
 *         h2d = the frame step's + sum over P of (8 n_depth + 4 (K + 2 L + n_outlier + n_trk) + L + n_trk)
 *               + (D ? R_s P + 8 D + 4 sum(D_w) + the solve's : 0)
 *         d2h = the frame step's + (D ? 4 P + sum over P of (12 + 9 K + 7 L + n_trk) + 8 D + 5 sum(B_w) + the solve's : 0)
 * where the solve's are kba_track_solve_ranked's (kba_track_group_solve_ranked's) over the D solving requests.
 * Allocations: the two calls' (their staging, grow-only, is shared with kba_track_frame_step and kba_track_keyframe_solve).
 * The group forms serve one request per track (req[n_tracks], lid: NULL or lid[n_tracks], out[n_tracks], res_*[n_tracks]):
 * step.n_kf == 0 sits the call out; a request with solve == NEVER or an unmet IF_SELECTED only runs the frame step; a failing
 * request returns its code and kba_last_error names its track; _opts takes one adjustment and one solve kba_options per track.
 * A single call is the group call's one-track case. */
#define KBA_STEP_SOLVE_NEVER 0
#define KBA_STEP_SOLVE_ALWAYS 1
#define KBA_STEP_SOLVE_IF_SELECTED 2
typedef struct kba_camera_step_request {
    kba_frame_step_request step;  /* step.kf_slot: the active keyframes before the frame                                      */
    uint8_t solve;              /* KBA_STEP_SOLVE_*                                                                           */
    uint8_t reserved_[3];
    int32_t n_cand;
    int32_t min_connecting, min_window, max_window;
    int32_t n_trk;
    const int32_t* lm_slot;     /* [n_cand] the landmarks the push could leave active, ascending landmark id                   */
    const int32_t* lm_new;      /* [n_cand] their tags: -2 active before the frame, -1 measured by it, k >= 0 step.new_slot[k]  */
    const uint8_t* lm_ground;   /* [n_cand] is_ground_plane of the candidates, or NULL (none)                                  */
    const kba_tracklet* trk;    /* [n_trk] the current frame's tracklets                                                       */
    const kba_label_class* classes;  /* [n_class] */
    int32_t n_class;
    int32_t n_outlier;
    const int32_t* outlier_slot;     /* [n_outlier] the caller's current outlier set                                           */
    double shrubbery_weight;
    const kba_select_params* params; /* the ranking, as kba_kfsolve_request                                                    */
    int32_t max_near, max_middle, max_far;
    int32_t n_depth;
    const kba_depth_entry* depth;
    int32_t (*draw)(void* ctx, int32_t n, int32_t* out);
    void* draw_ctx;
    const kba_window* sel;      /* the solve's scalars and ground mode, as kba_kfsolve_request                                 */
} kba_camera_step_request;
typedef struct kba_camera_step_out {  /* caller-owned */
    kba_frame_step_out step;
    uint8_t solved;             /* the solve block ran                                                                        */
    uint8_t reserved_[3];
    int32_t n_lm;               /* the solve's landmark list length (written when solved)                                     */
    int32_t* lm_index;          /* [n_cand] each candidate's position in that list, or -1 (written when solved)               */
    kba_kfsolve_out solve;      /* landmark arrays indexed by the compacted list                                              */
} kba_camera_step_out;
int kba_track_camera_step(kba_track* t, const kba_camera_step_request* req, const kba_frame_lidar* lid, const kba_options* opt_adjust,
                          const kba_options* opt_solve, kba_camera_step_out* out, kba_result* res_adjust, kba_result* res_solve);
/* req[n_tracks], lid NULL or lid[n_tracks], out[n_tracks], res_adjust[n_tracks], res_solve[n_tracks] */
int kba_track_group_camera_step(kba_track_group* g, const kba_camera_step_request* req, const kba_frame_lidar* lid,
                                const kba_options* opt_adjust, const kba_options* opt_solve, kba_camera_step_out* out,
                                kba_result* res_adjust, kba_result* res_solve);
/* opts_adjust[n_tracks], opts_solve[n_tracks]: track i's adjustment and solve run with its entries */
int kba_track_group_camera_step_opts(kba_track_group* g, const kba_camera_step_request* req, const kba_frame_lidar* lid,
                                     const kba_options* opts_adjust, const kba_options* opts_solve, kba_camera_step_out* out,
                                     kba_result* res_adjust, kba_result* res_solve);

#ifdef __cplusplus
}
#endif
#endif /* KBA_B200_H */
