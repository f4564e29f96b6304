// kba_device.cuh -- device-side data model and per-observation math of the H100 window solver.
//
// Layout rule: everything that is streamed per observation is SoA over the whole batch (component-major), so that
// a warp touching 32 consecutive observations issues fully coalesced 128-/256-byte transactions; everything that is
// per keyframe / per camera is tiny and staged into shared memory by the consuming CTA.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "kba_plan.h"

namespace kba {

constexpr int kMaxCam = 8;
constexpr int kPoseStride = 12;     // staged pose: R (9, row-major) + t (3)
constexpr int kCamStride = 16;      // staged camera: Rc (9) + tc (3) + f, cx, cy, pad
constexpr int kIterLogCap = 160;    // iteration records kept per window

// ---- per-window descriptor (immutable after upload) --------------------------------------------------------------
struct WinDesc {
    int n_kf, n_cam, n_lm, n_obs, n_gp;
    int kf_off, cam_off, lm_off, obs_off, gp_off;  // offsets into the batch-flat arrays
    int chunk_off, n_chunks;                        // landmark chunks (32 landmarks) of the panel-based Schur kernel
    int grp_off, n_groups;                          // landmark groups (8 landmarks) of the fused Schur kernel
    int scale_kf0, scale_kf1;
    double scale_weight, scale_value;
    double plane_reg_weight;
    int plane_dist_fixed, landmarks_fixed;
    int speed_kf;
    int idle;                                       // 1: the window sits this solve out (k_reset_state: PH_DONE at once);
                                                    //    set only by kba_track_group_solve
    double speed_weight, speed_dt;
    double speed_v_before[3];
    double speed_T_origin_before[7];
    long long s_off;                                // offset (doubles) of this window's reduced-system storage
    int nr_cap;                                     // allocated rows of the reduced system (multiple of 64)
    int max_rank;                                   // > 0: some landmark is seen by several cameras in one keyframe
    long long panel_off;                            // offset (doubles) of this window's dense V panel storage
};

// ---- per-window solver state (device resident, mutated by the kernels) ----------------------------------------------
enum Phase : int { PH_SOLVE_BEGIN = 0, PH_ITERATE = 1, PH_TRIM = 2, PH_DONE = 3 };

struct SolveSummary {
    double initial_cost, final_cost;
    int num_iterations, num_successful_steps, termination, num_landmarks, num_residual_blocks, pad;
};

struct IterRecord {
    double cost, cost_change, gradient_max_norm, step_norm, relative_decrease, radius;
    int iteration, solve_index, valid, successful;
};

struct WinState {
    int phase;
    int cur;               // index of the state buffer holding x (candidate = 1 - cur)
    int need_linearize;    // x changed: Jacobian + pose-Hessian kernels must run
    int iter0;             // the pending linearisation is iteration zero of a solve (Jacobi scaling is computed)
    int solve_index;       // index of the inner solve (summary slot)
    int round;             // trimming rounds completed
    int rounds_total;
    int retried;           // the current trimming-round solve is the 3x-iterations retry
    int is_final;          // current solve is the final refinement
    int max_iter;
    int iteration;
    int num_invalid;
    int last_successful;   // the previous iteration was a successful step (gates the gradient tolerance test)
    int n_f;               // columns of the reduced system in this solve
    int nr;                // n_f + 1 rounded up to 8
    int eval_failed;       // set by evaluation kernels (|z| < 0.01)
    int solve_failed;      // reduced Cholesky / finiteness failure of the current step
    int log_n;
    int n_solves;
    int n_lin_tiles;       // warp tiles of k_linearize (built by k_solve_begin for the active landmarks of this solve)
    double radius, decrease_factor;
    double x_cost, x_norm, gmax;
    // pose-side scalars of the current step (written by the reduced solve)
    double f_model, f_step_sq, f_xnorm_sq, f_gmax;
    unsigned long long t_solve_start;  // %globaltimer (ns) when the current inner solve began: max_solver_time is per solve
    SolveSummary solves[8];
};

// ---- batch-flat device arrays --------------------------------------------------------------------------------------------
struct SolveParams;
struct BatchDev {
    int n_win;
    int max_obs, max_lm, max_kf, max_gp;   // maxima over the batch (grid sizing)
    long long tot_obs, tot_lm, tot_kf, tot_cam, tot_gp;
    WinDesc* desc;
    WinState* state;
    IterRecord* log;          // [n_win][kIterLogCap]
    // keyframes
    double* pose0;            // [tot_kf*7] uploaded state
    double* plane0;           // [tot_kf*4]
    double* pose[2];          // [tot_kf*7] x / candidate (ping-pong)
    double* rt[2];            // [tot_kf*12] the same poses as R (9, row-major) | t (3): what the observation kernels stage
                              //             with one bulk copy (written by whoever writes pose[])
    double* plane[2];         // [tot_kf*4]
    uint8_t* kf_fixed;        // [tot_kf]
    int* off_pose;            // [tot_kf] column offset in the reduced system or -1
    int* off_dir;
    int* off_dist;
    double* bkf;              // [tot_kf*27] per-keyframe J_p^T J_p (21, upper-packed row-major) + J_p^T r (6)
    double* scale_f;          // [n_win * nr_cap_max] Jacobi scaling of the f columns (indexed desc.s... see kernels)
    // cameras
    double* cam;              // [tot_cam*16] staged camera parameters
    // landmarks
    double* lm0;              // [tot_lm*3]
    double* lm[2];            // [tot_lm*3]
    double* lm_weight;        // [tot_lm]
    uint8_t* lm_active;       // [tot_lm]
    uint8_t* lm_active0;      // all ones minus landmarks without residuals
    int* lm_ptr;              // [tot_lm + n_win] CSR (window-local observation offsets), window w starts at lm_off + w
    double* lm_scale;         // [tot_lm*3] Jacobi scaling of the landmark columns
    double* lm_linv;          // [tot_lm*6] inverse Cholesky factor of the damped C_j (lower, packed)
    double* lm_z;             // [tot_lm*3] L^-1 g_j
    double* lm_g;             // [tot_lm*3] g_j = J_l^T r
    double* lm_lambda;        // [tot_lm*3] LM damping of the landmark columns
    double* trim_val;         // [3][tot_lm] per-landmark maximum raw residual norm per group
    uint8_t* trim_reject;     // [tot_lm]
    // observations, landmark-major
    int* obs_kf;              // [tot_obs]
    int* obs_cam;
    int* obs_lm;              // window-local landmark index
    int* obs_rank;            // [tot_obs] 0, or k for the k-th further observation of the same (landmark, keyframe)
    float* obs_u, *obs_v, *obs_d;
    // observations, keyframe-major copy (built on device at upload)
    int* kf_ptr;              // [tot_kf + n_win]
    int* pm_lm;               // [tot_obs]
    int* pm_cam;
    float* pm_u, *pm_v, *pm_d;
    // materialised linearisation (SoA, component stride = tot_obs)
    double* res;              // [3][tot_obs]  robustified residual rows (u, v, depth)
    double* jp;               // [18][tot_obs] 3x6 d r~ / d (rot, trans)
    double* jl;               // [9][tot_obs]  3x3 d r~ / d landmark
    // dense per-chunk V panels for the TMA-fed Schur kernel: chunk c of window w occupies 96 columns x chunk_rs[c] rows,
    // column-major ([col][row]), at vpanel + desc.panel_off + chunk_poff[c]; rows = the chunk's 8-row tile range (+ rhs tile)
    double* vpanel;
    long long panel_cap;      // doubles reserved per window
    int* chunk_poff;          // [tot_chunks] offset (doubles) inside the window's panel storage
    int* chunk_rs;            // [tot_chunks] row stride (== 4 mod 16, 0 for chunks without free keyframes)
    // reductions
    double* cost_part_x;      // [n_win][cost_parts] cost partials of the linearisation at x
    double* cost_part_c;      // [n_win][cost_parts] cost partials at the candidate
    int cost_parts;
    // ---- one window sharded by landmark blocks over several GPUs (kba_shard.cu) ----
    int sharded;              // 1: this batch holds ONE window's shard; sums cross the ranks through LaunchCfg::xchg
    int lm_begin, lm_total;   // first landmark of this rank's block / landmarks of the whole window (caller's order)
    int shard_rank, shard_world;
    double* xs;               // [16 + world] exchanged scalars (ONE sum all-reduce after the back substitution): 0 model, 1 step^2,
                              //      2 |x|^2, 3 candidate cost, 4 eval-failed flag, 5 ground-plane cost at the candidate,
                              //      16 + r: gradient max-norm of rank r
    double* x_send;           // [nr_cap^2 + 27 n_kf (+ 65 n_kf + 1) + shard_cost_parts + 2] packed linearisation of this rank
    double* x_recv;           //      (k_shard_pack) and its sum over the ranks (ONE all-reduce per linearisation)
    double* trim_send;        // [3][lm_total] this rank's trimming values (+2, 0 where not owned), all-reduced into
    double* trim_glob;        // [3][lm_total]
    uint8_t* reject_glob;     // [lm_total]
    int shard_cost_parts;     // cost partial slots in the exchange: the largest cost_parts of the ranks (zero padded)
    int shard_gp;             // 1: some rank holds ground-plane residuals -- plane blocks, gp blocks and gp costs are window-wide
    double* gp_send;          // [lm_total] keyframe + 1 of this rank's landmarks' ground-plane residuals (0: none), summed into
    double* gp_kf_glob;       //      [lm_total] the same for the whole window (once per kba_batch_solve, k_shard_gp_gather)
    uint8_t* act_glob;        // [lm_total] landmark not trimmed in the whole window (k_reset_state, k_trim_select)
    uint8_t* kf_gp_glob;      // [n_kf] an active ground point of some rank is attached to the keyframe (k_shard_planes)
    int precision;            // 0: FP64; 1: residual / Jacobian blocks evaluated and stored in FP32 (res, jp, jl hold floats),
                              //    every accumulation (landmark blocks, Schur products, solve, cost) stays FP64
    int solve_tiled;          // 1: k_reduced_solve<true> (<= kTiledMaxRows rows, shared-memory resident)
    int solve_split;          // > 0: large system of a small batch, factorisation spread over this many CTAs per window
    int solve_banded;         // 1: above kPanelMaxRows rows: k_sred_reduce writes A, k_chol_trail_band updates the trailing matrix
    double* chol_w;           // [n_win][32*32] inverse of the current diagonal block's factor (split factorisation)
    double* chol_invd;        // [n_win][nr_cap_max] 1 / L_ii
    double* bs_part;          // [n_win][bs_parts][4]: model_e, step_sq, xnorm_sq, gmax_e
    int bs_parts;
    int nr_cap_max;           // largest nr_cap in the batch = stride of scale_f / lambda_f / grad_f / delta_f
    // reduced system
    double* sred;             // per window nr_cap x nr_cap (row-major, lower part valid) x p_split partial copies
    int p_split;
    double* delta_f;          // [n_win * nr_cap]
    double* lambda_f;         // [n_win * nr_cap]
    double* grad_f;           // [n_win * nr_cap]
    double* amat;             // per window nr_cap x nr_cap scratch for the factorisation
    // chunking of landmarks for the Schur kernel
    int* chunk_lm0;           // [tot_chunks] first landmark (window-local)
    int* chunk_lm1;           // [tot_chunks] one past last
    int* chunk_k0;            // [tot_chunks] first / last keyframe observed by the chunk's landmarks (host, static)
    int* chunk_k1;
    int* chunk_t0;            // [tot_chunks] 8-row tile range [t0, t1) of the reduced system the chunk touches (per solve)
    int* chunk_t1;
    int* obs_row;             // [tot_obs] first reduced-system row of the observation's pose block, -1: constant / inactive
    int* lm_orig;             // [tot_lm] caller's landmark index (landmarks are stored sorted by first keyframe)
    int tot_chunks;
    // fused small-window path (k_schur_fused): J_l is not materialised (J_l = translation columns of J_p times R), the V
    // panels exist only in shared memory; per 8-landmark group the keyframe range (host, static) and, per solve, the
    // 8-row tile range of the reduced system it touches and the rows of its shared-memory panel
    int fused;                // 1: every window of the batch has <= kFusedMaxRows reduced rows -> fused path, jl / vpanel unused
    int* grp_k0;              // [tot_groups]
    int* grp_k1;
    int* grp_t0;              // [tot_groups] tile range [t0, t1) aligned to 16-row blocks
    int* grp_t1;
    int* grp_tiles;           // [tot_groups] t0 | t1 << 8 | e0 << 16 | e1 << 24: [e0, e1) = the exact tile range inside
                              //   [t0, t1), right-hand-side tile included (what the consumer warps read, in one register)
    int* grp_rs;              // [tot_groups] panel rows (multiple of 8), 0: no free keyframe rows
    double* vobs;             // [18 * tot_obs] V_i = (J_p^T J_l) L^-T of every observation, unpadded.  Per landmark with
                              //   observations [p0, p1), n = p1 - p0: column c of observation i at 18 (obs_off + p0) + 6 n c + 6 i
                              //   (6 rows each), so a whole panel column of the landmark is ONE contiguous run
    int4* lm_run;             // [tot_lm] {a, m, row, 0}: observations p0 + a .. p0 + a + m - 1 are the landmark's observations
                              //   with variable poses and sit on consecutive reduced-system rows row, row + 6, ...;
                              //   m = 0: none, m = -1: they do not form one such run (gaps, several cameras, plane rows)
    int lin1;                 // 1: this solve linearises with k_linearize (fused path, FP64, <= 1 observation per landmark and keyframe);
                              //    set per solve by kba_batch_solve.  Also: the cost at x is evaluated at iteration zero only
    int2* lin_tile;           // [tot_obs / 16 + 2 n_win + 2] warp tiles of k_linearize: {first observation, count <= 32} (kba_linearize.cuh)
    unsigned long long* prof; // [16] cycle counters of a KBA_PROF build (nullptr otherwise)
    int tot_groups;
    int* n_active;            // [1] windows still running (device counter)
    unsigned long long* jac_obs;  // [1] observations linearised by the residual/Jacobian kernel since the last reset
    // ground-plane height residuals (one per ground landmark, attached to a keyframe by the host)
    int* gp_lm;               // [tot_gp] window-local (sorted) landmark index
    int* gp_kf;               // [tot_gp] keyframe index
    double* gp_weight;        // [tot_gp] ScaledLoss weight
    int* gp_of_lm;            // [tot_lm] window-local gp index of the landmark or -1
    int* gp_shared;           // [tot_gp] 1: the landmark is also observed from the gp keyframe (same pose rows)
    double* gp_lin;           // [14][tot_gp] robustified residual, J_f (pose 6, dir 3 local, dist 1), J_l (3)
    double* vgp;              // [30][tot_gp] V rows of the gp residual: (J_f^T J_l) L^-T, 10 x 3
    double* gp_kfb;           // [tot_kf*65] per keyframe: its 10 x 10 (pose | normal | distance) Gauss-Newton block over the active
                              //   gp residuals (55, lower-packed by rows) + the 10 gradient entries (k_gp_blocks)
    double* gp_cost_x;        // [n_win] robustified cost of the gp blocks at x / at the candidate (fixed-order sums)
    double* gp_cost_c;
    const SolveParams* wsp;   // [n_win] solver options of each window (every pass kernel reads its window's entry)
};

// kba_options subset used on the device, one per window (BatchDev::wsp) or per frame (MotionArgs::sp).  The host compares the
// bytes with what the device holds, so every byte is a field (no padding).
struct SolveParams {
    double gp_huber, gp_quantile;
    double depth_thres, reprojection_thres, depth_quantile, reprojection_quantile;
    double function_tolerance, gradient_tolerance, parameter_tolerance;
    double initial_radius, max_radius, min_radius, min_relative_decrease, min_lm_diagonal, max_lm_diagonal;
    int trim_solver_iterations, final_solver_iterations, min_residual_groups, max_consecutive_invalid_steps;
    double max_solver_time;  // seconds per inner solve (ceres max_solver_time_in_seconds), <= 0: none
    // trimming rounds (k_reset_state): num_trim_rounds, or -1 = num_rounds_option iff the window has more than
    // min_landmarks_for_trimming landmarks
    int rounds_override, min_landmarks_for_trimming, num_rounds_option, pad_;
};

__device__ __forceinline__ unsigned long long global_timer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// ---- small math ----------------------------------------------------------------------------------------------------------
template <typename T>
__host__ __device__ inline void quat_to_rot(const T* q, T* R) {
    // Eigen::Quaternion::toRotationMatrix, no normalisation (reference definitions.hpp:75-83)
    const T w = q[0], x = q[1], y = q[2], z = q[3];
    const T tx = 2 * x, ty = 2 * y, tz = 2 * z;
    const T twx = tx * w, twy = ty * w, twz = tz * w, txx = tx * x, txy = ty * x, txz = tz * x;
    const T tyy = ty * y, tyz = tz * y, tzz = tz * z;
    R[0] = 1 - (tyy + tzz); R[1] = txy - twz;       R[2] = txz + twy;
    R[3] = txy + twz;       R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
    R[6] = txz - twy;       R[7] = tyz + twx;       R[8] = 1 - (txx + tyy);
}

// Ceres QuaternionParameterization::Plus x Identity(3) (reference bundle_adjuster_keyframes.cpp:181-182)
__host__ __device__ inline void pose_plus(const double* p, const double* d, double* o) {
    const double nd = sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
    if (nd > 0.0) {
        const double s = sin(nd) / nd, c = cos(nd);
        const double q0 = c, q1 = s * d[0], q2 = s * d[1], q3 = s * d[2];
        o[0] = q0 * p[0] - q1 * p[1] - q2 * p[2] - q3 * p[3];
        o[1] = q0 * p[1] + q1 * p[0] + q2 * p[3] - q3 * p[2];
        o[2] = q0 * p[2] - q1 * p[3] + q2 * p[0] + q3 * p[1];
        o[3] = q0 * p[3] + q1 * p[2] - q2 * p[1] + q3 * p[0];
    } else {
        o[0] = p[0]; o[1] = p[1]; o[2] = p[2]; o[3] = p[3];
    }
    o[4] = p[4] + d[3]; o[5] = p[5] + d[4]; o[6] = p[6] + d[5];
}

// Robust loss of one residual block: ScaledLoss(CauchyLoss(a), w): rho = w b log(1 + s/b), rho' = w / (1 + s/b)
template <typename T, bool kCost = true>
__device__ inline void cauchy(T b, T w, T s, T& half_rho, T& sqrt_rho1) {
    const T sum = T(1) + s / b;
    half_rho = kCost ? T(0.5) * w * b * log(sum) : T(0);  // callers that only need the Jacobian rows skip the log
    sqrt_rho1 = sqrt(w / sum);
}

// One observation: reprojection (2 rows) + optional lidar depth row, robustified, in the factored form of its Jacobian.
// pose: staged R(9)+t(3); cam: staged Rc(9)+tc(3)+f,cx,cy.  With m = (rows of d Pi / d x_cam, robustified) * Rc (3x3, row-major)
// and a = R p, the Jacobian rows are d/d(delta_rot) = -2 (m_i x a), d/d(delta_t) = m_i, d/d(p) = m_i R, i.e.
//   J_pose = m [K | I] with K = -2 [a]x,   J_landmark = m R      (reference cost_functors_ceres.hpp:91-155,193-212),
// so every Gauss-Newton product follows from M = m^T m, m^T r and a.  kM: also form m.
// Returns false when |z_cam| < 0.01 (evaluation failure, cost_functors_ceres.hpp:78-83).
template <typename T, bool kM, bool kCost = true>
__device__ __forceinline__ bool eval_factored(const T* __restrict__ pose, const T* __restrict__ cam, const T p[3], T u, T v,
                                              T d, T wt, T b_repr, T b_depth, T r[3], T m[9], T a[3], T& half_rho_sum,
                                              T raw[2]) {
    a[0] = pose[0] * p[0] + pose[1] * p[1] + pose[2] * p[2];
    a[1] = pose[3] * p[0] + pose[4] * p[1] + pose[5] * p[2];
    a[2] = pose[6] * p[0] + pose[7] * p[1] + pose[8] * p[2];
    const T x0 = a[0] + pose[9], x1 = a[1] + pose[10], x2 = a[2] + pose[11];
    const T c0 = cam[0] * x0 + cam[1] * x1 + cam[2] * x2 + cam[9];
    const T c1 = cam[3] * x0 + cam[4] * x1 + cam[5] * x2 + cam[10];
    const T c2 = cam[6] * x0 + cam[7] * x1 + cam[8] * x2 + cam[11];
    if (!(fabs(c2) >= T(0.01))) return false;
    const bool has_d = d > T(0);
    const T rd = has_d ? c2 - d : T(0);  // formed first: c2 and d need not outlive the divisions below
    const T f = cam[12], iz = T(1) / c2;
    const T xn = c0 * iz, yn = c1 * iz;
    const T ru = f * xn + cam[13] - u, rv = f * yn + cam[14] - v;
    const T s = ru * ru + rv * rv;
    T hr, sq;
    cauchy<T, kCost>(b_repr, wt, s, hr, sq);
    half_rho_sum = hr;
    raw[0] = sqrt(s);
    raw[1] = T(-1);
    r[0] = sq * ru; r[1] = sq * rv; r[2] = T(0);
    T sqd = T(0);
    if (has_d) {
        T hrd;
        cauchy<T, kCost>(b_depth, wt, rd * rd, hrd, sqd);
        half_rho_sum += hrd;
        raw[1] = fabs(rd);
        r[2] = sqd * rd;
    }
    if (kM) {
        const T fz = f * iz * sq;  // robustified
        // m rows: (fz * Rc[0,:] - fz*xn * Rc[2,:]), (fz * Rc[1,:] - fz*yn * Rc[2,:]), sqd * Rc[2,:]
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            m[c] = fz * (cam[c] - xn * cam[6 + c]);
            m[3 + c] = fz * (cam[3 + c] - yn * cam[6 + c]);
            m[6 + c] = sqd * cam[6 + c];
        }
    }
    return true;
}

// index of entry (i, j) of a symmetric 3x3 matrix stored upper, row-major: 00 01 02 11 12 22
__host__ __device__ constexpr int sym3(int i, int j) {
    return i <= j ? 3 * i + j - i * (i + 1) / 2 : 3 * j + i - j * (j + 1) / 2;
}

// M = m^T m (sym3 layout) of a factored evaluation
__device__ __forceinline__ void gram_factored(const double m[9], double M[6]) {
    M[0] = m[0] * m[0] + m[3] * m[3] + m[6] * m[6];
    M[1] = m[0] * m[1] + m[3] * m[4] + m[6] * m[7];
    M[2] = m[0] * m[2] + m[3] * m[5] + m[6] * m[8];
    M[3] = m[1] * m[1] + m[4] * m[4] + m[7] * m[7];
    M[4] = m[1] * m[2] + m[4] * m[5] + m[7] * m[8];
    M[5] = m[2] * m[2] + m[5] * m[5] + m[8] * m[8];
}

// eval_factored with the Jacobian rows spelled out: J_pose (3x6, row-major) and J_landmark (3x3)
template <typename T, bool kJac, bool kCost = true>
__device__ inline bool eval_observation(const T* __restrict__ pose, const T* __restrict__ cam, const T p[3], T u, T v,
                                        T d, T wt, T b_repr, T b_depth, T r[3], T jp[18], T jl[9], T& half_rho_sum,
                                        T raw[2]) {
    T m[9], a[3];
    if (!eval_factored<T, kJac, kCost>(pose, cam, p, u, v, d, wt, b_repr, b_depth, r, m, a, half_rho_sum, raw)) return false;
    if (kJac) {
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            const T* mi = m + 3 * i;
            jp[6 * i + 0] = T(-2) * (mi[1] * a[2] - mi[2] * a[1]);
            jp[6 * i + 1] = T(-2) * (mi[2] * a[0] - mi[0] * a[2]);
            jp[6 * i + 2] = T(-2) * (mi[0] * a[1] - mi[1] * a[0]);
            jp[6 * i + 3] = mi[0];
            jp[6 * i + 4] = mi[1];
            jp[6 * i + 5] = mi[2];
#pragma unroll
            for (int c = 0; c < 3; ++c) jl[3 * i + c] = mi[0] * pose[c] + mi[1] * pose[3 + c] + mi[2] * pose[6 + c];
        }
    }
    return true;
}

// Streaming form of eval_observation for the residual/Jacobian kernel: every Jacobian row is written to its SoA slot
// as soon as it is formed, so at most one 3-vector m and the rotated point a stay live (64 registers -> 4 CTAs/SM).
// res/jp/jl point at this observation's slot of component 0; `stride` is the component stride (total observations).
// kJl: also store J_landmark (panel path)
// kArm: p and the translation of `pose` are taken relative to an anchor c (p - c and t + R c), so that x = R (p - c) + (t + R c)
// is formed from window-sized terms; arm = R c restores the rotation columns' lever arm a = R p = R (p - c) + R c, since the
// parametrisation rotates about the origin, not about c
template <typename T, bool kJl = true, bool kArm = false>
__device__ inline bool eval_observation_store(const T* __restrict__ pose, const T* __restrict__ cam, const T p[3], T u,
                                              T v, T d, T wt, T b_repr, T b_depth, T* __restrict__ res,
                                              T* __restrict__ jp, T* __restrict__ jl, size_t stride, bool write_jp,
                                              T& half_rho_sum, const T* __restrict__ arm = nullptr) {
    const T b0 = pose[0] * p[0] + pose[1] * p[1] + pose[2] * p[2];
    const T b1 = pose[3] * p[0] + pose[4] * p[1] + pose[5] * p[2];
    const T b2 = pose[6] * p[0] + pose[7] * p[1] + pose[8] * p[2];
    const T x0 = b0 + pose[9], x1 = b1 + pose[10], x2 = b2 + pose[11];
    const T a0 = kArm ? b0 + arm[0] : b0, a1 = kArm ? b1 + arm[1] : b1, a2 = kArm ? b2 + arm[2] : b2;
    const T c0 = cam[0] * x0 + cam[1] * x1 + cam[2] * x2 + cam[9];
    const T c1 = cam[3] * x0 + cam[4] * x1 + cam[5] * x2 + cam[10];
    const T c2 = cam[6] * x0 + cam[7] * x1 + cam[8] * x2 + cam[11];
    if (!(fabs(c2) >= T(0.01))) return false;
    const T f = cam[12], iz = T(1) / c2;
    const T xn = c0 * iz, yn = c1 * iz;
    const T ru = f * xn + cam[13] - u, rv = f * yn + cam[14] - v;
    T hr, sq;
    cauchy<T>(b_repr, wt, ru * ru + rv * rv, hr, sq);
    half_rho_sum = hr;
    T sqd = T(0), rd = T(0);
    if (d > T(0)) {
        rd = c2 - d;
        T hrd;
        cauchy<T>(b_depth, wt, rd * rd, hrd, sqd);
        half_rho_sum += hrd;
    }
    res[0] = sq * ru;
    res[stride] = sq * rv;
    res[2 * stride] = sqd * rd;
    const T fz = f * iz * sq;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        T m0, m1, m2;
        if (i == 0) { m0 = fz * (cam[0] - xn * cam[6]); m1 = fz * (cam[1] - xn * cam[7]); m2 = fz * (cam[2] - xn * cam[8]); }
        else if (i == 1) { m0 = fz * (cam[3] - yn * cam[6]); m1 = fz * (cam[4] - yn * cam[7]); m2 = fz * (cam[5] - yn * cam[8]); }
        else { m0 = sqd * cam[6]; m1 = sqd * cam[7]; m2 = sqd * cam[8]; }
        if (write_jp) {
            T* o = jp + (size_t)(6 * i) * stride;
            o[0] = T(-2) * (m1 * a2 - m2 * a1);
            o[stride] = T(-2) * (m2 * a0 - m0 * a2);
            o[2 * stride] = T(-2) * (m0 * a1 - m1 * a0);
            o[3 * stride] = m0;
            o[4 * stride] = m1;
            o[5 * stride] = m2;
        }
        if (kJl) {
            T* q = jl + (size_t)(3 * i) * stride;
            q[0] = m0 * pose[0] + m1 * pose[3] + m2 * pose[6];
            q[stride] = m0 * pose[1] + m1 * pose[4] + m2 * pose[7];
            q[2 * stride] = m0 * pose[2] + m1 * pose[5] + m2 * pose[8];
        }
    }
    return true;
}

// entry `idx` of a materialised linearisation stream (res / jp / jl): doubles, or floats when BatchDev::precision == 1
__device__ __forceinline__ double lin_load(const double* base, size_t idx, int precision) {
    return precision ? (double)reinterpret_cast<const float*>(base)[idx] : base[idx];
}

// stage keyframe poses (as R|t) and cameras of one window into shared memory
__device__ inline void stage_window(const WinDesc& wd, const double* __restrict__ pose7, const double* __restrict__ cam16,
                                    double* s_pose, double* s_cam) {
    for (int k = threadIdx.x; k < wd.n_kf; k += blockDim.x) {
        const double* p = pose7 + 7 * (size_t)(wd.kf_off + k);
        double R[9];
        quat_to_rot<double>(p, R);
#pragma unroll
        for (int i = 0; i < 9; ++i) s_pose[kPoseStride * k + i] = R[i];
        s_pose[kPoseStride * k + 9] = p[4];
        s_pose[kPoseStride * k + 10] = p[5];
        s_pose[kPoseStride * k + 11] = p[6];
    }
    for (int i = threadIdx.x; i < wd.n_cam * kCamStride; i += blockDim.x) s_cam[i] = cam16[(size_t)wd.cam_off * kCamStride + i];
}

// staged form of a pose: R (9, row-major) | t (3); kept next to pose[] by every kernel that writes a pose
__device__ inline void write_rt(double* rt12, const double* p7) {
    quat_to_rot<double>(p7, rt12);
    rt12[9] = p7[4]; rt12[10] = p7[5]; rt12[11] = p7[6];
}

// V_i of observation o (window-local index) of a landmark with observations [p0, p1): address of column c
__device__ __forceinline__ size_t vobs_index(size_t obs_off, int p0, int p1, int o, int c) {
    return 18 * (obs_off + (size_t)p0) + (size_t)(6 * (p1 - p0)) * c + (size_t)6 * (o - p0);
}

// ---- mbarrier / bulk-copy (TMA) primitives ------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_1d(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t done = 0;
    while (!done)
        asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}"
                     : "=r"(done)
                     : "r"(smem_u32(bar)), "r"(parity)
                     : "memory");
}

// Keyframe poses (R | t, BatchDev::rt) and cameras of one window into shared memory with two bulk copies issued by one
// thread (cp.async.bulk + mbarrier): the consuming CTA does no per-pose arithmetic and no scalar staging loads.
// s_pose / s_cam must be 16-byte aligned; `bar` is a CTA-local mbarrier used once.  Every thread of the CTA calls this.
__device__ inline void stage_window_bulk(const WinDesc& wd, const double* __restrict__ rt, const double* __restrict__ cam16,
                                         double* s_pose, double* s_cam, uint64_t* bar) {
    if (threadIdx.x == 0) {
        mbar_init(bar, 1);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const uint32_t bp = (uint32_t)(wd.n_kf * kPoseStride * sizeof(double)), bc = (uint32_t)(wd.n_cam * kCamStride * sizeof(double));
        mbar_expect_tx(bar, bp + bc);
        tma_load_1d(s_pose, rt + (size_t)kPoseStride * wd.kf_off, bp, bar);
        tma_load_1d(s_cam, cam16 + (size_t)kCamStride * wd.cam_off, bc, bar);
    }
    mbar_wait(bar, 0);
}

__device__ inline double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ inline double warp_max(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

}  // namespace kba
