// kba_motion.cu -- adjustPoseOnly (reference bundle_adjuster_keyframes.cpp:820-888) as ONE kernel per frame: one free 6-DoF pose
// against constant landmarks read from a track's store, the optional SpeedRegularizationVector2 prior, and solveTrimmed's
// trimming rounds.  One CTA runs the whole trimmed solve of its frame: the 6x6 system needs no Schur complement, no reduced
// solve over several CTAs and no host round trip per pass, so the batch path's 11-13 launches per iteration collapse into
// loop iterations of one block.  The decisions (LM controller, trimming select) are the batch kernels' own
// (kba_controller.cuh), so a frame takes the iterations the equivalent landmarks_fixed window takes through kba_solve_window.
#include "kba_device.cuh"
#include "kba_kernels.h"
#include "kba_regularisers.cuh"
#include "kba_controller.cuh"

#include <type_traits>

namespace kba {

constexpr int kMotionThreads = 256;
constexpr int kMotionWarps = kMotionThreads / 32;
constexpr int kNAcc = 28;  // B (21, upper-packed 6x6, rows rot 0-2 | trans 3-5) + g (6) + cost
constexpr int kNReg = 19;  // of those in registers: the rotation rows of B (15), K^T h (3), cost; M (6) and h (3) in shared memory

// Pose-side Gauss-Newton sums of one observation in factored form (kba_device.cuh: eval_factored): J_p = m [K | I] with
// K = -2 [a]x, so with M = m^T m and h = m^T r:  J_p^T J_p = [K^T M K, K^T M; M K, M],  J_p^T r = [K^T h; h]  (as k_pose_hessian,
// with the same split: 18 sums in registers, the 9 of M and h in this thread's column of s_acc)
__device__ __forceinline__ void add_pose_block(const double m[9], const double r[3], const double a[3], double acc[kNReg],
                                               double (*s_acc)[kMotionThreads]) {
    double mm[6], h[3];
    gram_factored(m, mm);
#pragma unroll
    for (int c = 0; c < 3; ++c) h[c] = m[c] * r[0] + m[3 + c] * r[1] + m[6 + c] * r[2];
#pragma unroll
    for (int i = 0; i < 3; ++i) {  // row i of P = K^T M: P[i][c] = 2 (a x M_c)_i
        const int i1 = (i + 1) % 3, i2 = (i + 2) % 3;
        double pr[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) pr[c] = 2.0 * (a[i1] * mm[sym3(i2, c)] - a[i2] * mm[sym3(i1, c)]);
        const int qd = 6 * i - i * (i - 1) / 2;  // packed index of (i, i) in the upper 6x6
#pragma unroll
        for (int j = i; j < 3; ++j) {  // (K^T M K)[i][j] = 2 (a x row_i(P))_j
            const int j1 = (j + 1) % 3, j2 = (j + 2) % 3;
            acc[qd + j - i] += 2.0 * (a[j1] * pr[j2] - a[j2] * pr[j1]);
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) acc[qd + 3 - i + c] += pr[c];
        acc[15 + i] += 2.0 * (a[i1] * h[i2] - a[i2] * h[i1]);
    }
#pragma unroll
    for (int q = 0; q < 6; ++q) s_acc[q][threadIdx.x] += mm[q];
#pragma unroll
    for (int c = 0; c < 3; ++c) s_acc[6 + c][threadIdx.x] += h[c];
}

// the staged form (R | t) of a 7-vector pose into shared memory
__device__ __forceinline__ void stage_rt(const double* p7, double* rt) {
    if (threadIdx.x == 0) write_rt(rt, p7);
    __syncthreads();
}

// One CTA per SM: at two (128 registers) the kernel spills; at one it takes 235 registers and none.
__global__ void __launch_bounds__(kMotionThreads, 1) k_adjust_pose(MotionArgs A) {
    const FrameDesc& F = A.fd[blockIdx.x];
    const SolveParams& sp = A.sp[blockIdx.x];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    __shared__ WinState s_st;
    __shared__ double s_pose[2][7];             // x / candidate (ping-pong by s_st.cur, as BatchDev::pose)
    __shared__ __align__(16) double s_rt[kPoseStride];
    __shared__ __align__(16) double s_cam[kMaxCam * kCamStride];
    __shared__ double s_red[kMotionWarps][kNAcc];
    __shared__ double s_acc[9][kMotionThreads];    // per-thread sums of M and h (add_pose_block)
    __shared__ double s_B[27];                  // B (21) and g (6) of the current linearisation
    __shared__ double s_scale[6];               // Jacobi scaling of the solve (iteration zero)
    __shared__ double s_L[36], s_fd[6], s_g[6], s_lam[6], s_y[6];  // thread 0's 6x6 step (shared: keeps the CTA's registers low)
    __shared__ double s_sum;                    // reduced candidate cost
    __shared__ int s_cnt[2];
    __shared__ TrimSmem s_trim;

    const int n_runs = F.n_runs;
    const int* rs = A.run_start + F.rs_off;
    const size_t mo = (size_t)F.meas_off;
    double* pw = A.run_pw + 4 * (size_t)F.run_off;
    unsigned char* act = A.run_active + F.run_off;
    unsigned char* rej = A.run_rej + F.run_off;
    double* tv = A.trim_val + F.run_off;        // group 0 (depth); group 1 (reprojection) at + total_runs
    IterRecord* log = A.log + (size_t)blockIdx.x * kIterLogCap;
    const double b_repr = sp.reprojection_thres * sp.reprojection_thres, b_depth = sp.depth_thres * sp.depth_thres;
    const bool speed = F.speed_weight > 0;
    // the frame's measurements (local copies: a lambda that captured the kernel parameter by reference would copy it to the stack)
    const int* __restrict__ cams = A.cam ? A.cam + mo : nullptr;
    const float* __restrict__ mu = A.u + mo;
    const float* __restrict__ mv = A.v + mo;
    const float* __restrict__ md = A.d + mo;
    double* tv_r = tv + A.total_runs;

    // ---- prologue: the frame's landmarks from the store (by slot), cameras, initial pose, solver state (k_reset_state) ----
    for (int r = tid; r < n_runs; r += kMotionThreads) {
        const int slot = A.lm_slot[mo + rs[r]];
        pw[4 * r + 0] = F.lm_pos[3 * (size_t)slot];
        pw[4 * r + 1] = F.lm_pos[3 * (size_t)slot + 1];
        pw[4 * r + 2] = F.lm_pos[3 * (size_t)slot + 2];
        pw[4 * r + 3] = F.lm_weight[slot];
        act[r] = 1;
    }
    for (int i = tid; i < F.n_cam * kCamStride; i += kMotionThreads) s_cam[i] = F.cam16[i];
    if (tid < 7) { s_pose[0][tid] = F.pose7[tid]; s_pose[1][tid] = F.pose7[tid]; }
    if (tid == 0) {
        WinState& st = s_st;
        st.phase = PH_SOLVE_BEGIN;
        st.cur = 0;
        st.solve_index = 0; st.round = 0; st.retried = 0; st.log_n = 0; st.n_solves = 0;
        st.rounds_total = F.rounds_total;
        st.is_final = (F.rounds_total == 0);
        st.eval_failed = 0; st.solve_failed = 0;
        st.f_model = 0; st.f_step_sq = 0; st.f_xnorm_sq = 0; st.f_gmax = 0;
    }
    __syncthreads();

    // every observation of the active runs at the staged pose s_rt: kLin -> B, g and the cost into s_red, else the cost only;
    // returns (block-uniformly) whether an observation failed to evaluate (|z_cam| < 0.01).  Fixed-order reduction: warp
    // butterflies, then thread 0 over the warps in index order.
    auto evaluate = [&](auto lin_tag) -> bool {
        constexpr bool kLin = decltype(lin_tag)::value;
        double acc[kLin ? kNReg : 1];
#pragma unroll
        for (int q = 0; q < (kLin ? kNReg : 1); ++q) acc[q] = 0.0;
        if constexpr (kLin) {
#pragma unroll
            for (int q = 0; q < 9; ++q) s_acc[q][tid] = 0.0;
        }
        int failed = 0;
        for (int r = tid; r < n_runs; r += kMotionThreads) {
            if (!act[r]) continue;
            const double4 q4 = *reinterpret_cast<const double4*>(pw + 4 * r);
            const double p[3] = {q4.x, q4.y, q4.z};
            for (int o = rs[r]; o < rs[r + 1]; ++o) {
                const int c = cams ? cams[o] : 0;
                double res[3], m[9], a[3], raw[2], hr;
                if (!eval_factored<double, kLin, true>(s_rt, s_cam + kCamStride * c, p, (double)mu[o], (double)mv[o],
                                                       (double)md[o], q4.w, b_repr, b_depth, res, m, a, hr, raw)) {
                    failed = 1;
                    continue;
                }
                if constexpr (kLin) {
                    add_pose_block(m, res, a, acc, s_acc);
                    acc[18] += hr;
                } else {
                    acc[0] += hr;
                }
            }
        }
        if constexpr (kLin) {  // output order: B (21), g (6), cost
#pragma unroll
            for (int q = 0; q < kNAcc; ++q) {
                const double t = q < 15 ? acc[q] : q < 21 ? s_acc[q - 15][tid] : q < 24 ? acc[q - 6] : q < 27 ? s_acc[q - 18][tid] : acc[18];
                const double v = warp_sum(t);
                if (lane == 0) s_red[warp][q] = v;
            }
        } else {
            const double v = warp_sum(acc[0]);
            if (lane == 0) s_red[warp][0] = v;
        }
        return __syncthreads_or(failed) != 0;
    };

    for (;;) {
        __syncthreads();
        const int phase = s_st.phase;
        if (phase == PH_DONE) break;

        if (phase == PH_SOLVE_BEGIN) {  // k_solve_begin: the program of this inner solve
            if (tid < 2) s_cnt[tid] = 0;
            __syncthreads();
            int n_blocks = 0, n_lm_in = 0;
            for (int r = tid; r < n_runs; r += kMotionThreads) {
                if (!act[r]) continue;
                n_lm_in++;
                for (int o = rs[r]; o < rs[r + 1]; ++o) n_blocks += (md[o] > 0.0f) ? 2 : 1;
            }
            if (n_blocks) atomicAdd(&s_cnt[0], n_blocks);
            if (n_lm_in) atomicAdd(&s_cnt[1], n_lm_in);
            __syncthreads();
            if (tid == 0) {
                WinState& st = s_st;
                st.n_f = (s_cnt[1] > 0 || speed) ? 6 : 0;  // the pose is in the program iff a residual block references it
                st.nr = (st.n_f + 1 + 7) & ~7;
                st.radius = sp.initial_radius;
                st.decrease_factor = 2.0;
                st.iteration = 0;
                st.num_invalid = 0;
                st.last_successful = 0;
                st.need_linearize = 1;
                st.iter0 = 1;
                st.eval_failed = 0;
                st.solve_failed = 0;
                st.max_iter = st.is_final ? sp.final_solver_iterations
                                          : (st.retried ? 3 * sp.trim_solver_iterations : sp.trim_solver_iterations);
                SolveSummary& s = st.solves[st.solve_index];
                s.initial_cost = s.final_cost = 0.0;
                s.num_iterations = 0; s.num_successful_steps = 0; s.termination = 1;
                s.num_landmarks = 0;  // landmark blocks are constant: none is in the program
                s.num_residual_blocks = s_cnt[0] + (speed ? 1 : 0);
                st.t_solve_start = global_timer_ns();
                st.phase = PH_ITERATE;
            }
            continue;
        }

        if (phase == PH_ITERATE) {
            const int cur = s_st.cur;
            if (s_st.need_linearize) {  // linearise at x
                stage_rt(s_pose[cur], s_rt);
                const bool failed = evaluate(std::true_type{});
                if (tid == 0) {
                    for (int q = 0; q < kNAcc; ++q) {
                        double v = 0.0;
                        for (int w = 0; w < kMotionWarps; ++w) v += s_red[w][q];
                        if (q < 27) s_B[q] = v; else if (s_st.iter0) s_st.x_cost = v;  // the regulariser's cost is added below
                    }
                    if (failed) s_st.eval_failed = 1;
                }
            }
            // ---- the 6x6 step (k_reduced_solve for one free pose and no landmark blocks), thread 0 ----
            if (tid == 0) {
                WinState& st = s_st;
                const bool eval_cost = st.need_linearize && st.iter0;
                if (st.eval_failed) st.solve_failed = 2;  // only reachable at iteration zero
                else if (st.n_f == 0) {                   // nothing to move: a zero step, invalid by its model change
                    for (int i = 0; i < 7; ++i) s_pose[1 - cur][i] = s_pose[cur][i];
                    st.f_model = 0; st.f_step_sq = 0; st.f_xnorm_sq = 0; st.f_gmax = 0;
                } else {
                    double* L = s_L, *fdiag = s_fd, *g = s_g, *lam = s_lam, *y = s_y;
                    for (int i = 0; i < 36; ++i) L[i] = 0.0;
                    for (int q = 0; q < 21; ++q) {
                        int a = 0, rem = q;
                        while (rem >= 6 - a) { rem -= 6 - a; ++a; }
                        const int b = a + rem;  // a <= b: lower entry (b, a)
                        L[6 * b + a] = s_B[q];
                        if (a == b) fdiag[a] = s_B[q];
                    }
                    for (int c = 0; c < 6; ++c) g[c] = s_B[21 + c];
                    if (speed) {  // SpeedRegularizationVector2, TrivialLoss * weight: rho' = w
                        double r[3], J[18];
                        speed_regulariser(s_pose[cur], F.speed_T_origin_before, F.speed_v_before, F.speed_dt, r, J);
                        if (eval_cost) st.x_cost += 0.5 * F.speed_weight * (r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
                        const double wgt = F.speed_weight;
                        for (int a = 0; a < 6; ++a) {
                            for (int b = 0; b <= a; ++b) L[6 * a + b] += wgt * (J[a] * J[b] + J[6 + a] * J[6 + b] + J[12 + a] * J[12 + b]);
                            fdiag[a] += wgt * (J[a] * J[a] + J[6 + a] * J[6 + a] + J[12 + a] * J[12 + a]);
                            g[a] += wgt * (J[a] * r[0] + J[6 + a] * r[1] + J[12 + a] * r[2]);
                        }
                    }
                    // Jacobi scaling (fixed at iteration zero of the solve) and the LM diagonal
                    for (int c = 0; c < 6; ++c) {
                        double s;
                        if (st.iter0) { s = 1.0 / (1.0 + sqrt(fdiag[c])); s_scale[c] = s; }
                        else s = s_scale[c];
                        const double s2 = s * s;
                        lam[c] = fmin(fmax(fdiag[c] * s2, sp.min_lm_diagonal), sp.max_lm_diagonal) / (st.radius * s2);
                        L[7 * c] += lam[c];
                    }
                    // Cholesky L L^T of the damped system (in place, lower), then L y = g and L^T (-d) = y
                    bool ok = true;
                    for (int j = 0; j < 6 && ok; ++j) {
                        double djj = L[7 * j];
                        for (int k = 0; k < j; ++k) djj -= L[6 * j + k] * L[6 * j + k];
                        if (!(djj > 0.0) || !isfinite(djj)) { ok = false; break; }
                        const double ljj = sqrt(djj), inv = 1.0 / ljj;
                        L[7 * j] = ljj;
                        for (int i = j + 1; i < 6; ++i) {
                            double v = L[6 * i + j];
                            for (int k = 0; k < j; ++k) v -= L[6 * i + k] * L[6 * j + k];
                            L[6 * i + j] = v * inv;
                        }
                    }
                    if (!ok) st.solve_failed = 1;
                    else {
                        for (int i = 0; i < 6; ++i) {
                            double v = g[i];
                            for (int k = 0; k < i; ++k) v -= L[6 * i + k] * y[k];
                            y[i] = v / L[7 * i];
                        }
                        for (int i = 5; i >= 0; --i) {
                            double v = y[i];
                            for (int k = i + 1; k < 6; ++k) v -= L[6 * k + i] * y[k];
                            y[i] = v / L[7 * i];
                        }
                        double model = 0.0, d[6], gneg[6], out[7];
                        bool bad = false;
                        for (int c = 0; c < 6; ++c) {
                            d[c] = -y[c];
                            if (!isfinite(d[c])) bad = true;
                            model += -g[c] * d[c] + lam[c] * d[c] * d[c];
                            gneg[c] = -g[c];
                        }
                        const double* p = s_pose[cur];
                        double step_sq = 0.0, xn_sq = 0.0, gmax = 0.0;
                        pose_plus(p, d, out);
                        for (int i = 0; i < 7; ++i) {
                            s_pose[1 - cur][i] = out[i];
                            const double e = out[i] - p[i];
                            step_sq += e * e; xn_sq += p[i] * p[i];
                        }
                        pose_plus(p, gneg, out);
                        for (int i = 0; i < 7; ++i) gmax = fmax(gmax, fabs(out[i] - p[i]));
                        st.f_model = model; st.f_step_sq = step_sq; st.f_xnorm_sq = xn_sq; st.f_gmax = gmax;
                        if (bad) st.solve_failed = 1;
                    }
                }
            }
            __syncthreads();
            // ---- the candidate's cost (only a valid step reads it) ----
            const bool need_cand = s_st.solve_failed == 0 && s_st.n_f > 0;
            bool cand_failed = false;
            if (need_cand) {
                stage_rt(s_pose[1 - cur], s_rt);
                cand_failed = evaluate(std::false_type{});
            }
            if (tid == 0) {
                WinState& st = s_st;
                if (need_cand) {
                    double c = 0.0;
                    for (int w = 0; w < kMotionWarps; ++w) c += s_red[w][0];
                    s_sum = c;
                    if (cand_failed) st.eval_failed = 1;
                }
                const double* P = s_pose[1 - cur];
                const double* cand_obs = &s_sum;
                lm_step(st, log, sp, true, true, 0.0, 0.0, 0.0, 0.0, [&F, P, cand_obs, speed]() {
                    double cand = *cand_obs;
                    if (speed) {
                        double r[3];
                        speed_regulariser(P, F.speed_T_origin_before, F.speed_v_before, F.speed_dt, r, nullptr);
                        cand += 0.5 * F.speed_weight * (r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
                    }
                    return cand;
                });
            }
            continue;
        }

        // ---- PH_TRIM: per-landmark maximum raw residual per group (k_trim_eval), quantile select (k_trim_select) ----
        stage_rt(s_pose[s_st.cur], s_rt);
        for (int r = tid; r < n_runs; r += kMotionThreads) {
            double m_d = -1.0, m_r = -1.0;
            if (act[r]) {
                const double4 q4 = *reinterpret_cast<const double4*>(pw + 4 * r);
                const double p[3] = {q4.x, q4.y, q4.z};
                for (int o = rs[r]; o < rs[r + 1]; ++o) {
                    const int c = cams ? cams[o] : 0;
                    double res[3], m[9], a[3], raw[2], hr;
                    if (!eval_factored<double, false, false>(s_rt, s_cam + kCamStride * c, p, (double)mu[o], (double)mv[o],
                                                             (double)md[o], q4.w, b_repr, b_depth, res, m, a, hr, raw))
                        continue;
                    m_r = fmax(m_r, raw[0]);
                    m_d = fmax(m_d, raw[1]);
                }
            }
            tv[r] = m_d;
            tv_r[r] = m_r;
            rej[r] = 0;
        }
        __syncthreads();
        auto oid = [](int j) { return j; };  // runs are in the caller's landmark order
        trim_select_group(s_trim, n_runs, sp.depth_quantile, sp.min_residual_groups, [tv](int j) { return tv[j]; }, oid, rej);
        trim_select_group(s_trim, n_runs, sp.reprojection_quantile, sp.min_residual_groups,
                          [tv_r](int j) { return tv_r[j]; }, oid, rej);
        // (no ground-plane group: a frame has no ground-plane residuals)
        for (int r = tid; r < n_runs; r += kMotionThreads)
            if (rej[r]) act[r] = 0;
        if (tid == 0) trim_advance(s_st);
    }

    // ---- results ----
    FrameRes& R = A.res[blockIdx.x];
    const WinState& st = s_st;
    if (tid < 7) R.pose[tid] = s_pose[st.cur][tid];
    if (tid == 0) {
        R.n_solves = st.n_solves; R.log_n = st.log_n; R.done = 1; R.pad = 0;
        for (int q = 0; q < 8; ++q) R.solves[q] = st.solves[q];
    }
    const int n_log = min(st.log_n, A.log_cap);
    for (int i = tid; i < n_log; i += kMotionThreads) A.res_log[(size_t)blockIdx.x * A.log_cap + i] = log[i];
    for (int r = tid; r < n_runs; r += kMotionThreads) A.res_rej[F.run_off + r] = act[r] ? 0 : 1;
}

void launch_adjust_pose(const MotionArgs& a, int n_frames, cudaStream_t s) {
    if (n_frames <= 0) return;
    k_adjust_pose<<<n_frames, kMotionThreads, 0, s>>>(a);
    LCHK("k_adjust_pose");
}

}  // namespace kba
