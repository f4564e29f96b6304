// kba_kernels.cu -- sm_90a kernels of the window solver.  One LM "pass" over a batch of windows is, for small windows
// (every window <= kFusedMaxRows reduced rows: BASELINE configs 1-3),
//   k_solve_begin [-> k_gp_eval<true>] -> k_linearize (kba_linearize.cuh: evaluation + landmark blocks + V rows, Jacobian in registers)
//   -> k_pose_hessian -> k_schur_fused (kba_schur_fused.cuh: warp-specialised FP64 tensor-core SYRK over bulk-copied V columns)
//   [-> k_sred_reduce] -> k_reduced_solve<tiled> -> k_backsub_v -> k_eval_obs<false> (candidate cost) [-> k_gp_eval<false>]
//   -> k_lm_update -> k_trim_eval -> k_trim_select
// and for large windows (BASELINE config 5), the FP32 mode or rigs with several observations per landmark and keyframe
//   k_panel_zero -> k_solve_begin -> k_eval_obs<true> (materialised residual/Jacobian, HBM streaming) [-> k_gp_eval<true>]
//   -> k_pose_hessian -> k_landmark_reduce -> k_obs_v | k_obs_v2 [-> k_gp_panel]   (kba_prep.cuh: landmark blocks, V panels)
//   -> k_schur_syrk | k_schur_fused (FP64 tensor-core SYRK) [-> k_sred_reduce]
//   -> k_reduced_solve (or, for large systems of small batches: stage 1, k_chol_diag/panel/trail per block, stage 2)
//   -> k_backsub -> k_eval_obs<false> [-> k_gp_eval<false>] -> k_lm_update -> k_trim_eval -> k_trim_select
// with k_shard_pack / k_shard_scalars / k_shard_trim_scatter and three NCCL all-reduces in between when one window is sharded over
// several GPUs (launch_pass).  Every kernel looks at the per-window state and returns immediately for windows that have nothing
// to do, so the host launches a fixed sequence without synchronising per iteration.
#include "kba_device.cuh"
#include "kba_kernels.h"
#include "kba_regularisers.cuh"
#include "kba_controller.cuh"
#include "kba_prep.cuh"
#include "kba_linearize.cuh"

#include <cfloat>
#include <cstdio>
#include <cstdlib>
#include <cmath>
#include <type_traits>

namespace kba {

// =====================================================================================================================
// solve begin: program layout (which parameter blocks are in the reduced program) + LM state reset
// =====================================================================================================================
// sharded window with ground points, before k_solve_begin: a keyframe's plane blocks are variable when an active ground point of
// ANY rank is attached to it (gp_kf_glob: k_shard_gp_gather; act_glob: the window-wide trimming decisions), so that every rank
// takes the layout of the plain solve of the whole window
__global__ void __launch_bounds__(256) k_shard_planes(BatchDev bd) {
    if (bd.state[0].phase != PH_SOLVE_BEGIN) return;
    const WinDesc& wd = bd.desc[0];
    for (int k = threadIdx.x; k < wd.n_kf; k += blockDim.x) bd.kf_gp_glob[k] = 0;
    __syncthreads();
    for (int j = threadIdx.x; j < bd.lm_total; j += blockDim.x) {
        const int kp = (int)bd.gp_kf_glob[j];
        if (kp > 0 && bd.act_glob[j]) bd.kf_gp_glob[kp - 1] = 1;  // benign race: every writer stores 1
    }
}

// 1024 threads: the layout tables of a solve's first pass are dependent-load chains per landmark / observation, and a trimmed
// solve begins three to four times
constexpr int kBeginThreads = 1024;
__global__ void __launch_bounds__(kBeginThreads) k_solve_begin(BatchDev bd) {
    const int w = blockIdx.x;
    const SolveParams& sp = bd.wsp[w];
    WinState& st = bd.state[w];
    if (st.phase != PH_SOLVE_BEGIN) return;
    const WinDesc wd = bd.desc[w];
    __shared__ int s_has[kMaxKf];
    __shared__ int s_plane[kMaxKf];  // keyframe's plane blocks are referenced by a ground-plane residual
    __shared__ int s_cnt[3];
    __shared__ int s_tile_chunk[513];
    for (int k = threadIdx.x; k < wd.n_kf; k += blockDim.x) { s_has[k] = 0; s_plane[k] = 0; }
    if (threadIdx.x < 3) s_cnt[threadIdx.x] = 0;
    __syncthreads();
    {
        int n_gp_act = 0;
        for (int gi = threadIdx.x; gi < wd.n_gp; gi += blockDim.x) {
            const size_t G = (size_t)wd.gp_off + gi;
            if (!bd.lm_active[wd.lm_off + bd.gp_lm[G]]) continue;
            s_has[bd.gp_kf[G]] = 1;
            s_plane[bd.gp_kf[G]] = 1;
            n_gp_act++;
        }
        atomicAdd(&s_cnt[2], n_gp_act);
    }
    const int* lm_ptr = bd.lm_ptr + wd.lm_off + w;
    int n_lm_in = 0, n_blocks = 0;
    for (int j = threadIdx.x; j < wd.n_lm; j += blockDim.x) {
        if (!bd.lm_active[wd.lm_off + j]) continue;
        const int o0 = lm_ptr[j], o1 = lm_ptr[j + 1];
        if (o1 > o0) n_lm_in++;
        for (int o = o0; o < o1; ++o) {
            s_has[bd.obs_kf[wd.obs_off + o]] = 1;  // benign race: every writer stores 1
            n_blocks += (bd.obs_d[wd.obs_off + o] > 0.0f) ? 2 : 1;
        }
    }
    atomicAdd(&s_cnt[0], n_lm_in);
    atomicAdd(&s_cnt[1], n_blocks);
    if (bd.sharded)  // another rank's landmarks may be the only ones seen from a keyframe: all free keyframes are variable
        for (int k = threadIdx.x; k < wd.n_kf; k += blockDim.x) {
            s_has[k] = 1;
            if (bd.shard_gp && bd.kf_gp_glob[k]) s_plane[k] = 1;  // ... and so may its ground points be (k_shard_planes)
        }
    __syncthreads();
    if (threadIdx.x == 0) {
        if (wd.scale_weight > 0) { s_has[wd.scale_kf0] = 1; s_has[wd.scale_kf1] = 1; }
        if (wd.speed_weight > 0) s_has[wd.speed_kf] = 1;
        if (wd.landmarks_fixed) s_cnt[0] = 0;  // landmark blocks are constant: none is in the program
        const bool chain = wd.plane_reg_weight > 0 && wd.n_kf > 1;  // adds pose, normal and distance blocks of every keyframe
        int n = 0, n_reg = 0;
        for (int k = 0; k < wd.n_kf; ++k) {
            const bool fixed = bd.kf_fixed[wd.kf_off + k];
            const bool var = (s_has[k] || chain) && !fixed;
            bd.off_pose[wd.kf_off + k] = var ? n : -1;
            if (var) n += 6;
            const bool pl = (s_plane[k] || chain) && !fixed;       // reference cpp:198-219: fixed keyframe -> plane constant
            bd.off_dir[wd.kf_off + k] = pl ? n : -1;
            if (pl) n += 3;
            const bool pd = pl && !wd.plane_dist_fixed;            // reference cpp:722-728
            bd.off_dist[wd.kf_off + k] = pd ? n : -1;
            if (pd) n += 1;
        }
        if (chain) n_reg = 3 * (wd.n_kf - 1) + wd.n_kf;
        st.n_f = n;
        st.nr = (n + 1 + 7) & ~7;
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
        s.num_landmarks = s_cnt[0];
        s.num_residual_blocks = s_cnt[1] + s_cnt[2] + n_reg + (wd.scale_weight > 0 ? 1 : 0) + (wd.speed_weight > 0 ? 1 : 0);
        st.t_solve_start = global_timer_ns();
        st.phase = PH_ITERATE;
    }
    __syncthreads();
    // per-observation row of the pose block in the reduced system (one load instead of a 4-deep dependent chain later)
    for (int o = threadIdx.x; o < wd.n_obs; o += blockDim.x) {
        const size_t oo = (size_t)wd.obs_off + o;
        const bool act = bd.lm_active[wd.lm_off + bd.obs_lm[oo]];
        bd.obs_row[oo] = act ? bd.off_pose[wd.kf_off + bd.obs_kf[oo]] : -1;
    }
    // 8-row tile range of the reduced system each landmark chunk touches (landmarks are sorted by first keyframe)
    for (int c = threadIdx.x; c < (bd.fused ? 0 : wd.n_chunks); c += blockDim.x) {
        int r0 = 1 << 30, r1 = -1;
        for (int k = bd.chunk_k0[wd.chunk_off + c]; k <= bd.chunk_k1[wd.chunk_off + c]; ++k) {
            const int off = bd.off_pose[wd.kf_off + k], od = bd.off_dir[wd.kf_off + k], oz = bd.off_dist[wd.kf_off + k];
            if (off >= 0) { r0 = min(r0, off); r1 = max(r1, off + 6); }
            if (od >= 0) { r0 = min(r0, od); r1 = max(r1, od + 3); }
            if (oz >= 0) { r0 = min(r0, oz); r1 = max(r1, oz + 1); }
        }
        bd.chunk_t0[wd.chunk_off + c] = (r1 < 0) ? 0 : r0 / 8;
        bd.chunk_t1[wd.chunk_off + c] = (r1 < 0) ? 0 : (r1 + 7) / 8;
    }
    // fused path: does a landmark's set of observations with variable poses form ONE run of consecutive reduced-system rows
    // (a track without gaps over free keyframes, one camera per keyframe)?  Then each of its three panel columns is one
    // contiguous segment and the Schur kernel fetches it with a single bulk copy (BatchDev::lm_run).  Fixed for the solve.
    if (bd.fused) {
        __syncthreads();  // obs_row is complete
        for (int j = threadIdx.x; j < wd.n_lm; j += blockDim.x) {
            const int o0 = lm_ptr[j], o1 = lm_ptr[j + 1];
            int n_start = 0, n_valid = 0, bad = 0, a = 0, row_a = 0, prev = -2;
            for (int o = o0; o < o1; ++o) {
                const size_t oo = (size_t)wd.obs_off + o;
                const int r = bd.obs_row[oo];
                if (r >= 0) {
                    ++n_valid;
                    if (prev < 0) { if (n_start++ == 0) { a = o - o0; row_a = r; } }
                    else if (r != prev + 6) bad = 1;
                    if (bd.obs_rank[oo] != 0) bad = 1;
                }
                prev = r;
            }
            int4 run = make_int4(0, 0, 0, 0);
            if (n_valid > 0) run = (bad || n_start != 1) ? make_int4(0, -1, 0, 0) : make_int4(a, n_valid, row_a, 0);
            bd.lm_run[wd.lm_off + j] = run;
        }
    }
    if (bd.fused) build_lin_tiles(bd, wd, st, w, s_tile_chunk);  // warp tiles of k_linearize over the active landmarks
    // fused path: 16-row-aligned and exact 8-row tile ranges and shared-memory panel rows of each 8-landmark group
    if (bd.fused) {
        const int trhs = st.n_f >> 3;
        for (int c = threadIdx.x; c < wd.n_groups; c += blockDim.x) {
            int r0 = 1 << 30, r1 = -1;
            for (int k = bd.grp_k0[wd.grp_off + c]; k <= bd.grp_k1[wd.grp_off + c]; ++k) {
                const int off = bd.off_pose[wd.kf_off + k], od = bd.off_dir[wd.kf_off + k], oz = bd.off_dist[wd.kf_off + k];
                if (off >= 0) { r0 = min(r0, off); r1 = max(r1, off + 6); }
                if (od >= 0) { r0 = min(r0, od); r1 = max(r1, od + 3); }
                if (oz >= 0) { r0 = min(r0, oz); r1 = max(r1, oz + 1); }
            }
            // range aligned to 16-row blocks (two tiles): every block of the range has both its tiles, the fused kernel then
            // needs no partial-block variants except for the right-hand-side tile
            const int t0 = (r1 < 0) ? 0 : (r0 / 16) * 2, t1 = (r1 < 0) ? 0 : ((r1 + 15) / 16) * 2;
            int rows = 0;  // rows of the group's shared-memory panel (the column stride is the constant kFMaxRs)
            if (t1 > t0) rows = 8 * (t1 - t0) + ((trhs >= t0 && trhs < t1) ? 0 : 8);
            // tiles of [t0, t1) outside [e0, e1) are zero in the panel: the kernel skips the products against them.  The
            // right-hand-side row, when it lies inside [t0, t1), is part of the panel too.
            int e0 = 0, e1 = 0;
            if (t1 > t0) {
                e0 = r0 / 8;
                e1 = (r1 + 7) / 8;
                if (trhs >= t0 && trhs < t1) e1 = max(e1, trhs + 1);
            }
            bd.grp_t0[wd.grp_off + c] = t0;
            bd.grp_t1[wd.grp_off + c] = t1;
            bd.grp_tiles[wd.grp_off + c] = t0 | t1 << 8 | e0 << 16 | e1 << 24;
            bd.grp_rs[wd.grp_off + c] = rows;
        }
    }
    if (!bd.fused) {  // layout of the dense V panels: per chunk 96 columns x rs rows (rs == 4 mod 16), column-major
        __syncthreads();
        if (threadIdx.x == 0) {
            const int trhs = st.n_f >> 3;
            int poff = 0;
            for (int c = 0; c < wd.n_chunks; ++c) {
                const int t0 = bd.chunk_t0[wd.chunk_off + c], t1 = bd.chunk_t1[wd.chunk_off + c];
                int rs = 0;
                if (t1 > t0) {
                    const int rows = 8 * (t1 - t0) + ((trhs >= t0 && trhs < t1) ? 0 : 8);
                    rs = ((rows - 4 + 15) / 16) * 16 + 4;
                }
                bd.chunk_rs[wd.chunk_off + c] = rs;
                bd.chunk_poff[wd.chunk_off + c] = poff;
                poff += 96 * rs;
            }
        }
    }
}

// zero the dense V panels of windows that are about to start a solve (the sparsity pattern is fixed within a solve:
// k_landmark_reduce / k_obs_v / k_gp_panel overwrite every structurally non-zero entry in each pass)
__global__ void __launch_bounds__(256) k_panel_zero(BatchDev bd) {
    const int w = blockIdx.y;
    if (bd.fused || bd.state[w].phase != PH_SOLVE_BEGIN || bd.desc[w].landmarks_fixed) return;
    double2* p = reinterpret_cast<double2*>(bd.vpanel + bd.desc[w].panel_off);
    const long long n2 = bd.panel_cap / 2;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n2; i += (long long)gridDim.x * blockDim.x)
        p[i] = make_double2(0.0, 0.0);
}

// =====================================================================================================================
// residual / Jacobian kernel: one thread per observation, landmark-major order, SoA in / SoA out.
//   kJac = true : linearisation at x -> residual (3), J_pose (3x6), J_landmark (3x3) per observation + cost partials
//   kJac = false: cost only, at the candidate point
// Algorithmic HBM bytes per observation (FP64, with depth row): 20 read + 240 written (DESIGN.md).
// =====================================================================================================================
template <bool kJac, int kMinBlocks, typename TLin, bool kJl = true>
__global__ void __launch_bounds__(256, kMinBlocks) k_eval_obs(BatchDev bd, int tiles) {
    // A CTA walks `tiles` consecutive 256-observation tiles of one window with a two-deep software pipeline: while tile
    // t is evaluated, the measurement / landmark loads of tile t+1 and the landmark-index load of tile t+2 are in
    // flight, so the dependent chain index -> landmark is hidden; the keyframe poses are staged once per CTA.
    const int w = blockIdx.y;
    WinState& st = bd.state[w];
    const WinDesc& wd = bd.desc[w];
    const int n_obs = wd.n_obs, obs_off = wd.obs_off, lm_off = wd.lm_off;
    if (st.phase != PH_ITERATE) return;
    if (kJac && !st.need_linearize) return;
    if (!kJac && st.solve_failed) return;
    __shared__ __align__(16) double s_pose[kMaxKf * kPoseStride];
    __shared__ __align__(16) double s_cam[kMaxCam * kCamStride];
    __shared__ __align__(8) uint64_t s_bar;
    __shared__ double s_red[8];
    __shared__ int s_cnt[8];
    __shared__ double s_b[2];  // the window's squared Cauchy scales (reprojection, depth), published by the staging barrier
    constexpr bool kF32 = sizeof(TLin) == 4;  // FP32 evaluation + storage of the linearisation (precision 1)
    __shared__ float s_pose_f[kF32 ? kMaxKf * kPoseStride : 1];
    __shared__ float s_cam_f[kF32 ? kMaxCam * kCamStride : 1];
    __shared__ float s_arm_f[kF32 ? kMaxKf * 3 : 1];  // R_k c: the rotation columns' lever arm at the anchor c
    double anc[3] = {0.0, 0.0, 0.0};
    const int buf = kJac ? st.cur : 1 - st.cur;
    const double* __restrict__ lm_buf = bd.lm[buf];
    const int i0 = blockIdx.x * tiles * 256 + threadIdx.x;
    // stage A: landmark index of a tile; stage B: everything else the evaluation reads
    int idx_b = (i0 < n_obs) ? bd.obs_lm[(size_t)obs_off + i0] : -1;                  // tile 0
    int idx_a = (tiles > 1 && i0 + 256 < n_obs) ? bd.obs_lm[(size_t)obs_off + i0 + 256] : -1;  // tile 1
    int L = -1, kfi = 0, cami = 0, row = -1;  // loaded values are not touched before their tile is evaluated; row: reduced-system row of the pose block (k_solve_begin), < 0: constant keyframe
    float u = 0.f, v = 0.f, d = 0.f;
    double p0 = 0, p1 = 0, p2 = 0, wgt = 0;
    unsigned char act = 0;
    if (idx_b >= 0) {
        const size_t o = (size_t)obs_off + i0;
        L = lm_off + idx_b;
        kfi = bd.obs_kf[o]; cami = bd.obs_cam[o];
        if (kJac) row = bd.obs_row[o];
        u = bd.obs_u[o]; v = bd.obs_v[o]; d = bd.obs_d[o];
        p0 = lm_buf[3 * (size_t)L]; p1 = lm_buf[3 * (size_t)L + 1]; p2 = lm_buf[3 * (size_t)L + 2];
        wgt = bd.lm_weight[L];
        act = bd.lm_active[L];
    }
    if (threadIdx.x == 0) {
        const SolveParams& sp = bd.wsp[w];
        s_b[0] = sp.reprojection_thres * sp.reprojection_thres; s_b[1] = sp.depth_thres * sp.depth_thres;
    }
    stage_window_bulk(wd, bd.rt[buf], bd.cam, s_pose, s_cam, &s_bar);  // poses (R | t) and cameras: two bulk copies
    if (kF32) {
        // FP32 blocks are formed relative to an anchor c, keyframe 0's centre -R_0^T t_0 (FP64) on a 64 m grid: a window
        // kilometres from the origin would otherwise round R p and t, each of the size of that distance, before they cancel
        // to a camera-frame point of a few metres.  p - c and t_k + R_k c are formed in FP64, so x = R p + t is unchanged in
        // exact arithmetic.  On the grid, a window whose keyframe 0 is within 32 m of the origin has c = 0 and the blocks it
        // had without the anchor, bit for bit; any other is evaluated as if it were that close.
        constexpr double kGrid = 64.0;
#pragma unroll
        for (int j = 0; j < 3; ++j)
            anc[j] = kGrid * rint(-(s_pose[j] * s_pose[9] + s_pose[3 + j] * s_pose[10] + s_pose[6 + j] * s_pose[11]) / kGrid);
        for (int i = threadIdx.x; i < wd.n_kf * kPoseStride; i += blockDim.x) {
            const int k = i / kPoseStride, e = i - k * kPoseStride;
            if (e < 9) {
                s_pose_f[i] = (float)s_pose[i];
            } else {
                const double* P = s_pose + kPoseStride * k + 3 * (e - 9);
                const double rc = P[0] * anc[0] + P[1] * anc[1] + P[2] * anc[2];
                s_pose_f[i] = (float)(s_pose[i] + rc);
                s_arm_f[3 * k + e - 9] = (float)rc;
            }
        }
        for (int i = threadIdx.x; i < wd.n_cam * kCamStride; i += blockDim.x) s_cam_f[i] = (float)s_cam[i];
        __syncthreads();
    }
    double cost = 0.0;
    int done = 0;
#pragma unroll 1
    for (int t = 0; t < tiles; ++t) {
        // issue the next tile's loads (stage B of t+1, stage A of t+2) before touching this tile's values
        const int i_n = i0 + (t + 1) * 256;
        int Ln = -1, kfn = 0, camn = 0, rown = -1;
        float un = 0.f, vn = 0.f, dn = 0.f;
        double q0 = 0, q1 = 0, q2 = 0, wn = 0;
        unsigned char actn = 0;
        if (idx_a >= 0) {
            const size_t o = (size_t)obs_off + i_n;
            Ln = lm_off + idx_a;
            kfn = bd.obs_kf[o]; camn = bd.obs_cam[o];
            if (kJac) rown = bd.obs_row[o];
            un = bd.obs_u[o]; vn = bd.obs_v[o]; dn = bd.obs_d[o];
            q0 = lm_buf[3 * (size_t)Ln]; q1 = lm_buf[3 * (size_t)Ln + 1]; q2 = lm_buf[3 * (size_t)Ln + 2];
            wn = bd.lm_weight[Ln];
            actn = bd.lm_active[Ln];
        }
        idx_a = (t + 2 < tiles && i_n + 256 < n_obs) ? bd.obs_lm[(size_t)obs_off + i_n + 256] : -1;
        if (L >= 0 && act) {
            const size_t o = (size_t)obs_off + i0 + t * 256;
            const int k = kfi, c = cami;
            const double p[3] = {p0, p1, p2};
            double hr = 0.0;
            bool ok;
            if (kJac && kF32) {
                // FP32 linearisation; the cost at x keeps the FP64 evaluation so that the step acceptance test compares
                // like with like (the candidate cost pass is FP64)
                double r[3], raw[2];
                ok = eval_observation<double, false>(
                    s_pose + kPoseStride * k, s_cam + kCamStride * c, p, (double)u, (double)v, (double)d, wgt,
                    s_b[0], s_b[1], r, nullptr, nullptr, hr, raw);
                if (ok) {
                    const float pf[3] = {(float)(p0 - anc[0]), (float)(p1 - anc[1]), (float)(p2 - anc[2])};
                    float hrf;
                    float* resf = reinterpret_cast<float*>(bd.res) + o;
                    float* jpf = reinterpret_cast<float*>(bd.jp) + o;
                    float* jlf = reinterpret_cast<float*>(bd.jl) + o;
                    eval_observation_store<float, kJl, true>(
                        s_pose_f + kPoseStride * k, s_cam_f + kCamStride * c, pf, u, v, d, (float)wgt,
                        (float)s_b[0], (float)s_b[1],
                        resf, jpf, jlf, (size_t)bd.tot_obs, row >= 0 || !kJl, hrf, s_arm_f + 3 * k);
                }
            } else if (kJac) {  // rows are stored to their SoA slots as they are formed
                ok = eval_observation_store<double, kJl>(
                    s_pose + kPoseStride * k, s_cam + kCamStride * c, p, (double)u, (double)v, (double)d, wgt,
                    s_b[0], s_b[1], bd.res + o, bd.jp + o,
                    bd.jl + o, (size_t)bd.tot_obs, row >= 0 || !kJl, hr);
            } else {
                double r[3], raw[2];
                ok = eval_observation<double, false>(
                    s_pose + kPoseStride * k, s_cam + kCamStride * c, p, (double)u, (double)v, (double)d, wgt,
                    s_b[0], s_b[1], r, nullptr, nullptr, hr, raw);
            }
            if (!ok) {
                st.eval_failed = 1;  // benign race
            } else {
                cost += hr;
                ++done;
            }
        }
        L = Ln; kfi = kfn; cami = camn; row = rown; u = un; v = vn; d = dn; p0 = q0; p1 = q1; p2 = q2; wgt = wn; act = actn;
    }
    cost = warp_sum(cost);
    if (kJac) done = __reduce_add_sync(0xffffffffu, done);
    if ((threadIdx.x & 31) == 0) { s_red[threadIdx.x >> 5] = cost; s_cnt[threadIdx.x >> 5] = done; }
    __syncthreads();
    if (threadIdx.x < tiles) {  // slot blockIdx.x * tiles carries the CTA's sum, its other slots are zero
        double s = 0.0;
        if (threadIdx.x == 0)
            for (int q = 0; q < 8; ++q) s += s_red[q];
        const int slot = blockIdx.x * tiles + threadIdx.x;
        if (slot < bd.cost_parts) (kJac ? bd.cost_part_x : bd.cost_part_c)[(size_t)w * bd.cost_parts + slot] = s;
    }
    if (kJac && threadIdx.x == 0) {  // observation count for the roofline report (one atomic per CTA)
        int cnt = 0;
        for (int q = 0; q < 8; ++q) cnt += s_cnt[q];
        if (cnt) atomicAdd(bd.jac_obs, (unsigned long long)cnt);
    }
}

// 8 tiles per CTA; two CTAs per SM for the linearisation, four for the cost.  The cost slots a CTA writes follow the tile count.
constexpr int kEvalTiles = 8;
template <bool kJac>
static void launch_eval_obs(const BatchDev& bd, cudaStream_t s) {
    const dim3 g((bd.max_obs + 256 * kEvalTiles - 1) / (256 * kEvalTiles), bd.n_win);
    if (!kJac) { k_eval_obs<false, 4, double><<<g, 256, 0, s>>>(bd, kEvalTiles); return; }
    // fused path (kJl = false): J_l is not materialised, its consumers form it as (translation columns of J_p) R
    if (bd.precision == 1) {
        if (bd.fused) k_eval_obs<true, 2, float, false><<<g, 256, 0, s>>>(bd, kEvalTiles);
        else k_eval_obs<true, 2, float, true><<<g, 256, 0, s>>>(bd, kEvalTiles);
    } else {
        if (bd.fused) k_eval_obs<true, 2, double, false><<<g, 256, 0, s>>>(bd, kEvalTiles);
        else k_eval_obs<true, 2, double, true><<<g, 256, 0, s>>>(bd, kEvalTiles);
    }
    LCHK("k_eval_obs");
}

// =====================================================================================================================
// ground-plane height residuals r = n . (R p + t) + dist with ScaledLoss(HuberLoss(0.1), w) (reference
// cost_functors_ceres.hpp:355-392, bundle_adjuster_keyframes.cpp:517-562).  One CTA per window (a few hundred blocks).
//   kJac: robustified residual + J_f (pose 6 | plane normal 3, local | distance 1) + J_l (3) -> gp_lin, cost at x
//   else: cost at the candidate
// =====================================================================================================================
template <bool kJac>
__global__ void __launch_bounds__(256) k_gp_eval(BatchDev bd) {
    const int w = blockIdx.x;
    const WinState& st = bd.state[w];
    if (st.phase != PH_ITERATE) return;
    if (kJac && !st.need_linearize) return;
    if (!kJac && st.solve_failed) return;
    const WinDesc& wd = bd.desc[w];
    if (wd.n_gp == 0) return;
    __shared__ double s_red[8];
    const int buf = kJac ? st.cur : 1 - st.cur;
    const size_t TG = (size_t)bd.tot_gp;
    double cost = 0.0;
    for (int gi = threadIdx.x; gi < wd.n_gp; gi += blockDim.x) {
        const size_t G = (size_t)wd.gp_off + gi;
        const int L = wd.lm_off + bd.gp_lm[G];
        if (!bd.lm_active[L]) continue;
        const int k = bd.gp_kf[G];
        const double* ps = bd.pose[buf] + 7 * (size_t)(wd.kf_off + k);
        const double* pl = bd.plane[buf] + 4 * (size_t)(wd.kf_off + k);
        const double* p = bd.lm[buf] + 3 * (size_t)L;
        double R[9], a[3], px[3];
        const double r = gp_height(ps, pl, p, R, a, px);
        const double n[3] = {pl[0], pl[1], pl[2]};
        const double wt = bd.gp_weight[G];
        double rho, rho1;
        gp_huber(r * r, bd.wsp[w].gp_huber, rho, rho1);
        cost += 0.5 * wt * rho;
        if (kJac) {
            const double sq = sqrt(wt * rho1);
            double* o = bd.gp_lin + G;
            o[0] = sq * r;
            o[1 * TG] = sq * -2.0 * (n[1] * a[2] - n[2] * a[1]);
            o[2 * TG] = sq * -2.0 * (n[2] * a[0] - n[0] * a[2]);
            o[3 * TG] = sq * -2.0 * (n[0] * a[1] - n[1] * a[0]);
            o[4 * TG] = sq * n[0]; o[5 * TG] = sq * n[1]; o[6 * TG] = sq * n[2];
            const double nn = n[0] * n[0] + n[1] * n[1] + n[2] * n[2], inv = 1.0 / sqrt(nn);
            const double npx = (n[0] * px[0] + n[1] * px[1] + n[2] * px[2]) / nn;
            o[7 * TG] = sq * (px[0] - n[0] * npx) * inv;
            o[8 * TG] = sq * (px[1] - n[1] * npx) * inv;
            o[9 * TG] = sq * (px[2] - n[2] * npx) * inv;
            o[10 * TG] = sq;
            o[11 * TG] = sq * (n[0] * R[0] + n[1] * R[3] + n[2] * R[6]);
            o[12 * TG] = sq * (n[0] * R[1] + n[1] * R[4] + n[2] * R[7]);
            o[13 * TG] = sq * (n[0] * R[2] + n[1] * R[5] + n[2] * R[8]);
        }
    }
    cost = warp_sum(cost);
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = cost;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int q = 0; q < 8; ++q) s += s_red[q];
        (kJac ? bd.gp_cost_x : bd.gp_cost_c)[w] = s;
    }
}
template __global__ void k_gp_eval<true>(BatchDev);
template __global__ void k_gp_eval<false>(BatchDev);

// per-keyframe ground-plane Gauss-Newton block after k_gp_eval<true>: the 55 lower-packed entries of the 10 x 10 (pose | normal |
// distance) block and the 10 gradient entries, summed over the keyframe's active gp residuals in index order.  One warp per
// keyframe, eight keyframes per CTA.  A separate array (not the reduced solve's own loop) so that a sharded window can exchange it.
__global__ void __launch_bounds__(256) k_gp_blocks(BatchDev bd) {
    const int w = blockIdx.y;
    const WinState& st = bd.state[w];
    if (st.phase != PH_ITERATE || !st.need_linearize) return;
    const WinDesc& wd = bd.desc[w];
    const int k = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (wd.n_gp == 0 || k >= wd.n_kf) return;
    const size_t TG = (size_t)bd.tot_gp;
    double acc[3] = {0.0, 0.0, 0.0};
    int ea[3], eb[3];
#pragma unroll
    for (int s = 0; s < 3; ++s) {
        const int e = lane + 32 * s;
        int a = 0, b = 0;
        if (e < 55) { while ((a + 1) * (a + 2) / 2 <= e) ++a; b = e - a * (a + 1) / 2; }
        else if (e < 65) { a = e - 55; b = -1; }
        else { a = -1; b = -1; }
        ea[s] = a; eb[s] = b;
    }
    for (int gi = 0; gi < wd.n_gp; ++gi) {
        const size_t G = (size_t)wd.gp_off + gi;
        if (bd.gp_kf[G] != k || !bd.lm_active[wd.lm_off + bd.gp_lm[G]]) continue;
#pragma unroll
        for (int s = 0; s < 3; ++s) {
            if (ea[s] < 0) continue;
            const double va = bd.gp_lin[(1 + ea[s]) * TG + G];
            const double vb = (eb[s] >= 0) ? bd.gp_lin[(1 + eb[s]) * TG + G] : bd.gp_lin[G];
            acc[s] += va * vb;
        }
    }
#pragma unroll
    for (int s = 0; s < 3; ++s)
        if (ea[s] >= 0) bd.gp_kfb[(size_t)(wd.kf_off + k) * 65 + lane + 32 * s] = acc[s];
}

// =====================================================================================================================
// pose-side Gauss-Newton blocks: one CTA per (keyframe, window) walks the keyframe-major copy of the observations,
// re-evaluates the Jacobian rows (cheaper than gathering the materialised J_pose across sectors) and reduces
// B_k = sum J_p^T J_p (21 unique) and g_k = sum J_p^T r (6) with a fixed-shape tree -> deterministic, no atomics.
// =====================================================================================================================
__global__ void __launch_bounds__(256, 2) k_pose_hessian(BatchDev bd) {
    const int w = blockIdx.y, k = blockIdx.x;
    const WinState& st = bd.state[w];
    if (st.phase != PH_ITERATE || !st.need_linearize) return;
    const WinDesc& wd = bd.desc[w];
    if (k >= wd.n_kf || bd.off_pose[wd.kf_off + k] < 0) return;
    __shared__ double s_pose[kPoseStride];
    __shared__ double s_cam[kMaxCam * kCamStride];
    __shared__ double s_red[8][27];
    // per thread: the sums of M = m^T m (6) and m^T r (3).  In registers, next to the 18 other sums and the prefetched loads,
    // they would be spilled at 128 registers; every observation adds to them once
    __shared__ double s_acc[9][256];
    __shared__ long long s_ob;                              // the window's first observation, its landmark offset, the end of
    __shared__ int s_lm_off, s_e1;                          // this keyframe's observations: re-read in every iteration (below)
    __shared__ double s_b[2];                               // the window's squared Cauchy scales (reprojection, depth), likewise
    if (threadIdx.x == 0) {
        s_ob = wd.obs_off; s_lm_off = wd.lm_off; s_e1 = bd.kf_ptr[wd.kf_off + w + k + 1];
        const SolveParams& sp = bd.wsp[w];
        s_b[0] = sp.reprojection_thres * sp.reprojection_thres; s_b[1] = sp.depth_thres * sp.depth_thres;
        const double* p = bd.pose[st.cur] + 7 * (size_t)(wd.kf_off + k);
        double R[9];
        quat_to_rot<double>(p, R);
        for (int i = 0; i < 9; ++i) s_pose[i] = R[i];
        s_pose[9] = p[4]; s_pose[10] = p[5]; s_pose[11] = p[6];
    }
    for (int i = threadIdx.x; i < wd.n_cam * kCamStride; i += blockDim.x) s_cam[i] = bd.cam[(size_t)wd.cam_off * kCamStride + i];
    __syncthreads();
    // outputs 0..14 (the rotation rows of B_k) and 21..23 (K^T h) in registers: acc[0..17]; 15..20 and 24..26 in s_acc
    double acc[18];
#pragma unroll
    for (int q = 0; q < 18; ++q) acc[q] = 0.0;
#pragma unroll
    for (int q = 0; q < 9; ++q) s_acc[q][threadIdx.x] = 0.0;
    const int* kp = bd.kf_ptr + wd.kf_off + w;
    const int e0 = kp[k], e1 = kp[k + 1];
    // two-deep software pipeline like k_eval_obs: the landmark index of iteration i+2 and the measurement / landmark
    // loads of iteration i+1 are in flight while iteration i is evaluated; loaded values are not touched before use
    const double* __restrict__ lm_buf = bd.lm[st.cur];
    const size_t ob = (size_t)wd.obs_off;
    int e = e0 + threadIdx.x;
    int idx_b = (e < e1) ? bd.pm_lm[ob + e] : -1;
    int idx_a = (e + (int)blockDim.x < e1) ? bd.pm_lm[ob + e + blockDim.x] : -1;
    int L = -1, cam = 0;
    float u = 0.f, v = 0.f, d = 0.f;
    double p0 = 0, p1 = 0, p2 = 0, wgt = 0;
    unsigned char act = 0;
    if (idx_b >= 0) {
        L = wd.lm_off + idx_b;
        cam = bd.pm_cam[ob + e]; u = bd.pm_u[ob + e]; v = bd.pm_v[ob + e]; d = bd.pm_d[ob + e];
        p0 = lm_buf[3 * (size_t)L]; p1 = lm_buf[3 * (size_t)L + 1]; p2 = lm_buf[3 * (size_t)L + 2];
        wgt = bd.lm_weight[L]; act = bd.lm_active[L];
    }
#pragma unroll 1
    for (; e < s_e1; e += blockDim.x) {
        // the staged pose and the window's offsets are read from shared memory in every iteration: hoisted out of the loop,
        // they would be spilled
        asm volatile("" ::: "memory");
        const size_t obs0 = (size_t)s_ob;
        const int e_end = s_e1, lm0 = s_lm_off;
        const int en = e + blockDim.x;
        int Ln = -1, camn = 0;
        float un = 0.f, vn = 0.f, dn = 0.f;
        double q0 = 0, q1 = 0, q2 = 0, wn = 0;
        unsigned char actn = 0;
        if (idx_a >= 0) {
            Ln = lm0 + idx_a;
            camn = bd.pm_cam[obs0 + en]; un = bd.pm_u[obs0 + en]; vn = bd.pm_v[obs0 + en]; dn = bd.pm_d[obs0 + en];
            q0 = lm_buf[3 * (size_t)Ln]; q1 = lm_buf[3 * (size_t)Ln + 1]; q2 = lm_buf[3 * (size_t)Ln + 2];
            wn = bd.lm_weight[Ln]; actn = bd.lm_active[Ln];
        }
        idx_a = (en + (int)blockDim.x < e_end) ? bd.pm_lm[obs0 + en + blockDim.x] : -1;
        if (act) {
            const double p[3] = {p0, p1, p2};
            double r[3], m[9], a[3], raw[2], hr;
            if (eval_factored<double, true, false>(s_pose, s_cam + kCamStride * cam, p, (double)u, (double)v, (double)d,
                                                   wgt, s_b[0], s_b[1], r, m, a, hr, raw)) {
                // J_p = m [K | I] with K = -2 [a]x (kba_device.cuh: eval_factored), so with M = m^T m and h = m^T r
                //   J_p^T J_p = [K^T M K, K^T M; M K, M],  J_p^T r = [K^T h; h],  K^T v = 2 a x v,  (row_i(P) K) = 2 a x row_i(P)
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
            }  // an evaluation failure is flagged by k_eval_obs
        }
        L = Ln; cam = camn; u = un; v = vn; d = dn; p0 = q0; p1 = q1; p2 = q2; wgt = wn; act = actn;
    }
#pragma unroll
    for (int q = 0; q < 27; ++q) {
        const double t = q < 15 ? acc[q] : q < 21 ? s_acc[q - 15][threadIdx.x] : q < 24 ? acc[q - 6] : s_acc[q - 18][threadIdx.x];
        const double v = warp_sum(t);
        if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5][q] = v;
    }
    __syncthreads();
    if (threadIdx.x < 27) {
        double s = 0.0;
        for (int q = 0; q < 8; ++q) s += s_red[q][threadIdx.x];
        bd.bkf[(size_t)(wd.kf_off + k) * 27 + threadIdx.x] = s;
    }
}

// =====================================================================================================================
// Schur complement accumulation as a dense SYRK on the FP64 tensor cores:
//   Sred = sum_j V_j V_j^T   with V_j the (n_f + 1) x 3 column block of landmark j (rows = pose rows of its
//   observations, plus the right-hand-side row z_j^T).  CTA = 64x64 output block x a range of landmark chunks;
//   the V panel of a chunk (32 landmarks = 96 columns) is scattered into shared memory, then mma.sync m8n8k4 f64.
// =====================================================================================================================
constexpr int kLC = 32;            // landmarks per chunk
constexpr int kKC = 3 * kLC;       // panel columns per chunk

// reduced-system row of component r (0..5 pose, 6..8 plane normal, 9 plane distance) of keyframe k, -1 if constant
__device__ __forceinline__ int gp_row(const BatchDev& bd, const WinDesc& wd, int k, int r) {
    if (r < 6) { const int o = bd.off_pose[wd.kf_off + k]; return o < 0 ? -1 : o + r; }
    if (r < 9) { const int o = bd.off_dir[wd.kf_off + k]; return o < 0 ? -1 : o + r - 6; }
    return bd.off_dist[wd.kf_off + k];
}

__device__ __forceinline__ void dmma(double& c0, double& c1, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
                 : "+d"(c0), "+d"(c1)
                 : "d"(a), "d"(b));
}

constexpr int kGS = 64 + 4;  // row stride of the column-major 64-row panel slices (== 4 mod 16: conflict-free fragments)

__global__ void __launch_bounds__(256, 2) k_schur_syrk(BatchDev bd) {
    // Generic kernel for reduced systems of more than 184 rows: CTA = one 64x64 block (bi >= bj) of Sred x a range of
    // landmark chunks.  The two 64-row slices of a chunk's dense V panel are copied (coalesced, zeros where the chunk has
    // no rows) into shared memory, column-major like the panel itself; chunks that do not touch both row blocks are
    // skipped -- landmarks are sorted by first keyframe, so that is most of them.
    const int w = blockIdx.z;
    const WinState& st = bd.state[w];
    if (st.phase != PH_ITERATE || st.solve_failed) return;
    const WinDesc& wd = bd.desc[w];
    if (wd.landmarks_fixed) return;
    int bi = 0, rem = blockIdx.x;
    while (rem > bi) { rem -= bi + 1; ++bi; }
    const int bj = rem;
    const int nrows = st.n_f + 1;  // pose rows + rhs row
    if (bi * 64 >= nrows) return;
    const bool diag = (bi == bj);
    extern __shared__ double smem[];
    double* pa = smem;                        // [96][kGS]
    double* pb = diag ? pa : smem + kKC * kGS;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double acc[8][2];
#pragma unroll
    for (int t = 0; t < 8; ++t) acc[t][0] = acc[t][1] = 0.0;
    const int trhs = st.n_f >> 3;
    const bool a_rhs = trhs >= 8 * bi && trhs < 8 * bi + 8, b_rhs = trhs >= 8 * bj && trhs < 8 * bj + 8;
    const double* pbase = bd.vpanel + wd.panel_off;
    // chunks are dealt round-robin to the p_split CTAs of a block pair: the chunks that touch a given pair are
    // neighbours in the sorted order, contiguous ranges would leave them all with one CTA
    for (int ch = blockIdx.y; ch < wd.n_chunks; ch += bd.p_split) {
        const int t0 = bd.chunk_t0[wd.chunk_off + ch], t1 = bd.chunk_t1[wd.chunk_off + ch];
        const int rs = bd.chunk_rs[wd.chunk_off + ch];
        if (rs == 0) continue;
        const bool a_hit = (8 * bi < t1 && 8 * bi + 8 > t0) || a_rhs, b_hit = (8 * bj < t1 && 8 * bj + 8 > t0) || b_rhs;
        if (!(a_hit && b_hit)) continue;
        const double* pan = pbase + bd.chunk_poff[wd.chunk_off + ch];
        const bool rhs_in = trhs >= t0 && trhs < t1;
        __syncthreads();  // previous chunk's MMA done before the slices are overwritten
        for (int idx = threadIdx.x; idx < (diag ? 1 : 2) * kKC * 64; idx += blockDim.x) {
            const int which = idx / (kKC * 64), e = idx - which * (kKC * 64);
            const int c = e >> 6, r = e & 63;
            const int g = 64 * (which ? bj : bi) + r, tile = g >> 3;
            double v = 0.0;
            if (tile >= t0 && tile < t1) v = pan[(size_t)c * rs + g - 8 * t0];
            else if (tile == trhs && !rhs_in) v = pan[(size_t)c * rs + 8 * (t1 - t0) + (g & 7)];
            (which ? pb : pa)[c * kGS + r] = v;
        }
        __syncthreads();
        const double* acol = pa + (lane & 3) * kGS + 8 * warp + (lane >> 2);
        const double* bcol = pb + (lane & 3) * kGS + (lane >> 2);
#pragma unroll 4
        for (int kk = 0; kk < kKC; kk += 4) {
            const double a = acol[kk * kGS];
#pragma unroll
            for (int t = 0; t < 8; ++t) {
                if (diag && t > warp) continue;
                dmma(acc[t][0], acc[t][1], a, bcol[kk * kGS + 8 * t]);
            }
        }
    }
    // store the partial block (row-major, leading dimension nr_cap)
    double* out = bd.sred + wd.s_off * (size_t)bd.p_split + (size_t)blockIdx.y * wd.nr_cap * wd.nr_cap;
    const int row = bi * 64 + 8 * warp + (lane >> 2);
#pragma unroll
    for (int t = 0; t < 8; ++t) {
        if (diag && t > warp) continue;
        const int col = bj * 64 + 8 * t + 2 * (lane & 3);
        out[(size_t)row * wd.nr_cap + col] = acc[t][0];
        out[(size_t)row * wd.nr_cap + col + 1] = acc[t][1];
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// Register-resident, TMA-fed kernel for reduced systems of up to kFusedMaxRows rows (<= 30 free keyframes): ONE CTA owns the whole
// lower triangle of Sred as accumulator tiles spread over 16 warps.  k_landmark_reduce / k_obs_v have already laid V out
// as dense column-major chunk panels in global memory (zeros included), so a panel half (48 columns x rs rows, <= 75 KB) arrives with ONE
// cp.async.bulk into a 2-stage shared-memory ring while the tensor-core loop works on the other stage: no scatter, no
// zero fill, no index loads in this kernel.  rs == 4 (mod 16) keeps the m8n8k4 fragment loads bank-conflict free.
// ---------------------------------------------------------------------------------------------------------------------
}  // namespace kba
#include "kba_schur_fused.cuh"
namespace kba {

constexpr int kHalfCols = 48;
constexpr int kStageDoubles = kHalfCols * kFMaxRs;

constexpr int kBlockSlots = 5;  // ceil(12*13/2 / 16) 16x16 blocks per warp for up to kFusedMaxRows reduced rows
// Which 16x16 blocks (linear index bi (bi + 1) / 2 + bj of the 12-row lower triangle) a warp owns.  The accumulators are
// registers, so the map is static; a chunk only touches the blocks inside its keyframe row range (a sub-square of the
// triangle plus the right-hand-side row), and with the plain cyclic map the busiest warp of such a chunk owns ~1.5x the
// mean number of active tiles while the per-stage barrier waits for it.  This table was searched offline (random swaps,
// objective = sum over chunks of the busiest warp's tile count, on config-2 windows plus generic sliding ranges):
// balance 0.65 -> 0.75 on windows that were not part of the search.
__constant__ signed char kSyrkBlockOfSlot[16][kBlockSlots] = {
    {8, 29, 44, 60, 76}, {2, 24, 35, 49, 55}, {14, 22, 47, 61, 77}, {15, 34, 38, 58, 69}, {5, 20, 28, 52, 56},
    {4, 19, 36, 63, 73}, {3, 17, 40, 62, 72}, {6, 30, 42, 59, 70},  {13, 33, 37, 54, 66}, {7, 18, 41, 45, 75},
    {1, 23, 39, 64, 71}, {10, 27, 31, 50, 67}, {0, 25, 51, 57, 68}, {11, 26, 46, 65, 74}, {9, 16, 43, 48, -1},
    {12, 21, 32, 53, -1}};

__global__ void __launch_bounds__(512, 1) k_schur_syrk_tma(BatchDev bd) {
    const int w = blockIdx.y;
    const WinState& st = bd.state[w];
    if (st.phase != PH_ITERATE || st.solve_failed) return;
    const WinDesc& wd = bd.desc[w];
    if (wd.landmarks_fixed) return;
    extern __shared__ __align__(128) double stage[];  // [2][kStageDoubles]
    __shared__ __align__(8) uint64_t full[2];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int nt = (st.n_f + 1 + 7) >> 3, trhs = st.n_f >> 3;
    if (tid == 0) {
        mbar_init(&full[0], 1);
        mbar_init(&full[1], 1);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    __syncthreads();
    // each warp owns kBlockSlots 16x16 blocks (2x2 m8n8k4 tiles) of the lower triangle: two A and two B fragments feed
    // four DMMAs, i.e. one shared-memory load per DMMA instead of two
    double acc[kBlockSlots][4][2];
#pragma unroll
    for (int s = 0; s < kBlockSlots; ++s)
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[s][q][0] = acc[s][q][1] = 0.0;
    const int nb2 = (nt + 1) >> 1;
    int my_bi[kBlockSlots], my_bj[kBlockSlots];  // this warp's blocks (an empty slot gets a row past the triangle)
#pragma unroll
    for (int s = 0; s < kBlockSlots; ++s) {
        const int t = kSyrkBlockOfSlot[warp][s];
        int bi = 1 << 20, bj = 0;
        if (t >= 0) {
            bi = (int)((sqrtf(8.0f * (float)t + 1.0f) - 1.0f) * 0.5f);
            while ((bi + 1) * (bi + 2) / 2 <= t) ++bi;
            while (bi * (bi + 1) / 2 > t) --bi;
            bj = t - bi * (bi + 1) / 2;
        }
        my_bi[s] = bi; my_bj[s] = bj;
    }
    const int per = (wd.n_chunks + bd.p_split - 1) / bd.p_split;
    const int ch0 = blockIdx.x * per, ch1 = min(wd.n_chunks, ch0 + per);
    const int* crs = bd.chunk_rs + wd.chunk_off;
    const double* pbase = bd.vpanel + wd.panel_off;
    const int fr = lane >> 2, fc = lane & 3;
    int ic = ch0, ih = 0, slot_i = 0;  // issue cursor (chunk, half, stage)
    while (ic < ch1 && crs[ic] == 0) ++ic;
    int cc = ic, chh = 0, slot_c = 0;  // consume cursor
    uint32_t ph0 = 0, ph1 = 0;
    auto issue = [&]() {
        if (ic >= ch1) return;
        if (tid == 0) {
            const int rs = crs[ic];
            const uint32_t bytes = (uint32_t)(kHalfCols * rs * sizeof(double));
            mbar_expect_tx(&full[slot_i], bytes);
            tma_load_1d(stage + (size_t)slot_i * kStageDoubles,
                        pbase + bd.chunk_poff[wd.chunk_off + ic] + (size_t)ih * kHalfCols * rs, bytes, &full[slot_i]);
        }
        slot_i ^= 1;
        if (ih == 0) ih = 1;
        else { ih = 0; ++ic; while (ic < ch1 && crs[ic] == 0) ++ic; }
    };
    issue();
    while (cc < ch1) {
        issue();  // the other stage was released by the __syncthreads that ended the previous iteration
        if (slot_c == 0) { mbar_wait(&full[0], ph0); ph0 ^= 1; } else { mbar_wait(&full[1], ph1); ph1 ^= 1; }
        const int rs = crs[cc];
        const int t0 = bd.chunk_t0[wd.chunk_off + cc], t1 = bd.chunk_t1[wd.chunk_off + cc];
        const double* sb = stage + (size_t)slot_c * kStageDoubles + (size_t)fc * rs + fr;
        auto tile_row = [&](int i) -> int {  // panel row of tile i in this chunk, -1 if the chunk has no such rows
            if (i >= t0 && i < t1) return 8 * (i - t0);
            if (i == trhs) return 8 * (t1 - t0);
            return -1;
        };
#pragma unroll
        for (int s = 0; s < kBlockSlots; ++s) {
            const int bi = my_bi[s], bj = my_bj[s];
            if (bi >= nb2) continue;
            const int ri0 = tile_row(2 * bi), ri1 = tile_row(2 * bi + 1), rj0 = tile_row(2 * bj), rj1 = tile_row(2 * bj + 1);
            if ((ri0 < 0 && ri1 < 0) || (rj0 < 0 && rj1 < 0)) continue;
            const double* pa0 = sb + max(ri0, 0);
            const double* pa1 = sb + max(ri1, 0);
            const double* pb0 = sb + max(rj0, 0);
            const double* pb1 = sb + max(rj1, 0);
            const double mi0 = ri0 < 0 ? 0.0 : 1.0, mi1 = ri1 < 0 ? 0.0 : 1.0;
            const bool diag = bi == bj;
            if (ri0 >= 0 && ri1 >= 0 && rj0 >= 0 && rj1 >= 0) {
#pragma unroll 4
                for (int kk = 0; kk < kHalfCols; kk += 4) {
                    const size_t o = (size_t)kk * rs;
                    const double a0 = pa0[o], a1 = pa1[o], b0 = pb0[o], b1 = pb1[o];
                    dmma(acc[s][0][0], acc[s][0][1], a0, b0);
                    if (!diag) dmma(acc[s][1][0], acc[s][1][1], a0, b1);
                    dmma(acc[s][2][0], acc[s][2][1], a1, b0);
                    dmma(acc[s][3][0], acc[s][3][1], a1, b1);
                }
            } else {  // a block on the edge of the chunk's keyframe range: zero the missing fragments
#pragma unroll 2
                for (int kk = 0; kk < kHalfCols; kk += 4) {
                    const size_t o = (size_t)kk * rs;
                    const double a0 = pa0[o] * mi0, a1 = pa1[o] * mi1, b0 = pb0[o], b1 = pb1[o];
                    if (rj0 >= 0) {
                        dmma(acc[s][0][0], acc[s][0][1], a0, b0);
                        dmma(acc[s][2][0], acc[s][2][1], a1, b0);
                    }
                    if (rj1 >= 0) {
                        if (!diag) dmma(acc[s][1][0], acc[s][1][1], a0, b1);
                        dmma(acc[s][3][0], acc[s][3][1], a1, b1);
                    }
                }
            }
        }
        __syncthreads();
        slot_c ^= 1;
        if (chh == 0) chh = 1;
        else { chh = 0; ++cc; while (cc < ch1 && crs[cc] == 0) ++cc; }
    }
    double* out = bd.sred + wd.s_off * (size_t)bd.p_split + (size_t)blockIdx.x * wd.nr_cap * wd.nr_cap;
#pragma unroll
    for (int s = 0; s < kBlockSlots; ++s) {
        const int bi = my_bi[s], bj = my_bj[s];
        if (bi >= nb2) continue;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int i = 2 * bi + (q >> 1), j = 2 * bj + (q & 1);
            if (i >= nt || j > i) continue;
            double* o = out + (size_t)(8 * i + fr) * wd.nr_cap + 8 * j + 2 * fc;
            o[0] = acc[s][q][0];
            o[1] = acc[s][q][1];
        }
    }
}

// =====================================================================================================================
// reduced system: assemble S = F + Lambda - sum V V^T (+ rhs as an augmented row), blocked Cholesky in place, solve,
// candidate poses.  One CTA per window.
// =====================================================================================================================
constexpr int kNB = 32;           // Cholesky block size
constexpr int kPanelStride = 36;  // row stride of the shared-memory panel copy (row-major path)

// Views of the reduced system: row-major in global memory (any size), or the lower triangle packed as 8x8 tiles in
// shared memory (<= 192 rows).  Inside a tile the two 8x4 halves are stored one after the other, which is exactly the
// m8n8k4 fragment order: lane (fr, fc) reads half h at h*32 + fr*4 + fc -- conflict free.
struct RowMajorMat {
    double* p; int ld;
    __device__ __forceinline__ double& operator()(int r, int c) const { return p[(size_t)r * ld + c]; }
};
struct TiledMat {
    double* p;
    __device__ __forceinline__ double* tile(int I, int J) const { return p + (size_t)(I * (I + 1) / 2 + J) * 64; }
    __device__ __forceinline__ double& operator()(int r, int c) const {
        return tile(r >> 3, c >> 3)[((c & 4) << 3) + ((r & 7) << 2) + (c & 3)];
    }
};

// Cholesky of the 32x32 block in D (shared memory, row stride PS, lower part; identity-padded beyond the live rows)
// by one warp, lane = row.  Two levels: the columns are taken 8 at a time -- a left-looking update from the columns
// already done (operands from shared memory), then the 8 columns are factored in registers with shuffles.  The pivot
// uses rsqrt, whose value 1 / L_jj is kept in inv[] for the triangular solves that follow (no division on their
// critical path).  Returns false on a non-positive pivot.
__device__ inline bool warp_chol32(double* D, int PS, double* inv, int lane) {
    bool ok = true;
#pragma unroll 1
    for (int jb = 0; jb < 4; ++jb) {
        const int c0 = 8 * jb;
        double r[8];
#pragma unroll
        for (int c = 0; c < 8; ++c) r[c] = D[lane * PS + c0 + c];
#pragma unroll 2
        for (int q = 0; q < c0; ++q) {
            const double lq = D[lane * PS + q];
#pragma unroll
            for (int c = 0; c < 8; ++c) r[c] -= lq * D[(c0 + c) * PS + q];
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const double djj = __shfl_sync(0xffffffffu, r[j], c0 + j);
            if (!(djj > 0.0) || !isfinite(djj)) ok = false;
            const double rs = rsqrt(djj);
            const double lij = (lane == c0 + j) ? djj * rs : r[j] * rs;
            r[j] = lij;
            if (lane == c0 + j) inv[c0 + j] = rs;
#pragma unroll
            for (int c = j + 1; c < 8; ++c) {
                const double lcj = __shfl_sync(0xffffffffu, lij, c0 + c);
                r[c] -= lij * lcj;
            }
        }
        __syncwarp();
#pragma unroll
        for (int c = 0; c < 8; ++c) D[lane * PS + c0 + c] = (c0 + c <= lane) ? r[c] : 0.0;
        __syncwarp();
    }
    return ok;
}

#ifdef KBA_PHASE_CLOCKS  // debug build: cycle counts of the phases of k_reduced_solve for window 0
#define PHASE_DECL long long clk_[12] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0}; long long last_ = clock64()
#define PHASE_MARK(i) do { if (tid == 0 && w == 0) { clk_[i] = clock64(); last_ = clk_[i]; } } while (0)
#define PHASE_ACC(i) do { if (tid == 0 && w == 0) { const long long t_ = clock64(); clk_[i] += t_ - last_; last_ = t_; } } while (0)
#define PHASE_PRINT do { if (tid == 0 && w == 0) printf("reduced_solve cycles: sred %lld blocks %lld scale %lld chol %lld (diag %lld panel %lld trail %lld) backsub %lld tail %lld\n", clk_[1] - clk_[0], clk_[2] - clk_[1], clk_[3] - clk_[2], clk_[4] - clk_[3], clk_[8], clk_[9], clk_[10], clk_[5] - clk_[4], clk_[6] - clk_[5]); } while (0)
#else
#define PHASE_DECL
#define PHASE_MARK(i)
#define PHASE_ACC(i)
#define PHASE_PRINT
#endif

// partial Schur sums of the p_split CTAs of a window -> slot 0, fixed order (only launched when p_split > 1, i.e. when
// the batch is too small to fill the GPU with one CTA per window)
// mode 0: fold the partials and (row-major solve) write A; 1: fold only; 2: write A from slot 0 (after the exchange)
__global__ void __launch_bounds__(256) k_sred_reduce(BatchDev bd, int mode) {
    const int w = blockIdx.y;
    const WinState& st = bd.state[w];
    if (st.phase != PH_ITERATE || st.solve_failed) return;
    const WinDesc& wd = bd.desc[w];
    if (wd.landmarks_fixed) return;
    const int ld = wd.nr_cap, n = st.n_f;
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    // tiled solve (<= 192 rows), mode 0: this kernel also writes A = -Sred in the tile-packed order of the solve kernel's shared
    // memory (TiledMat), zero padding included, so that the single CTA of k_reduced_solve copies it linearly instead of gathering
    // element by element (its assembly was 37 k of the kernel's 237 k cycles at 174 rows)
    const bool pack = mode == 0 && bd.solve_tiled;
    const int rows_t = (n + 8) & ~7;
    if (idx >= (pack ? rows_t : n + 1) * ld) return;
    const int r = idx / ld, c = idx - r * ld;
    if (pack) {
        if (c >= rows_t || (c >> 3) > (r >> 3)) return;
        if (c > r || r > n) {  // padding inside the packed triangle
            TiledMat{bd.amat + wd.s_off}(r, c) = -0.0;
            return;
        }
    } else if (c > r) return;
    double* sp0 = bd.sred + wd.s_off * (size_t)bd.p_split;
    const size_t pstride = (size_t)ld * ld;
    double s = 0.0;
    int used = bd.p_split;  // partials that were written: all of them, or (fused Schur kernel) those of the CTAs that own groups
    if (bd.fused) { int per; schur_split(wd.n_groups, bd.p_split, per, used); }
    if (mode == 2) s = sp0[idx];
    else
    for (int p0 = 0; p0 < used; p0 += 16) {  // 16 independent loads in flight, summed in slot order
        double v[16];
#pragma unroll
        for (int q = 0; q < 16; ++q) v[q] = (p0 + q < used) ? sp0[(size_t)(p0 + q) * pstride + idx] : 0.0;
#pragma unroll
        for (int q = 0; q < 16; ++q) s += v[q];
    }
    if (mode != 2) sp0[idx] = s;
    // row-major solve: A = -Sred is written here by the whole GPU instead of by the single CTA of the solve kernel
    if (mode != 1 && !bd.solve_tiled) bd.amat[wd.s_off + idx] = (r == n && c == n) ? 0.0 : -s;
    if (pack) TiledMat{bd.amat + wd.s_off}(r, c) = (r == n && c == n) ? -0.0 : -s;
}

// stage 0: the whole solve in this one CTA.  Large reduced systems of small batches split it (launch_pass): stage 1 =
// assembly, Jacobi scaling and damping only; then per 32-column block k_chol_diag / k_chol_panel / k_chol_trail spread
// the factorisation over many SMs (one SM's FP64 throughput bounds the n^3/3 trailing flops of a 594-row system);
// stage 2 = back substitution and candidate state only.
template <bool kTiled>
__global__ void __launch_bounds__(512, 1) k_reduced_solve(BatchDev bd, int stage) {
    const int w = blockIdx.x;
    const SolveParams& sp = bd.wsp[w];
    WinState& st = bd.state[w];
    if (st.phase != PH_ITERATE) return;
    const WinDesc& wd = bd.desc[w];
    const int tid = threadIdx.x, nth = blockDim.x;
    const int n = st.n_f, ld = wd.nr_cap;
    extern __shared__ __align__(16) double sm[];  // 16: the packed copy of A arrives in double2 units
    double* s_fdiag = sm;                 // [ld] squared column norms of J (f part)
    double* s_g = s_fdiag + ld;           // [ld] gradient J^T r (f part)
    double* s_y = s_g + ld;               // [ld]
    double* s_lam = s_y + ld;             // [ld]
    double* s_invd = s_lam + ld;          // [ld] 1 / L_ii (tiled path)
    double* s_inv = s_invd + ld;          // [kNB] 1 / L_ii of the block being factored
    double* s_D = s_inv + kNB;            // [kNB][kNB+1]
    double* s_P = s_D + kNB * (kNB + 1);  // row-major path: [ld][kNB+1] panel; tiled path: the packed lower triangle
    using Mat = typename std::conditional<kTiled, TiledMat, RowMajorMat>::type;
    Mat A;
    if constexpr (kTiled) A.p = s_P;
    else { A.p = bd.amat + wd.s_off; A.ld = ld; }
    __shared__ int s_fail;
    __shared__ double s_red[16][4];
    if (tid == 0) s_fail = 0;
    PHASE_DECL;
    PHASE_MARK(0);
    if (stage == 2) {  // the factor is in A (global), what the tail needs comes back from global memory
        if (st.solve_failed) return;  // also set by stage 1 (evaluation failure) and by k_chol_diag (not positive definite)
        for (int c = tid; c < n; c += nth) {
            s_g[c] = bd.grad_f[(size_t)w * bd.nr_cap_max + c];
            s_lam[c] = bd.lambda_f[(size_t)w * bd.nr_cap_max + c];
            s_invd[c] = bd.chol_invd[(size_t)w * bd.nr_cap_max + c];
        }
        __syncthreads();
    }
    if (stage != 2) {
    // ---- cost at x and evaluation failure (fresh linearisation only) ----
    // cost at x: every fresh linearisation, or -- one-kernel linearisation -- at iteration zero only (k_lm_update carries the accepted
    // candidate's cost over afterwards, kba_linearize.cuh)
    const bool eval_cost = bd.lin1 ? (st.need_linearize && st.iter0) : (st.need_linearize != 0);
    if (eval_cost && tid < 32) {  // warp 0: strided partial sums, then a butterfly (fixed shape)
        double c = 0.0;
        for (int q = tid; q < bd.cost_parts; q += 32) c += bd.cost_part_x[(size_t)w * bd.cost_parts + q];
        c = warp_sum(c);
        if (tid == 0) st.x_cost = c;  // regulariser cost added below
    }
    __syncthreads();
    if (st.eval_failed) {  // only reachable at iteration zero: "Residual and Jacobian evaluation failed."
        if (tid == 0) st.solve_failed = 2;
        return;
    }
    if (st.solve_failed) return;  // landmark block not positive definite -> invalid step

    for (int i = tid; i < ld; i += nth) { s_fdiag[i] = 0.0; s_g[i] = 0.0; }
    // ---- A(lower, rows 0..n incl. augmented row n) = - sum_p Sred_p ----
    {
        const double* sp0 = bd.sred + wd.s_off * (size_t)bd.p_split;
        const size_t pstride = (size_t)ld * ld;
        const int np = 1;  // with p_split > 1, k_sred_reduce has folded the partials into slot 0
        const int rows = kTiled ? ((n + 8) & ~7) : n + 1;  // tiled: whole tile rows, zero padded
        bool done_by_reduce = !kTiled && (bd.p_split > 1 || bd.sharded || bd.solve_banded) && !wd.landmarks_fixed;  // see k_sred_reduce
        if (kTiled && bd.p_split > 1 && !bd.sharded && !wd.landmarks_fixed) {
            // k_sred_reduce left A tile-packed and padded in global memory (L2): a linear copy, 16 bytes per thread and load
            const int ntr = rows >> 3;
            const int n2 = ntr * (ntr + 1) / 2 * 32;  // double2 elements
            const double2* src = reinterpret_cast<const double2*>(bd.amat + wd.s_off);
            double2* dst = reinterpret_cast<double2*>(s_P);
            for (int i0 = tid; i0 < n2; i0 += 4 * nth) {
                double2 v[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) if (i0 + u * nth < n2) v[u] = src[i0 + u * nth];
#pragma unroll
                for (int u = 0; u < 4; ++u) if (i0 + u * nth < n2) dst[i0 + u * nth] = v[u];
            }
            done_by_reduce = true;
        }
        // eight independent loads in flight per thread: the sums sit in L2, one load per iteration exposed its full latency
        const int total = done_by_reduce ? 0 : rows * ld;
        for (int idx0 = tid; idx0 < total; idx0 += 8 * nth) {
            double v[8];
            int rr[8], cc[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                const int idx = idx0 + u * nth;
                const int r = idx / ld, c = idx - r * ld;
                const bool skip = idx >= total || (kTiled ? (c >= rows || (c >> 3) > (r >> 3)) : (c > r || c >= n + 1));
                rr[u] = skip ? -1 : r; cc[u] = c;
                double s = 0.0;
                if (!skip && !wd.landmarks_fixed && c <= r && r <= n && !(r == n && c == n))  // motion-only: nothing was eliminated
                    for (int p = 0; p < np; ++p) s += sp0[p * pstride + (size_t)r * ld + c];
                v[u] = s;
            }
#pragma unroll
            for (int u = 0; u < 8; ++u)
                if (rr[u] >= 0) A(rr[u], cc[u]) = -v[u];
        }
    }
    __syncthreads();
    PHASE_MARK(1);
    // ---- + per-keyframe Gauss-Newton blocks ----
    for (int idx = tid; idx < wd.n_kf * 27; idx += nth) {
        const int k = idx / 27, q = idx - 27 * k;
        const int off = bd.off_pose[wd.kf_off + k];
        if (off < 0) continue;
        const double v = bd.bkf[(size_t)(wd.kf_off + k) * 27 + q];
        if (q < 21) {
            int a = 0, rem = q;
            while (rem >= 6 - a) { rem -= 6 - a; ++a; }
            const int b = a + rem;  // a <= b
            A(off + b, off + a) += v;
            if (a == b) s_fdiag[off + a] = v;
        } else {
            s_g[off + q - 21] = v;
        }
    }
    __syncthreads();
    // ---- + ground-plane blocks: per keyframe the 10 x 10 (pose | normal | distance) Gauss-Newton block of k_gp_blocks (on a
    //      sharded window: its sum over the ranks, so a rank without ground points adds the others' blocks) ----
    if (wd.n_gp > 0 || bd.shard_gp) {
        for (int idx = tid; idx < wd.n_kf * 65; idx += nth) {
            const int k = idx / 65, e = idx - 65 * k;
            int a, b;
            if (e < 55) { a = 0; while ((a + 1) * (a + 2) / 2 <= e) ++a; b = e - a * (a + 1) / 2; }
            else { a = e - 55; b = -1; }
            const int ra = gp_row(bd, wd, k, a);
            if (ra < 0) continue;
            const double v = bd.gp_kfb[(size_t)(wd.kf_off + k) * 65 + e];
            if (b < 0) { s_g[ra] += v; continue; }
            const int rb = gp_row(bd, wd, k, b);
            if (rb < 0) continue;
            A(ra, rb) += v;
            if (a == b) s_fdiag[ra] += v;
        }
        __syncthreads();
    }
    // ---- ground-plane regularisation chain (reference cpp:769-818), warp 0 cooperatively ----
    if (tid < 32 && wd.plane_reg_weight > 0 && wd.n_kf > 1) {
        const int lane = tid;
        const double wgt = wd.plane_reg_weight;
        const double* P = bd.pose[st.cur];
        const double* PL = bd.plane[st.cur];
        for (int k0 = 0; k0 + 1 < wd.n_kf; ++k0) {
            const int k1 = k0 + 1;
            const double* n0 = PL + 4 * (size_t)(wd.kf_off + k0), *n1 = PL + 4 * (size_t)(wd.kf_off + k1);
            {   // VectorDifferenceRegularization(dir1, dir0), weight 3w
                const double sq = sqrt(3.0 * wgt);
                double P1[9], P0[9], J[18], r[3];
                dir_plus_jacobian(n1, P1);
                dir_plus_jacobian(n0, P0);
                for (int i = 0; i < 3; ++i) {
                    r[i] = sq * (n1[i] - n0[i]);
                    for (int c = 0; c < 3; ++c) { J[6 * i + c] = sq * P1[3 * i + c]; J[6 * i + 3 + c] = -sq * P0[3 * i + c]; }
                }
                const int off[2] = {bd.off_dir[wd.kf_off + k1], bd.off_dir[wd.kf_off + k0]}, sz[2] = {3, 3};
                warp_add_block(A, s_fdiag, s_g, 3, r, 2, off, sz, J, lane);
            }
            {   // GroundPlaneDistanceRegularization(dist1, dist0), weight w
                const double sq = sqrt(wgt);
                const double r[1] = {sq * (n1[3] - n0[3])}, J[2] = {sq, -sq};
                const int off[2] = {bd.off_dist[wd.kf_off + k1], bd.off_dist[wd.kf_off + k0]}, sz[2] = {1, 1};
                warp_add_block(A, s_fdiag, s_g, 1, r, 2, off, sz, J, lane);
            }
            {   // GroundPlaneMotionRegularization(pose0, pose1, dir0), weight 2w
                const double sq = sqrt(2.0 * wgt);
                double j0[6], j1[6], jd[3], J[15];
                const double rm = plane_motion(P + 7 * (size_t)(wd.kf_off + k0), P + 7 * (size_t)(wd.kf_off + k1), n0, j0, j1, jd);
                for (int c = 0; c < 6; ++c) { J[c] = sq * j0[c]; J[6 + c] = sq * j1[c]; }
                for (int c = 0; c < 3; ++c) J[12 + c] = sq * jd[c];
                const double r[1] = {sq * rm};
                const int off[3] = {bd.off_pose[wd.kf_off + k0], bd.off_pose[wd.kf_off + k1], bd.off_dir[wd.kf_off + k0]};
                const int sz[3] = {6, 6, 3};
                warp_add_block(A, s_fdiag, s_g, 1, r, 3, off, sz, J, lane);
            }
        }
        for (int k = 0; k < wd.n_kf; ++k) {  // VectorDifferenceRegularization2((0,0,1)), weight w
            const double* n = PL + 4 * (size_t)(wd.kf_off + k);
            const double sq = sqrt(wgt);
            double Pn[9], J[9], r[3] = {sq * (0.0 - n[0]), sq * (0.0 - n[1]), sq * (1.0 - n[2])};
            dir_plus_jacobian(n, Pn);
            for (int i = 0; i < 9; ++i) J[i] = -sq * Pn[i];
            const int off[1] = {bd.off_dir[wd.kf_off + k]}, sz[1] = {3};
            warp_add_block(A, s_fdiag, s_g, 3, r, 1, off, sz, J, lane);
        }
        if (lane == 0 && eval_cost) st.x_cost += plane_chain_cost(wd, P, PL);
    }
    if (tid == 0 && (wd.n_gp > 0 || bd.shard_gp) && eval_cost) st.x_cost += bd.gp_cost_x[w];
    __syncthreads();
    // ---- regularisers (thread 0; a handful of residuals) ----
    if (tid == 0 && wd.scale_weight > 0) {
        const double* P = bd.pose[st.cur];
        double r, j1[6], j0[6];
        scale_regulariser(P + 7 * (size_t)(wd.kf_off + wd.scale_kf1), P + 7 * (size_t)(wd.kf_off + wd.scale_kf0),
                          wd.scale_value, r, j1, j0);
        const double sq = sqrt(wd.scale_weight);  // TrivialLoss * weight: rho' = w
        if (eval_cost) st.x_cost += 0.5 * wd.scale_weight * r * r;
        const int o1 = bd.off_pose[wd.kf_off + wd.scale_kf1], o0 = bd.off_pose[wd.kf_off + wd.scale_kf0];
        double J[12]; int cols[12]; int m = 0;
        if (o1 >= 0) for (int a = 0; a < 6; ++a) { J[m] = sq * j1[a]; cols[m++] = o1 + a; }
        if (o0 >= 0) for (int a = 0; a < 6; ++a) { J[m] = sq * j0[a]; cols[m++] = o0 + a; }
        const double rr = sq * r;
        for (int a = 0; a < m; ++a) {
            for (int b = 0; b < m; ++b)
                if (cols[b] <= cols[a]) A(cols[a], cols[b]) += J[a] * J[b];
            s_fdiag[cols[a]] += J[a] * J[a];
            s_g[cols[a]] += J[a] * rr;
        }
    }
    if (tid == 0 && wd.speed_weight > 0) {  // SpeedRegularizationVector2 of adjustPoseOnly (reference cpp:835-853)
        double r[3], J[18];
        speed_regulariser(bd.pose[st.cur] + 7 * (size_t)(wd.kf_off + wd.speed_kf), wd.speed_T_origin_before, wd.speed_v_before,
                          wd.speed_dt, r, J);
        if (eval_cost) st.x_cost += 0.5 * wd.speed_weight * (r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
        const int o = bd.off_pose[wd.kf_off + wd.speed_kf];
        if (o >= 0) {
            const double wgt = wd.speed_weight;  // rho' = w: J^T J and J^T r scale by w
            for (int a = 0; a < 6; ++a) {
                for (int b = 0; b <= a; ++b)
                    A(o + a, o + b) += wgt * (J[a] * J[b] + J[6 + a] * J[6 + b] + J[12 + a] * J[12 + b]);
                s_fdiag[o + a] += wgt * (J[a] * J[a] + J[6 + a] * J[6 + a] + J[12 + a] * J[12 + a]);
                s_g[o + a] += wgt * (J[a] * r[0] + J[6 + a] * r[1] + J[12 + a] * r[2]);
            }
        }
    }
    __syncthreads();
    PHASE_MARK(2);
    // ---- Jacobi scaling, damping, augmented row ----
    double* scale_f = bd.scale_f + (size_t)w * bd.nr_cap_max;
    double* lambda_f = bd.lambda_f + (size_t)w * bd.nr_cap_max;
    double* grad_f = bd.grad_f + (size_t)w * bd.nr_cap_max;
    for (int c = tid; c < n; c += nth) {
        double s;
        if (st.iter0) { s = 1.0 / (1.0 + sqrt(s_fdiag[c])); scale_f[c] = s; }
        else s = scale_f[c];
        const double s2 = s * s;
        const double lam = fmin(fmax(s_fdiag[c] * s2, sp.min_lm_diagonal), sp.max_lm_diagonal) / (st.radius * s2);
        s_lam[c] = lam;
        lambda_f[c] = lam;
        grad_f[c] = s_g[c];
        A(c, c) += lam;
        A(n, c) += s_g[c];  // augmented row: g_f - V z
    }
    __syncthreads();
    }  // stage != 2
    if (stage == 1) return;

    PHASE_MARK(3);
    // ---- blocked Cholesky (NB = 32) with the augmented row n carried along: diagonal block by one warp (registers +
    //      shuffles), panel by forward substitution (thread per row), trailing update on the FP64 tensor cores --
    //      tiled: operands and result straight from the tile-packed shared-memory storage; row-major: operands from
    //      the shared-memory copy of the panel (s_P, row stride 36: conflict-free fragments), result tiles in global ----
    const int lane = tid & 31, warp = tid >> 5, fr = lane >> 2, fc = lane & 3;
    const int NT = (n + 8) >> 3;  // tile rows, including the one holding the augmented row
    const int PS = kNB + 1;
    for (int kb = 0; kb < (stage == 0 ? n : 0); kb += kNB) {
        const int nb = min(kNB, n - kb);
        for (int idx = tid; idx < kNB * kNB; idx += nth) {  // stage the diagonal block, identity padded
            const int r = idx >> 5, c = idx & 31;
            s_D[r * PS + c] = (r < nb && c <= r) ? A(kb + r, kb + c) : ((r == c) ? 1.0 : 0.0);
        }
        __syncthreads();
        if (warp == 0 && !warp_chol32(s_D, PS, s_inv, lane)) s_fail = 1;
        __syncthreads();
        PHASE_ACC(8);
        if (s_fail) break;
        for (int idx = tid; idx < nb * kNB; idx += nth) {
            const int r = idx >> 5, c = idx & 31;
            if (c <= r) A(kb + r, kb + c) = s_D[r * PS + c];
        }
        if (tid < nb) s_invd[kb + tid] = s_inv[tid];
        // panel: rows below the block, including the augmented row n; X L^T = B column by column, each finished
        // column is eliminated from the remaining ones right away (independent FMAs, short critical path)
        const int r0 = kb + nb, m = n + 1 - r0;
        if constexpr (!kTiled) {  // coalesced copy of the panel rows into shared memory, zero padded to whole tiles
            for (int idx = tid; idx < ((m + 7) & ~7) * kNB; idx += nth) {
                const int i = idx >> 5, c = idx & 31;
                s_P[i * kPanelStride + c] = (i < m && c < nb) ? A(r0 + i, kb + c) : 0.0;
            }
            __syncthreads();
        }
        // Four lanes per row: lane a of a quad owns the columns c = 4 e + a.  Step q: the owner of column q scales it and
        // hands it to the quad (one shuffle), every lane eliminates it from its own later columns -- the same operations on the
        // same values in the same order as one thread per row, but 572 instead of 143 busy threads and a quarter of the
        // dependent chain per thread.
        {
            const int quad = tid >> 2, qa = tid & 3;
            const volatile double* vD = s_D;  // volatile: keeps the factor entries from being hoisted out of the row loop
            for (int ib = 0; ib < m; ib += nth >> 2) {  // warp-uniform trip count: every lane takes part in the shuffles
                const int i = ib + quad;
                const bool live = i < m;
                double x[kNB / 4];
#pragma unroll
                for (int e = 0; e < kNB / 4; ++e) {
                    const int c = 4 * e + qa;
                    if constexpr (kTiled) x[e] = (live && c < nb) ? A(r0 + i, kb + c) : 0.0;
                    else x[e] = live ? s_P[i * kPanelStride + c] : 0.0;
                }
#pragma unroll
                for (int q = 0; q < kNB; ++q) {
                    const int oe = q >> 2, oa = q & 3;
                    double xq = x[oe] * s_inv[q];  // meaningful on the owner lane only
                    xq = __shfl_sync(0xffffffffu, xq, (lane & ~3) | oa);
                    if (qa == oa) x[oe] = xq;
#pragma unroll
                    for (int e = oe; e < kNB / 4; ++e) {
                        const int c = 4 * e + qa;
                        if (e > oe || qa > oa) x[e] -= xq * vD[c * PS + q];
                    }
                }
#pragma unroll
                for (int e = 0; e < kNB / 4; ++e) {
                    const int c = 4 * e + qa;
                    if constexpr (kTiled) { if (live && c < nb) A(r0 + i, kb + c) = x[e]; }
                    else { if (live) s_P[i * kPanelStride + c] = x[e]; }
                }
            }
        }
        __syncthreads();
        if constexpr (!kTiled) {  // the factor's panel back to global memory (coalesced); s_P feeds the tensor cores
            for (int idx = tid; idx < m * kNB; idx += nth) {
                const int i = idx >> 5, c = idx & 31;
                if (c < nb) A(r0 + i, kb + c) = s_P[i * kPanelStride + c];
            }
        }
        PHASE_ACC(9);
        if (nb < kNB) break;  // last block: only the augmented row is left below it
        // trailing update: tile (I, J) -= sum_K tile(I, K) tile(J, K)^T over the 4 panel tile columns
        const int T0 = r0 >> 3, mt = NT - T0, ntile = mt * (mt + 1) / 2;
        auto tile_ij = [](int t, int& i, int& j) {
            i = (int)((sqrtf(8.0f * (float)t + 1.0f) - 1.0f) * 0.5f);
            while ((i + 1) * (i + 2) / 2 <= t) ++i;
            while (i * (i + 1) / 2 > t) --i;
            j = t - i * (i + 1) / 2;
        };
        if constexpr (kTiled) {
            for (int t = warp; t < ntile; t += nth >> 5) {
                int i, j;
                tile_ij(t, i, j);
                double a0 = 0.0, a1 = 0.0, b0 = 0.0, b1 = 0.0;  // two independent accumulator chains
                const double* pa = A.tile(T0 + i, kb >> 3) + fr * 4 + fc;
                const double* pb = A.tile(T0 + j, kb >> 3) + fr * 4 + fc;
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    dmma(a0, a1, pa[64 * k], pb[64 * k]);
                    dmma(b0, b1, pa[64 * k + 32], pb[64 * k + 32]);
                }
                double2* pc = reinterpret_cast<double2*>(A.tile(T0 + i, T0 + j) + (fc >> 1) * 32 + fr * 4 + (fc & 1) * 2);
                double2 cv = *pc;
                cv.x -= a0 + b0;
                cv.y -= a1 + b1;
                *pc = cv;
            }
        } else {
            // result tiles live in global memory (L2): the tile of the NEXT iteration is requested before this one's
            // tensor-core work so that its latency is hidden
            struct Req { int i, j; double2* pc; bool wr; double2 cv; };
            auto fetch = [=](int t) {
                Req q;
                q.i = (int)((sqrtf(8.0f * (float)t + 1.0f) - 1.0f) * 0.5f);
                while ((q.i + 1) * (q.i + 2) / 2 <= t) ++q.i;
                while (q.i * (q.i + 1) / 2 > t) --q.i;
                q.j = t - q.i * (q.i + 1) / 2;
                const int gr = r0 + 8 * q.i + fr, gc = r0 + 8 * q.j + 2 * fc;
                q.wr = gr <= n;  // rows past the augmented row do not exist in the row-major storage
                q.pc = reinterpret_cast<double2*>(A.p + (size_t)(q.wr ? gr : n) * A.ld + gc);
                q.cv = q.wr ? *q.pc : make_double2(0.0, 0.0);
                return q;
            };
            int t = warp;
            Req cur = fetch(t < ntile ? t : 0);
            while (t < ntile) {
                const int tn = t + (nth >> 5);
                const Req nxt = fetch(tn < ntile ? tn : t);
                double a0 = 0.0, a1 = 0.0, b0 = 0.0, b1 = 0.0;
                const double* pa = s_P + (8 * cur.i + fr) * kPanelStride + fc;
                const double* pb = s_P + (8 * cur.j + fr) * kPanelStride + fc;
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    dmma(a0, a1, pa[8 * k], pb[8 * k]);
                    dmma(b0, b1, pa[8 * k + 4], pb[8 * k + 4]);
                }
                if (cur.wr) {
                    cur.cv.x -= a0 + b0;
                    cur.cv.y -= a1 + b1;
                    *cur.pc = cur.cv;
                }
                t = tn;
                cur = nxt;
            }
        }
        __syncthreads();
        PHASE_ACC(10);
    }
    if (s_fail) {
        if (tid == 0) st.solve_failed = 1;
        return;
    }
    PHASE_MARK(4);
    // ---- blocked back substitution L^T d = y (y = augmented row), delta_f = -d ----
    for (int c = tid; c < n; c += nth) s_y[c] = A(n, c);
    __syncthreads();
    for (int kb = ((n - 1) / kNB) * kNB; kb >= 0; kb -= kNB) {
        const int nb = min(kNB, n - kb);
        for (int idx = tid; idx < kNB * kNB; idx += nth) {  // stage the diagonal block of L
            const int r = idx >> 5, c = idx & 31;
            s_D[r * PS + c] = (r < nb && c <= r) ? A(kb + r, kb + c) : 0.0;
        }
        __syncthreads();
        if (warp == 0) {  // lane k owns unknown kb + k of the diagonal block
            double yk = (lane < nb) ? s_y[kb + lane] : 0.0;
            const double ik = (lane < nb) ? s_invd[kb + lane] : 0.0;
#pragma unroll 4
            for (int i = nb - 1; i >= 0; --i) {
                const double lik = s_D[i * PS + lane];  // zero above the diagonal
                const double di = __shfl_sync(0xffffffffu, yk * ik, i);
                yk = (lane == i) ? di : yk - lik * di;
            }
            if (lane < nb) s_y[kb + lane] = yk;
        }
        __syncthreads();
        for (int k = tid; k < kb; k += nth) {
            double acc = s_y[k];
            for (int i = 0; i < nb; ++i) acc -= A(kb + i, k) * s_y[kb + i];
            s_y[k] = acc;
        }
        __syncthreads();
    }
    PHASE_MARK(5);
    double* delta_f = bd.delta_f + (size_t)w * bd.nr_cap_max;
    double model = 0.0;
    int bad = 0;
    for (int c = tid; c < n; c += nth) {
        const double d = -s_y[c];
        delta_f[c] = d;
        if (!isfinite(d)) bad = 1;
        model += -s_g[c] * d + s_lam[c] * d * d;
    }
    // ---- candidate poses, step / state norms, gradient max-norm of the pose blocks ----
    double step_sq = 0.0, xn_sq = 0.0, gmax = 0.0;
    const double* Pc = bd.pose[st.cur];
    double* Pn = bd.pose[1 - st.cur];
    for (int k = tid; k < wd.n_kf; k += nth) {
        const double* p = Pc + 7 * (size_t)(wd.kf_off + k);
        double* q = Pn + 7 * (size_t)(wd.kf_off + k);
        const int off = bd.off_pose[wd.kf_off + k];
        double* qrt = bd.rt[1 - st.cur] + kPoseStride * (size_t)(wd.kf_off + k);
        if (off < 0) {
            for (int i = 0; i < 7; ++i) q[i] = p[i];
            write_rt(qrt, p);
            continue;
        }
        double d[6], gneg[6], out[7];
        for (int i = 0; i < 6; ++i) { d[i] = -s_y[off + i]; gneg[i] = -s_g[off + i]; }
        pose_plus(p, d, out);
        write_rt(qrt, out);
        for (int i = 0; i < 7; ++i) { q[i] = out[i]; const double e = out[i] - p[i]; step_sq += e * e; xn_sq += p[i] * p[i]; }
        pose_plus(p, gneg, out);
        for (int i = 0; i < 7; ++i) gmax = fmax(gmax, fabs(out[i] - p[i]));
    }
    // plane blocks: normal through FixScaleVectorPlus, distance Euclidean; constant ones are copied
    for (int k = tid; k < wd.n_kf; k += nth) {
        const double* pl = bd.plane[st.cur] + 4 * (size_t)(wd.kf_off + k);
        double* ql = bd.plane[1 - st.cur] + 4 * (size_t)(wd.kf_off + k);
        const int od = bd.off_dir[wd.kf_off + k], oz = bd.off_dist[wd.kf_off + k];
        if (od < 0) { ql[0] = pl[0]; ql[1] = pl[1]; ql[2] = pl[2]; }
        else {
            double d[3], gneg[3], out[3];
            for (int i = 0; i < 3; ++i) { d[i] = -s_y[od + i]; gneg[i] = -s_g[od + i]; }
            dir_plus(pl, d, out);
            for (int i = 0; i < 3; ++i) { ql[i] = out[i]; const double e = out[i] - pl[i]; step_sq += e * e; xn_sq += pl[i] * pl[i]; }
            dir_plus(pl, gneg, out);
            for (int i = 0; i < 3; ++i) gmax = fmax(gmax, fabs(out[i] - pl[i]));
        }
        if (oz < 0) ql[3] = pl[3];
        else {
            const double d = -s_y[oz];
            ql[3] = pl[3] + d;
            step_sq += d * d; xn_sq += pl[3] * pl[3];
            gmax = fmax(gmax, fabs(s_g[oz]));
        }
    }
    model = warp_sum(model); step_sq = warp_sum(step_sq); xn_sq = warp_sum(xn_sq); gmax = warp_max(gmax);
    if (bad) s_fail = 1;
    if ((tid & 31) == 0) { s_red[tid >> 5][0] = model; s_red[tid >> 5][1] = step_sq; s_red[tid >> 5][2] = xn_sq; s_red[tid >> 5][3] = gmax; }
    __syncthreads();
    if (tid == 0) {
        double a = 0, b = 0, c = 0, g = 0;
        for (int q = 0; q < (nth >> 5); ++q) { a += s_red[q][0]; b += s_red[q][1]; c += s_red[q][2]; g = fmax(g, s_red[q][3]); }
        st.f_model = a; st.f_step_sq = b; st.f_xnorm_sq = c; st.f_gmax = g;
        if (s_fail) st.solve_failed = 1;
    }
    PHASE_MARK(6);
    PHASE_PRINT;
}

// ---------------------------------------------------------------------------------------------------------------------
// Split factorisation of a large reduced system (row-major A in global memory), one 32-column block per launch triple.
// ---------------------------------------------------------------------------------------------------------------------
// diagonal block: Cholesky by one warp, then W = L11^-1 (lane j solves column j), both to global memory
__global__ void __launch_bounds__(32) k_chol_diag(BatchDev bd, int kb) {
    const int w = blockIdx.x, lane = threadIdx.x;
    WinState& st = bd.state[w];
    if (st.phase != PH_ITERATE || st.solve_failed || kb >= st.n_f) return;
    const WinDesc& wd = bd.desc[w];
    const int n = st.n_f, ld = wd.nr_cap, nb = min(kNB, n - kb), PS = kNB + 1;
    double* A = bd.amat + wd.s_off;
    __shared__ double s_D[kNB * (kNB + 1)];
    __shared__ double s_inv[kNB];
    for (int r = 0; r < kNB; ++r)  // row r of the block: coalesced, identity padded
        s_D[r * PS + lane] = (r < nb && lane <= r) ? A[(size_t)(kb + r) * ld + kb + lane] : ((r == lane) ? 1.0 : 0.0);
    __syncwarp();
    if (!warp_chol32(s_D, PS, s_inv, lane)) { if (lane == 0) st.solve_failed = 1; return; }
    for (int r = 0; r < nb; ++r)
        if (lane <= r) A[(size_t)(kb + r) * ld + kb + lane] = s_D[r * PS + lane];
    if (lane < nb) bd.chol_invd[(size_t)w * bd.nr_cap_max + kb + lane] = s_inv[lane];
    // column `lane` of L11^-1 by forward substitution (the identity padding keeps rows >= nb trivial)
    double wv[kNB];
#pragma unroll
    for (int i = 0; i < kNB; ++i) {
        double acc = (i == lane) ? 1.0 : 0.0;
#pragma unroll
        for (int k = 0; k < i; ++k) acc -= s_D[i * PS + k] * wv[k];
        wv[i] = acc * s_inv[i];
    }
    double* W = bd.chol_w + (size_t)w * kNB * kNB;  // row-major: W[c][q] = (L11^-1)[c][q]
#pragma unroll
    for (int i = 0; i < kNB; ++i) W[i * kNB + lane] = wv[i];
}

// panel: X = B L11^-T = B W^T on the tensor cores, one warp per 8-row strip below the block (incl. the augmented row)
__global__ void __launch_bounds__(512) k_chol_panel(BatchDev bd, int kb) {
    const int w = blockIdx.y;
    const WinState& st = bd.state[w];
    if (st.phase != PH_ITERATE || st.solve_failed || kb >= st.n_f) return;
    const WinDesc& wd = bd.desc[w];
    const int n = st.n_f, ld = wd.nr_cap, nb = min(kNB, n - kb);
    const int r0 = kb + nb, m = n + 1 - r0;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, fr = lane >> 2, fc = lane & 3;
    __shared__ double s_W[kNB * kPanelStride];
    for (int idx = tid; idx < kNB * kNB; idx += blockDim.x)
        s_W[(idx >> 5) * kPanelStride + (idx & 31)] = bd.chol_w[(size_t)w * kNB * kNB + idx];
    __syncthreads();
    const int strip = blockIdx.x * 16 + warp;
    if (8 * strip >= m) return;
    double* A = bd.amat + wd.s_off;
    const int gr = r0 + 8 * strip + fr;
    const bool live = gr <= n;
    double a[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) a[k] = (live && 4 * k + fc < nb) ? A[(size_t)gr * ld + kb + 4 * k + fc] : 0.0;
    double c[4][2];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
        c[t][0] = c[t][1] = 0.0;
#pragma unroll
        for (int k = 0; k < 8; ++k) dmma(c[t][0], c[t][1], a[k], s_W[(8 * t + fr) * kPanelStride + 4 * k + fc]);
    }
    __syncwarp();  // every lane has read its part of the strip before any of it is overwritten
    if (live) {
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            const int cc = 8 * t + 2 * fc;
            if (cc < nb) A[(size_t)gr * ld + kb + cc] = c[t][0];
            if (cc + 1 < nb) A[(size_t)gr * ld + kb + cc + 1] = c[t][1];
        }
    }
}

// trailing update A22 -= X X^T: every CTA copies the panel into shared memory and takes every gridDim.x-th share of
// the result tiles (tensor cores, result tiles read-modify-written in global memory)
__global__ void __launch_bounds__(512, 1) k_chol_trail(BatchDev bd, int kb) {
    const int w = blockIdx.y;
    const WinState& st = bd.state[w];
    if (st.phase != PH_ITERATE || st.solve_failed || kb + kNB >= st.n_f) return;  // nothing below a last, partial block
    const WinDesc& wd = bd.desc[w];
    const int n = st.n_f, ld = wd.nr_cap;
    const int r0 = kb + kNB, m = n + 1 - r0, mt = (m + 7) >> 3, ntile = mt * (mt + 1) / 2;
    const int tid = threadIdx.x, lane = tid & 31, fr = lane >> 2, fc = lane & 3;
    extern __shared__ double s_P[];  // [8 * mt][kPanelStride]
    double* A = bd.amat + wd.s_off;
    for (int idx = tid; idx < 8 * mt * kNB; idx += blockDim.x) {
        const int i = idx >> 5, c = idx & 31;
        s_P[i * kPanelStride + c] = (i < m) ? A[(size_t)(r0 + i) * ld + kb + c] : 0.0;
    }
    __syncthreads();
    const int nw = gridDim.x * (blockDim.x >> 5);
    for (int t = blockIdx.x * (blockDim.x >> 5) + (tid >> 5); t < ntile; t += nw) {
        int i = (int)((sqrtf(8.0f * (float)t + 1.0f) - 1.0f) * 0.5f);
        while ((i + 1) * (i + 2) / 2 <= t) ++i;
        while (i * (i + 1) / 2 > t) --i;
        const int j = t - i * (i + 1) / 2;
        const int gr = r0 + 8 * i + fr, gc = r0 + 8 * j + 2 * fc;
        const bool wr = gr <= n;
        double2* pc = reinterpret_cast<double2*>(A + (size_t)(wr ? gr : n) * ld + gc);
        double2 cv = wr ? *pc : make_double2(0.0, 0.0);  // requested before the tensor-core work
        double a0 = 0.0, a1 = 0.0, b0 = 0.0, b1 = 0.0;
        const double* pa = s_P + (8 * i + fr) * kPanelStride + fc;
        const double* pb = s_P + (8 * j + fr) * kPanelStride + fc;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            dmma(a0, a1, pa[8 * k], pb[8 * k]);
            dmma(b0, b1, pa[8 * k + 4], pb[8 * k + 4]);
        }
        if (wr) {
            cv.x -= a0 + b0;
            cv.y -= a1 + b1;
            *pc = cv;
        }
    }
}

// trailing update above kPanelMaxRows rows, where no CTA holds the whole panel: the result is cut into 64x64 blocks (I >= J)
// and every CTA takes every gridDim.x-th block, staging only the 64 panel rows of its row band and the 64 of its column band
// (36 KB whatever n).  Warp w computes the 16x8 tiles (w & 3, 4 (w >> 2) .. 4 (w >> 2) + 3) of the block on m16n8k8 DMMA: one
// accumulator per tile, the 32 panel columns summed in column order from zero, then subtracted from the element -- the same
// operations for an element whichever CTA owns its block, so any solve_split gives the same bits.
constexpr int kBandRows = 64;
__global__ void __launch_bounds__(256, 2) k_chol_trail_band(BatchDev bd, int kb) {
    const int w = blockIdx.y;
    const WinState& st = bd.state[w];
    if (st.phase != PH_ITERATE || st.solve_failed || kb + kNB >= st.n_f) return;  // nothing below a last, partial block
    const WinDesc& wd = bd.desc[w];
    const int n = st.n_f, ld = wd.nr_cap;
    const int r0 = kb + kNB, m = n + 1 - r0, nbk = (m + kBandRows - 1) / kBandRows, npair = nbk * (nbk + 1) / 2;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, fr = lane >> 2, fc = lane & 3;
    __shared__ double s_X[2][kBandRows * kPanelStride];  // panel rows of the row band, of the column band
    double* A = bd.amat + wd.s_off;
    const int ta = warp & 3, tb0 = 4 * (warp >> 2);  // 16-row strip, first of the warp's four 8-column tiles
    for (int p = blockIdx.x; p < npair; p += gridDim.x) {
        int I = (int)((sqrtf(8.0f * (float)p + 1.0f) - 1.0f) * 0.5f);
        while ((I + 1) * (I + 2) / 2 <= p) ++I;
        while (I * (I + 1) / 2 > p) --I;
        const int J = p - I * (I + 1) / 2;
        for (int idx = tid; idx < 2 * kBandRows * kNB; idx += blockDim.x) {
            const int h = idx / (kBandRows * kNB), i = (idx >> 5) & (kBandRows - 1), c = idx & 31;
            const int row = kBandRows * (h ? J : I) + i;
            s_X[h][i * kPanelStride + c] = row < m ? A[(size_t)(r0 + row) * ld + kb + c] : 0.0;
        }
        // the result elements this lane updates, requested before the tensor-core work: rows gr, gr + 8, columns gc, gc + 1
        const int gr = r0 + kBandRows * I + 16 * ta + fr;
        double2 cv[4][2];
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            const int gc = r0 + kBandRows * J + 8 * (tb0 + t) + 2 * fc;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = gr + 8 * h;
                cv[t][h] = make_double2(0.0, 0.0);
                if (r <= n && gc + 1 <= r) cv[t][h] = *reinterpret_cast<const double2*>(A + (size_t)r * ld + gc);
                else if (r <= n && gc <= r) cv[t][h].x = A[(size_t)r * ld + gc];
            }
        }
        __syncthreads();
        // a 16x8 tile that lies above the diagonal of a diagonal block, or below the last row, is not computed
        const bool rows_live = kBandRows * I + 16 * ta < m;
        double c[4][4];
#pragma unroll
        for (int t = 0; t < 4; ++t) c[t][0] = c[t][1] = c[t][2] = c[t][3] = 0.0;
        if (rows_live) {
            const double* pa = s_X[0] + (16 * ta + fr) * kPanelStride + fc;
            const double* pb = s_X[1] + (8 * tb0 + fr) * kPanelStride + fc;
#pragma unroll
            for (int k = 0; k < kNB; k += 8) {
                const double a0 = pa[k], a1 = pa[8 * kPanelStride + k], a2 = pa[k + 4], a3 = pa[8 * kPanelStride + k + 4];
#pragma unroll
                for (int t = 0; t < 4; ++t)
                    if (I > J || 8 * (tb0 + t) <= 16 * ta + 15)
                        dmma16k8(c[t], a0, a1, a2, a3, pb[8 * t * kPanelStride + k], pb[8 * t * kPanelStride + k + 4]);
            }
        }
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            const int gc = r0 + kBandRows * J + 8 * (tb0 + t) + 2 * fc;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = gr + 8 * h;
                double2 v = cv[t][h];
                v.x -= c[t][2 * h];
                v.y -= c[t][2 * h + 1];
                if (r <= n && gc + 1 <= r) *reinterpret_cast<double2*>(A + (size_t)r * ld + gc) = v;
                else if (r <= n && gc <= r) A[(size_t)r * ld + gc] = v.x;
            }
        }
        __syncthreads();  // the next block's panel rows overwrite s_X
    }
}

// =====================================================================================================================
// back-substitution: delta_p_j = -L^-T (z_j + sum_i V_i^T delta_f,i); candidate landmarks; deterministic partial sums
// =====================================================================================================================
__global__ void __launch_bounds__(256) k_backsub(BatchDev bd) {
    // 16 lanes per landmark (tracks average ~13 observations); every shuffle sits outside the divergent parts
    const int w = blockIdx.y;
    const WinState& st = bd.state[w];
    if (st.phase != PH_ITERATE) return;
    const WinDesc& wd = bd.desc[w];
    const int hl = threadIdx.x & 15, grp = threadIdx.x >> 4;
    const int j = blockIdx.x * 16 + grp;
    __shared__ double s_red[16][4];
    double model = 0.0, step_sq = 0.0, xn_sq = 0.0, gmax = 0.0;
    const bool have = j < wd.n_lm;
    const int L = wd.lm_off + (have ? j : 0);
    const double* pc = bd.lm[st.cur] + 3 * (size_t)L;
    double* pn = bd.lm[1 - st.cur] + 3 * (size_t)L;
    const int* lm_ptr = bd.lm_ptr + wd.lm_off + w;
    const int o0 = have ? lm_ptr[j] : 0, o1 = have ? lm_ptr[j + 1] : 0;
    const bool in = have && bd.lm_active[L] && o1 > o0 && !wd.landmarks_fixed && !st.solve_failed;
    const size_t base = (size_t)wd.obs_off;
    const double* delta_f = bd.delta_f + (size_t)w * bd.nr_cap_max;
    double t[3] = {0, 0, 0};
    const int gl = (in && wd.n_gp > 0) ? bd.gp_of_lm[L] : -1;
    bool mine = false;  // panel mode: the gp block's pose rows were added onto one of this landmark's observation rows
    if (in) {
        const double* pcol = nullptr;
        int prs = 0, prow0 = 0;
        {
            const int ch = wd.chunk_off + (j >> 5);
            prs = bd.chunk_rs[ch];
            prow0 = 8 * bd.chunk_t0[ch];
            pcol = bd.vpanel + wd.panel_off + bd.chunk_poff[ch] + (size_t)(3 * (j & 31)) * prs;
        }
        const int gk = (gl >= 0) ? bd.gp_kf[wd.gp_off + gl] : -1;
        for (int o = o0 + hl; o < o1; o += 16) {
            if (gk >= 0) mine |= (bd.obs_kf[base + o] == gk);
            const int off = bd.obs_row[base + o];  // row of the observation's pose block (k_solve_begin), -1: constant
            if (off < 0) continue;
            // the panel rows hold the sum over the rig's cameras: read them once (rank 0)
            if (bd.obs_rank[base + o] != 0) continue;
            const double* q = pcol + (off - prow0);
#pragma unroll
            for (int r = 0; r < 6; ++r) {
                const double d = delta_f[off + r];
                t[0] += q[r] * d; t[1] += q[prs + r] * d; t[2] += q[2 * prs + r] * d;
            }
        }
    }
    const unsigned any = __ballot_sync(0xffffffffu, mine) & (0xffffu << (threadIdx.x & 16));
    if (gl >= 0 && hl < 10 && !(any != 0u && hl < 6)) {  // row `hl` of the gp block's 10 x 3 V
        const int row = gp_row(bd, wd, bd.gp_kf[wd.gp_off + gl], hl);
        if (row >= 0) {
            const double d = delta_f[row];
#pragma unroll
            for (int c = 0; c < 3; ++c) t[c] += bd.vgp[(size_t)(3 * hl + c) * bd.tot_gp + wd.gp_off + gl] * d;
        }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int m = 8; m >= 1; m >>= 1) t[c] += __shfl_xor_sync(0xffffffffu, t[c], m);
    if (have && hl == 0) {
        if (!in) {
            pn[0] = pc[0]; pn[1] = pc[1]; pn[2] = pc[2];
        } else {
            const double* z = bd.lm_z + 3 * (size_t)L;
            const double* li = bd.lm_linv + 6 * (size_t)L;  // i00; i10 i11; i20 i21 i22
            const double t0 = t[0] + z[0], t1 = t[1] + z[1], t2 = t[2] + z[2];
            // delta_p = -Linv^T t
            const double d0 = -(li[0] * t0 + li[1] * t1 + li[3] * t2);
            const double d1 = -(li[2] * t1 + li[4] * t2);
            const double d2 = -(li[5] * t2);
            const double* g = bd.lm_g + 3 * (size_t)L;
            const double* lam = bd.lm_lambda + 3 * (size_t)L;
            pn[0] = pc[0] + d0; pn[1] = pc[1] + d1; pn[2] = pc[2] + d2;
            model = -(g[0] * d0 + g[1] * d1 + g[2] * d2) + lam[0] * d0 * d0 + lam[1] * d1 * d1 + lam[2] * d2 * d2;
            step_sq = d0 * d0 + d1 * d1 + d2 * d2;
            xn_sq = pc[0] * pc[0] + pc[1] * pc[1] + pc[2] * pc[2];
            gmax = fmax(fabs(g[0]), fmax(fabs(g[1]), fabs(g[2])));
            if (!isfinite(d0) || !isfinite(d1) || !isfinite(d2)) model = nan("");
        }
    }
    if (hl == 0) { s_red[grp][0] = model; s_red[grp][1] = step_sq; s_red[grp][2] = xn_sq; s_red[grp][3] = gmax; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double a = 0, b = 0, c = 0, g = 0;
        for (int q = 0; q < 16; ++q) { a += s_red[q][0]; b += s_red[q][1]; c += s_red[q][2]; g = fmax(g, s_red[q][3]); }
        double* out = bd.bs_part + ((size_t)w * bd.bs_parts + blockIdx.x) * 4;
        out[0] = a; out[1] = b; out[2] = c; out[3] = g;
    }
}

// Fused path: sum_i V_i^T delta_f,i from the compact per-observation V (k_obs_v2; landmark-column-major): each lane reads
// its observation's three 48-byte column segments with nine 128-bit loads, consecutive lanes consecutive segments.
// Tried and dropped: requesting the V segments before obs_row has come back and the landmark's L^-1 / z / g / lambda before the
// reduction (one round of memory latency instead of three) made the headline step slower -- not profiled further.
// kLoop: the CTAs of a window stride over its 16-landmark units (grid.x < n_units, LaunchCfg::bs_grid); unit = partial-sum slot
template <bool kLoop>
__global__ void __launch_bounds__(256) k_backsub_v(BatchDev bd, int n_units) {
    const int w = blockIdx.y;
    const WinState& st = bd.state[w];
    if (st.phase != PH_ITERATE) return;
    const WinDesc& wd = bd.desc[w];
    __shared__ double s_red[16][4];
    const int hl = threadIdx.x & 15, grp = threadIdx.x >> 4;
    for (int unit = blockIdx.x; unit < n_units; unit += gridDim.x) {
    const int j = unit * 16 + grp;
    double model = 0.0, step_sq = 0.0, xn_sq = 0.0, gmax = 0.0;
    const bool have = j < wd.n_lm;
    const int L = wd.lm_off + (have ? j : 0);
    const double* pc = bd.lm[st.cur] + 3 * (size_t)L;
    double* pn = bd.lm[1 - st.cur] + 3 * (size_t)L;
    const int* lm_ptr = bd.lm_ptr + wd.lm_off + w;
    const int o0 = have ? lm_ptr[j] : 0, o1 = have ? lm_ptr[j + 1] : 0;
    const bool in = have && bd.lm_active[L] && o1 > o0 && !wd.landmarks_fixed && !st.solve_failed;
    const size_t base = (size_t)wd.obs_off;
    const double* delta_f = bd.delta_f + (size_t)w * bd.nr_cap_max;
    double t[3] = {0, 0, 0};
    if (in) {
        for (int o = o0 + hl; o < o1; o += 16) {
            const int off = bd.obs_row[base + o];  // row of the observation's pose block (k_solve_begin), -1: constant
            if (off < 0) continue;
            double d[6];
#pragma unroll
            for (int r = 0; r < 6; ++r) d[r] = delta_f[off + r];
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const double2* v = reinterpret_cast<const double2*>(bd.vobs + vobs_index(base, o0, o1, o, c));
#pragma unroll
                for (int h = 0; h < 3; ++h) {
                    const double2 x = v[h];
                    t[c] += x.x * d[2 * h] + x.y * d[2 * h + 1];
                }
            }
        }
        const int gl = (wd.n_gp > 0) ? bd.gp_of_lm[L] : -1;
        if (gl >= 0 && hl < 10) {  // row `hl` of the gp block's 10 x 3 V
            const int row = gp_row(bd, wd, bd.gp_kf[wd.gp_off + gl], hl);
            if (row >= 0) {
                const double d = delta_f[row];
#pragma unroll
                for (int c = 0; c < 3; ++c) t[c] += bd.vgp[(size_t)(3 * hl + c) * bd.tot_gp + wd.gp_off + gl] * d;
            }
        }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int m = 8; m >= 1; m >>= 1) t[c] += __shfl_xor_sync(0xffffffffu, t[c], m);
    if (have && hl == 0) {
        if (!in) {
            pn[0] = pc[0]; pn[1] = pc[1]; pn[2] = pc[2];
        } else {
            const double* z = bd.lm_z + 3 * (size_t)L;
            const double* li = bd.lm_linv + 6 * (size_t)L;  // i00; i10 i11; i20 i21 i22
            const double t0 = t[0] + z[0], t1 = t[1] + z[1], t2 = t[2] + z[2];
            // delta_p = -Linv^T t
            const double d0 = -(li[0] * t0 + li[1] * t1 + li[3] * t2);
            const double d1 = -(li[2] * t1 + li[4] * t2);
            const double d2 = -(li[5] * t2);
            const double* g = bd.lm_g + 3 * (size_t)L;
            const double* lam = bd.lm_lambda + 3 * (size_t)L;
            pn[0] = pc[0] + d0; pn[1] = pc[1] + d1; pn[2] = pc[2] + d2;
            model = -(g[0] * d0 + g[1] * d1 + g[2] * d2) + lam[0] * d0 * d0 + lam[1] * d1 * d1 + lam[2] * d2 * d2;
            step_sq = d0 * d0 + d1 * d1 + d2 * d2;
            xn_sq = pc[0] * pc[0] + pc[1] * pc[1] + pc[2] * pc[2];
            gmax = fmax(fabs(g[0]), fmax(fabs(g[1]), fabs(g[2])));
            if (!isfinite(d0) || !isfinite(d1) || !isfinite(d2)) model = nan("");
        }
    }
    if (hl == 0) { s_red[grp][0] = model; s_red[grp][1] = step_sq; s_red[grp][2] = xn_sq; s_red[grp][3] = gmax; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double a = 0, b = 0, c = 0, g = 0;
        for (int q = 0; q < 16; ++q) { a += s_red[q][0]; b += s_red[q][1]; c += s_red[q][2]; g = fmax(g, s_red[q][3]); }
        double* out = bd.bs_part + ((size_t)w * bd.bs_parts + unit) * 4;
        out[0] = a; out[1] = b; out[2] = c; out[3] = g;
    }
    if constexpr (!kLoop) break;
    if (unit + (int)gridDim.x < n_units) __syncthreads();  // s_red is rewritten by the next unit
    }  // units
}

// =====================================================================================================================
// LM controller: one thread per window.  Mirrors ceres 1.13 TrustRegionMinimizer + LevenbergMarquardtStrategy as
// restated in SURVEY.md A.6, and the solveTrimmed outer loop (reference robust_solving.cpp:140-248).
// =====================================================================================================================
// ---- sharded window: local partial sums -> the exchanged scalar block; flags out of / into the window state ----
__global__ void __launch_bounds__(32) k_shard_scalars(BatchDev bd) {  // after k_backsub and k_eval_obs<false>
    // one warp, the partials summed in k_lm_update's order: with one rank the exchanged scalars are the plain solve's bits
    const WinState& st = bd.state[0];
    const WinDesc& wd = bd.desc[0];
    const int lane = threadIdx.x;
    double a = 0, b = 0, c = 0, cc = 0, g = 0;
    if (st.phase == PH_ITERATE) {
        for (int q = lane; q < (wd.n_lm + 15) / 16; q += 32) {
            const double* p = bd.bs_part + (size_t)q * 4;
            a += p[0]; b += p[1]; c += p[2]; g = fmax(g, p[3]);
        }
        for (int q = lane; q < bd.cost_parts; q += 32) cc += bd.cost_part_c[q];
    }
    a = warp_sum(a); b = warp_sum(b); c = warp_sum(c); g = warp_max(g);
    cc = warp_sum(cc);
    if (lane == 0) {
        bd.xs[0] = a; bd.xs[1] = b; bd.xs[2] = c; bd.xs[3] = cc;
        bd.xs[4] = (st.phase == PH_ITERATE && st.eval_failed) ? 1.0 : 0.0;
        bd.xs[5] = (st.phase == PH_ITERATE && wd.n_gp > 0) ? bd.gp_cost_c[0] : 0.0;  // k_gp_eval<false>
        // the gradient max-norm rides in the same SUM all-reduce: one slot per rank, the others contribute zero
        for (int r = 0; r < bd.shard_world; ++r) bd.xs[16 + r] = (r == bd.shard_rank) ? g : 0.0;
    }
}
// The ONE exchange of a linearisation: [ reduced system (Schur sums + right-hand side) | pose blocks | (window with ground points:
// per-keyframe gp blocks, gp cost at x) | cost partials at x | evaluation-failed flag, landmark-block-not-PD flag ] packed into
// BatchDev::x_send, summed over the ranks into x_recv.  A rank without ground points contributes zeros to the gp segment.
// Out of place by construction: a pass that does not re-linearise (rejected step) packs the same local values again.
__host__ __device__ inline long long shard_gp_doubles(int shard_gp, int n_kf) { return shard_gp ? 65LL * n_kf + 1 : 0; }
__global__ void __launch_bounds__(256) k_shard_pack(BatchDev bd) {
    const WinState& st = bd.state[0];
    const WinDesc& wd = bd.desc[0];
    const size_t n_s = (size_t)wd.nr_cap * wd.nr_cap, n_b = (size_t)wd.n_kf * 27, n_c = (size_t)bd.shard_cost_parts;
    const size_t n_g = (size_t)shard_gp_doubles(bd.shard_gp, wd.n_kf), n_kb = (size_t)wd.n_kf * 65;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool on = st.phase == PH_ITERATE, gp = on && wd.n_gp > 0;
    if (i < n_s) bd.x_send[i] = on ? bd.sred[i] : 0.0;
    else if (i < n_s + n_b) bd.x_send[i] = on ? bd.bkf[i - n_s] : 0.0;
    else if (i < n_s + n_b + n_kb && n_g) bd.x_send[i] = gp ? bd.gp_kfb[i - n_s - n_b] : 0.0;
    else if (i == n_s + n_b + n_kb && n_g) bd.x_send[i] = gp ? bd.gp_cost_x[0] : 0.0;
    else if (i < n_s + n_b + n_g + n_c) {  // the ranks' slot counts differ: the segment has the largest, zero padded
        const size_t q = i - n_s - n_b - n_g;
        bd.x_send[i] = (on && q < (size_t)bd.cost_parts) ? bd.cost_part_x[q] : 0.0;
    }
    else if (i == n_s + n_b + n_g + n_c) bd.x_send[i] = (on && st.eval_failed) ? 1.0 : 0.0;
    else if (i == n_s + n_b + n_g + n_c + 1) bd.x_send[i] = (on && st.solve_failed) ? 1.0 : 0.0;
}
__global__ void k_shard_flags(BatchDev bd) {  // after the exchange: a failure on any rank is a failure of the window
    WinState& st = bd.state[0];
    if (threadIdx.x != 0 || st.phase != PH_ITERATE) return;
    const WinDesc& wd = bd.desc[0];
    const double* f = bd.x_recv + (size_t)wd.nr_cap * wd.nr_cap + (size_t)wd.n_kf * 27 + shard_gp_doubles(bd.shard_gp, wd.n_kf) +
                      bd.shard_cost_parts;
    if (f[0] > 0.0) st.eval_failed = 1;
    if (f[1] > 0.0 && !st.solve_failed) st.solve_failed = 1;
}
// trimming values of this rank's landmarks into their slots of the window-wide array (0 = not mine, v + 2 otherwise)
__global__ void __launch_bounds__(256) k_shard_trim_scatter(BatchDev bd) {
    const WinState& st = bd.state[0];
    if (st.phase != PH_TRIM) return;
    const WinDesc& wd = bd.desc[0];
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= wd.n_lm) return;
    const int gidx = bd.lm_begin + bd.lm_orig[j];
    for (int g = 0; g < 3; ++g) bd.trim_send[(size_t)g * bd.lm_total + gidx] = bd.trim_val[(size_t)g * bd.tot_lm + j] + 2.0;
}
// keyframe + 1 of this rank's ground points into their window-wide slots (gp_send is zero elsewhere); summed over the ranks
// (launch_shard_gather), every rank knows which keyframe each ground point of the whole window is attached to
__global__ void __launch_bounds__(256) k_shard_gp_gather(BatchDev bd) {
    const WinDesc& wd = bd.desc[0];
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= wd.n_gp) return;
    const size_t G = (size_t)wd.gp_off + g;
    bd.gp_send[bd.lm_begin + bd.lm_orig[wd.lm_off + bd.gp_lm[G]]] = (double)(bd.gp_kf[G] + 1);
}

__global__ void __launch_bounds__(128) k_lm_update(BatchDev bd) {
    // one warp per window: the lanes reduce the partial sums (fixed shape: strided partials, then a butterfly), lane 0
    // then runs the controller
    const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (w >= bd.n_win) return;
    WinState& st = bd.state[w];
    if (st.phase != PH_ITERATE) return;
    const WinDesc& wd = bd.desc[w];
    double e_model = 0, e_step = 0, e_xn = 0, e_g = 0, cand_sum = 0;
    for (int q = lane; q < (wd.n_lm + 15) / 16; q += 32) {
        const double* p = bd.bs_part + ((size_t)w * bd.bs_parts + q) * 4;
        e_model += p[0]; e_step += p[1]; e_xn += p[2]; e_g = fmax(e_g, p[3]);
    }
    for (int q = lane; q < bd.cost_parts; q += 32) cand_sum += bd.cost_part_c[(size_t)w * bd.cost_parts + q];
    e_model = warp_sum(e_model); e_step = warp_sum(e_step); e_xn = warp_sum(e_xn); e_g = warp_max(e_g);
    cand_sum = warp_sum(cand_sum);
    if (lane != 0) return;
    if (bd.sharded) {  // sums over all ranks (k_shard_scalars + all-reduce), identical on every rank
        e_model = bd.xs[0]; e_step = bd.xs[1]; e_xn = bd.xs[2]; cand_sum = bd.xs[3];
        e_g = 0.0;
        for (int r = 0; r < bd.shard_world; ++r) e_g = fmax(e_g, bd.xs[16 + r]);
        if (bd.xs[4] > 0.0) st.eval_failed = 1;
    }
    // the candidate's state (the controller flips st.cur only after it has asked for the candidate's cost)
    const double* P = bd.pose[1 - st.cur];
    const double* PL = bd.plane[1 - st.cur];
    const double* gp_cost = bd.sharded ? bd.xs + 5 : bd.gp_cost_c + w;
    const bool has_gp = wd.n_gp > 0 || bd.shard_gp;
    lm_step(st, bd.log + (size_t)w * kIterLogCap, bd.wsp[w], !bd.sharded, bd.lin1 != 0, e_model, e_step, e_xn, e_g,
            [&wd, cand_sum, P, PL, gp_cost, has_gp]() {
        double cand = cand_sum;
        if (wd.scale_weight > 0) {
            double r;
            scale_regulariser(P + 7 * (size_t)(wd.kf_off + wd.scale_kf1), P + 7 * (size_t)(wd.kf_off + wd.scale_kf0),
                              wd.scale_value, r, nullptr, nullptr);
            cand += 0.5 * wd.scale_weight * r * r;
        }
        if (wd.speed_weight > 0) {
            double r[3];
            speed_regulariser(P + 7 * (size_t)(wd.kf_off + wd.speed_kf), wd.speed_T_origin_before, wd.speed_v_before, wd.speed_dt, r,
                              nullptr);
            cand += 0.5 * wd.speed_weight * (r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
        }
        if (has_gp) cand += *gp_cost;
        if (wd.plane_reg_weight > 0 && wd.n_kf > 1) cand += plane_chain_cost(wd, P, PL);
        return cand;
    });
}

// =====================================================================================================================
// trimming (reference robust_solving.cpp:67-125, trimmer_quantile.hpp:40-63)
// =====================================================================================================================
// per-landmark maximum of the un-robustified block norms, per residual group (0 depth, 1 reprojection, 2 ground plane)
__global__ void __launch_bounds__(256) k_trim_eval(BatchDev bd) {
    const int w = blockIdx.y;
    const WinState& st = bd.state[w];
    if (st.phase != PH_TRIM) return;
    const WinDesc& wd = bd.desc[w];
    const SolveParams& sp = bd.wsp[w];
    __shared__ double s_pose[kMaxKf * kPoseStride];
    __shared__ double s_cam[kMaxCam * kCamStride];
    stage_window(wd, bd.pose[st.cur], bd.cam, s_pose, s_cam);
    __syncthreads();
    const int lane = threadIdx.x & 31;
    // 64 landmarks per CTA (8 rounds of one landmark per warp): the kernel is launched in every pass and idles in all but the one or
    // two trimming passes of a solve, so its idle launch over a large batch should be few CTAs
    for (int it = 0; it < 8; ++it) {
    const int j = (blockIdx.x * 8 + it) * 8 + (threadIdx.x >> 5);
    if (j >= wd.n_lm) continue;
    const int L = wd.lm_off + j;
    double m_d = -1.0, m_r = -1.0;
    if (bd.lm_active[L]) {
        const int* lm_ptr = bd.lm_ptr + wd.lm_off + w;
        const double* lm = bd.lm[st.cur] + 3 * (size_t)L;
        const double p[3] = {lm[0], lm[1], lm[2]};
        for (int o = lm_ptr[j] + lane; o < lm_ptr[j + 1]; o += 32) {
            const size_t oo = (size_t)wd.obs_off + o;
            double r[3], raw[2], hr;
            if (!eval_observation<double, false>(s_pose + kPoseStride * bd.obs_kf[oo], s_cam + kCamStride * bd.obs_cam[oo],
                                                 p, (double)bd.obs_u[oo], (double)bd.obs_v[oo], (double)bd.obs_d[oo],
                                                 bd.lm_weight[L], sp.reprojection_thres * sp.reprojection_thres,
                                                 sp.depth_thres * sp.depth_thres, r, nullptr, nullptr, hr, raw))
                continue;
            m_r = fmax(m_r, raw[0]);
            m_d = fmax(m_d, raw[1]);
        }
        m_r = warp_max(m_r);
        m_d = warp_max(m_d);
    }
    if (lane == 0) {
        bd.trim_val[0 * (size_t)bd.tot_lm + L] = m_d;
        bd.trim_val[1 * (size_t)bd.tot_lm + L] = m_r;
        double m_g = -1.0;  // ground-plane group: |n . (R p + t) + dist| of the landmark's gp block
        const int gl = (wd.n_gp > 0 && bd.lm_active[L]) ? bd.gp_of_lm[L] : -1;
        if (gl >= 0) {
            const int k = bd.gp_kf[wd.gp_off + gl];
            const double* ps = s_pose + kPoseStride * k;
            const double* pl = bd.plane[st.cur] + 4 * (size_t)(wd.kf_off + k);
            const double* lm = bd.lm[st.cur] + 3 * (size_t)L;
            double px[3];
            for (int i = 0; i < 3; ++i) px[i] = ps[3 * i] * lm[0] + ps[3 * i + 1] * lm[1] + ps[3 * i + 2] * lm[2] + ps[9 + i];
            m_g = fabs(pl[0] * px[0] + pl[1] * px[1] + pl[2] * px[2] + pl[3]);
        }
        bd.trim_val[2 * (size_t)bd.tot_lm + L] = m_g;
    }
    }
}

// quantile rejection per group by exact rank (ties broken by landmark index, trim_select_group), then start the next solve
__global__ void __launch_bounds__(512) k_trim_select(BatchDev bd) {
    const int w = blockIdx.x;
    const SolveParams& sp = bd.wsp[w];
    WinState& st = bd.state[w];
    if (st.phase != PH_TRIM) return;
    const WinDesc& wd = bd.desc[w];
    __shared__ TrimSmem s_trim;
    const double quant[3] = {sp.depth_quantile, sp.reprojection_quantile, sp.gp_quantile};
    // sharded window: the values of ALL ranks' landmarks (k_shard_trim_scatter + all-reduce), indexed by the caller's
    // window-wide landmark index, stored as v + 2; every rank takes the same decisions and applies them to its own block
    const bool sh = bd.sharded != 0;
    const int n_items = sh ? bd.lm_total : wd.n_lm;
    const int* orig = bd.lm_orig + wd.lm_off;  // ties are broken by the caller's landmark index
    auto oid = [&](int j) { return sh ? j : orig[j]; };
    uint8_t* rej = sh ? bd.reject_glob : bd.trim_reject + wd.lm_off;
    for (int j = threadIdx.x; j < n_items; j += blockDim.x) rej[j] = 0;
    for (int g = 0; g < 3; ++g) {
        const double* vbase = sh ? bd.trim_glob + g * (size_t)bd.lm_total : bd.trim_val + g * (size_t)bd.tot_lm + wd.lm_off;
        const double voff = sh ? 2.0 : 0.0;
        auto val = [&](int j) { return vbase[j] - voff; };
        trim_select_group(s_trim, n_items, quant[g], sp.min_residual_groups, val, oid, rej);
    }
    __syncthreads();
    for (int j = threadIdx.x; j < wd.n_lm; j += blockDim.x)
        if (rej[sh ? bd.lm_begin + orig[j] : j]) bd.lm_active[wd.lm_off + j] = 0;
    if (sh && bd.shard_gp)  // the same decisions for the whole window: which ground points still hold plane blocks (k_solve_begin)
        for (int j = threadIdx.x; j < bd.lm_total; j += blockDim.x)
            if (rej[j]) bd.act_glob[j] = 0;
    __syncthreads();
    if (threadIdx.x == 0) trim_advance(st);
}

__global__ void k_count_active(BatchDev bd) {
    const int w = blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= bd.n_win) return;
    if (bd.state[w].phase != PH_DONE) atomicAdd(bd.n_active, 1);
}

// reset of the solver state from the uploaded values
__global__ void k_reset_state(BatchDev bd) {
    const int w = blockIdx.x;
    const WinDesc& wd = bd.desc[w];
    for (int i = threadIdx.x; i < wd.n_kf * 7; i += blockDim.x) {
        const double v = bd.pose0[(size_t)wd.kf_off * 7 + i];
        bd.pose[0][(size_t)wd.kf_off * 7 + i] = v;
        bd.pose[1][(size_t)wd.kf_off * 7 + i] = v;
    }
    for (int k = threadIdx.x; k < wd.n_kf; k += blockDim.x) {
        double rt12[kPoseStride];
        write_rt(rt12, bd.pose0 + 7 * (size_t)(wd.kf_off + k));
        for (int i = 0; i < kPoseStride; ++i) {
            bd.rt[0][kPoseStride * (size_t)(wd.kf_off + k) + i] = rt12[i];
            bd.rt[1][kPoseStride * (size_t)(wd.kf_off + k) + i] = rt12[i];
        }
    }
    for (int i = threadIdx.x; i < wd.n_kf * 4; i += blockDim.x) {
        const double v = bd.plane0[(size_t)wd.kf_off * 4 + i];
        bd.plane[0][(size_t)wd.kf_off * 4 + i] = v;
        bd.plane[1][(size_t)wd.kf_off * 4 + i] = v;
    }
    for (int i = threadIdx.x; i < wd.n_lm * 3; i += blockDim.x) {
        const double v = bd.lm0[(size_t)wd.lm_off * 3 + i];
        bd.lm[0][(size_t)wd.lm_off * 3 + i] = v;
        bd.lm[1][(size_t)wd.lm_off * 3 + i] = v;
    }
    for (int i = threadIdx.x; i < wd.n_lm; i += blockDim.x) bd.lm_active[wd.lm_off + i] = 1;
    if (bd.sharded && bd.shard_gp)
        for (int j = threadIdx.x; j < bd.lm_total; j += blockDim.x) bd.act_glob[j] = 1;
    if (threadIdx.x == 0) {
        WinState& st = bd.state[w];
        st.phase = wd.idle ? PH_DONE : PH_SOLVE_BEGIN;  // an idle window (kba_track_group_solve) never iterates: no solve, no log
        st.cur = 0;
        st.solve_index = 0; st.round = 0; st.retried = 0; st.log_n = 0; st.n_solves = 0;
        const SolveParams& sp = bd.wsp[w];
        int rounds = sp.rounds_override;
        if (rounds < 0) rounds = ((bd.sharded ? bd.lm_total : wd.n_lm) > sp.min_landmarks_for_trimming) ? sp.num_rounds_option : 0;
        if (rounds > 6) rounds = 6;
        st.rounds_total = rounds;
        st.is_final = (rounds == 0);
        st.eval_failed = 0; st.solve_failed = 0;
    }
}

// =====================================================================================================================
// launch wrappers
// =====================================================================================================================
int launch_check_enabled() {
    static const int on = [] { const char* e = getenv("KBA_LAUNCH_CHECK"); return (e && e[0] == '1') ? 1 : 0; }();
    return on;
}
static cudaError_t g_launch_check_first = cudaSuccess;
void launch_check_report(const char* kernel, cudaError_t e) {
    if (g_launch_check_first == cudaSuccess) fprintf(stderr, "[kba] launch of %s failed: %s\n", kernel, cudaGetErrorString(e));
    g_launch_check_first = e;
}
static inline size_t schur_smem() { return (size_t)2 * kKC * kGS * sizeof(double); }
static inline size_t schur_tma_smem() { return (size_t)2 * kStageDoubles * sizeof(double); }
static inline size_t solve_smem(int ld) { return ((size_t)5 * ld + kNB + kNB * (kNB + 1) + (size_t)(ld + 8) * kPanelStride) * sizeof(double); }
static inline size_t trail_smem(int ld) { return (size_t)(ld + 8) * kPanelStride * sizeof(double); }
// stages 1 and 2 of k_reduced_solve<false> never touch the panel copy: all that grows with the rows above kPanelMaxRows
static inline size_t solve_stage_smem(int ld) { return ((size_t)5 * ld + kNB + kNB * (kNB + 1)) * sizeof(double); }
static inline size_t solve_tiled_smem(int ld) {
    const int nt = ld / 8;
    return ((size_t)5 * ld + kNB + kNB * (kNB + 1) + (size_t)nt * (nt + 1) / 2 * 64) * sizeof(double);
}

// Opt-in dynamic shared memory of the solve kernels.  The attribute is per function (per device), not per batch: a later,
// smaller batch must never lower what an earlier, larger batch still launches with (a persistent window next to one-shot
// solves did exactly that: "invalid argument" at the next launch) -- so the sizes only ever grow, per device.
cudaError_t configure_kernels(int nr_cap_max) {
    static int hi_tiled[64] = {0}, hi_rows[64] = {0};
    static size_t hi_solve[64] = {0};
    static bool fixed_done[64] = {false};
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    dev &= 63;
    if (!fixed_done[dev]) {
        e = cudaFuncSetAttribute(k_schur_syrk, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)schur_smem());
        if (e != cudaSuccess) return e;
        e = cudaFuncSetAttribute(k_schur_syrk_tma, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)schur_tma_smem());
        if (e != cudaSuccess) return e;
        e = cudaFuncSetAttribute(k_schur_fused<6>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)schur_fused_smem());
        if (e != cudaSuccess) return e;
        e = cudaFuncSetAttribute(k_schur_fused<7>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)schur_fused_smem());
        if (e != cudaSuccess) return e;
        fixed_done[dev] = true;
    }
    if (nr_cap_max <= kTiledMaxRows && nr_cap_max > hi_tiled[dev]) {
        e = cudaFuncSetAttribute(k_reduced_solve<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)solve_tiled_smem(nr_cap_max));
        if (e != cudaSuccess) return e;
        hi_tiled[dev] = nr_cap_max;
    }
    // above kPanelMaxRows: k_chol_trail is not launched, and k_reduced_solve<false> runs stages 1 and 2 only
    if (nr_cap_max <= kPanelMaxRows && nr_cap_max > hi_rows[dev]) {
        e = cudaFuncSetAttribute(k_chol_trail, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)trail_smem(nr_cap_max));
        if (e != cudaSuccess) return e;
        hi_rows[dev] = nr_cap_max;
    }
    const size_t solve = nr_cap_max <= kPanelMaxRows ? solve_smem(nr_cap_max) : solve_stage_smem(nr_cap_max);
    if (solve > hi_solve[dev]) {
        e = cudaFuncSetAttribute(k_reduced_solve<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)solve);
        if (e != cudaSuccess) return e;
        hi_solve[dev] = solve;
    }
    return cudaSuccess;
}

// grid.x of a kernel whose CTAs stride over a window's units (k_linearize: 8 warp tiles, k_backsub_v: 16 landmarks).  Every pass is
// launched for every window of the batch and the unit count is an upper bound, so with one CTA per unit most CTAs of a large batch
// only find out that they have nothing to do; num/den of the units per window come from a sweep on the headline workload
// (k_linearize: 1/8, k_backsub_v: 1/3; any grid gives bit-identical results), as long as the strided grid still fills `waves` waves
// of the kernel's resident CTAs (k_linearize: six of three CTAs per SM -- a batch of 64 config-2 windows strides; k_backsub_v: eight
// of two): a CTA then runs several units back to back, and the last, partly filled wave stays a small share of the launch.  Smaller
// batches keep one CTA per unit (latency: every SM busy).
// `cfg`: -1 = this rule, 0 = one CTA per unit, > 0 = that many (KBA_LIN_GRID / KBA_BS_GRID).
static int strided_grid(int cfg, int n_units, int num, int den, int n_win, int sm_count, int ctas_per_sm, int waves) {
    if (cfg == 0) return n_units;
    if (cfg > 0) return cfg < n_units ? cfg : n_units;
    const int g = (n_units * num + den - 1) / den;
    return ((long long)g * n_win >= (long long)waves * ctas_per_sm * sm_count && g >= 1) ? g : n_units;
}

int launch_shard_gather(const BatchDev& bd, const LaunchCfg& lc, cudaStream_t s) {
    if (!bd.sharded || !bd.shard_gp) return 0;
    cudaMemsetAsync(bd.gp_send, 0, sizeof(double) * (size_t)bd.lm_total, s);
    if (bd.tot_gp > 0) k_shard_gp_gather<<<(unsigned)((bd.tot_gp + 255) / 256), 256, 0, s>>>(bd);
    LCHK("k_shard_gp_gather");
    return lc.xchg.allreduce(lc.xchg.user, bd.gp_send, bd.gp_kf_glob, bd.lm_total, 0, s);
}

void launch_reset(const BatchDev& bd, const LaunchCfg& lc, cudaStream_t s) {
    k_reset_state<<<bd.n_win, 256, 0, s>>>(bd); LCHK("k_reset_state");
}

int launch_pass(const BatchDev& bd, const LaunchCfg& lc, Counters* cnt, cudaStream_t s) {
    const int B = bd.n_win;
    const dim3 g_obs((bd.max_obs + 255) / 256, B);
    const dim3 g_lm((bd.max_lm + 63) / 64, B);
    if (!bd.fused) k_panel_zero<<<dim3(64, B), 256, 0, s>>>(bd);  // the fused path has no global V panels
    LCHK("k_panel_zero");
    if (bd.sharded && bd.shard_gp) k_shard_planes<<<1, 256, 0, s>>>(bd);
    LCHK("k_shard_planes");
    k_solve_begin<<<B, kBeginThreads, 0, s>>>(bd); LCHK("k_solve_begin");
    const bool timed = lc.time_jacobian && lc.ev_pool && *lc.ev_used + 2 <= lc.ev_cap;
    // one-kernel linearisation (kba_linearize.cuh): fused path, FP64, at most one observation per (landmark, keyframe)
    const bool lin1 = bd.lin1 != 0;
    if (lin1) {
        if (bd.tot_gp > 0) {
            k_gp_eval<true><<<B, 256, 0, s>>>(bd);
            k_gp_blocks<<<dim3((bd.max_kf + 7) / 8, B), 256, 0, s>>>(bd);
        }
        LCHK("k_gp_eval");
        if (timed) cudaEventRecord(lc.ev_pool[(*lc.ev_used)++], s);
        const int n_units = (lin_tile_bound(bd.max_obs, bd.max_lm) + kLinWarps - 1) / kLinWarps;
        const dim3 g_lin(strided_grid(lc.knobs.lin_grid, n_units, 1, 8, B, lc.sm_count, kLinMinBlocks, 6), B);  // CTAs of a window stride over its units
        if ((int)g_lin.x < n_units) k_linearize<true><<<g_lin, kLinThreads, 0, s>>>(bd, n_units);
        else k_linearize<false><<<g_lin, kLinThreads, 0, s>>>(bd, n_units);
        LCHK("k_linearize");
        if (timed) cudaEventRecord(lc.ev_pool[(*lc.ev_used)++], s);
        k_pose_hessian<<<dim3(bd.max_kf, B), 256, 0, s>>>(bd); LCHK("k_pose_hessian");
    } else {
        if (timed) cudaEventRecord(lc.ev_pool[(*lc.ev_used)++], s);
        launch_eval_obs<true>(bd, s);
        if (timed) cudaEventRecord(lc.ev_pool[(*lc.ev_used)++], s);
        if (bd.tot_gp > 0) {
            k_gp_eval<true><<<B, 256, 0, s>>>(bd);
            k_gp_blocks<<<dim3((bd.max_kf + 7) / 8, B), 256, 0, s>>>(bd);
        }
        LCHK("k_gp_eval");
        k_pose_hessian<<<dim3(bd.max_kf, B), 256, 0, s>>>(bd); LCHK("k_pose_hessian");
    }
    if (bd.fused) {
        if (!lin1) {
            k_landmark_reduce<true><<<dim3((bd.max_lm + 15) / 16, B), 256, 0, s>>>(bd); LCHK("k_landmark_reduce");
            k_obs_v2<<<g_obs, 256, 0, s>>>(bd); LCHK("k_obs_v2");
        }
        const dim3 gf(bd.p_split, B);
        if (lc.plan.fused_slots == 7) k_schur_fused<7><<<gf, 512, schur_fused_smem(), s>>>(bd);
        else k_schur_fused<6><<<gf, 512, schur_fused_smem(), s>>>(bd);
        LCHK("k_schur_fused");
    } else {
        k_landmark_reduce<false><<<dim3((bd.max_lm + 15) / 16, B), 256, 0, s>>>(bd); LCHK("k_landmark_reduce");
        for (int round = 0; round <= lc.max_rank; ++round) k_obs_v<<<g_obs, 256, 0, s>>>(bd, round);
        LCHK("k_obs_v");
        if (bd.tot_gp > 0) k_gp_panel<<<dim3((bd.max_gp * 10 + 255) / 256, B), 256, 0, s>>>(bd);
        LCHK("k_gp_panel");
    }
    if (bd.fused) {
    } else if (lc.plan.small_syrk) {
        k_schur_syrk_tma<<<dim3(bd.p_split, B), 512, schur_tma_smem(), s>>>(bd); LCHK("k_schur_syrk_tma");
    } else {
        const int nb = lc.plan.nr_cap_max / 64;
        k_schur_syrk<<<dim3(nb * (nb + 1) / 2, bd.p_split, B), 256, schur_smem(), s>>>(bd); LCHK("k_schur_syrk");
    }
    const dim3 g_red((lc.plan.nr_cap_max * lc.plan.nr_cap_max + 255) / 256, B);
    BatchDev bc = bd;  // consumer view of the reduced system
    if (bd.sharded) {
        // the one exchange of the linearisation: reduced system (Schur sums + right-hand side), pose blocks, ground-plane blocks and
        // cost, cost at x
        if (bd.p_split > 1) k_sred_reduce<<<g_red, 256, 0, s>>>(bd, 1);
        LCHK("k_sred_reduce");
        const LaunchCfg::WinDescHost& wh = lc.shard_win;
        const long long n_s = (long long)wh.nr_cap * wh.nr_cap, n_b = (long long)wh.n_kf * 27, n_g = shard_gp_doubles(bd.shard_gp, wh.n_kf);
        const long long n_x = n_s + n_b + n_g + bd.shard_cost_parts + 2;
        k_shard_pack<<<(unsigned)((n_x + 255) / 256), 256, 0, s>>>(bd); LCHK("k_shard_pack");
        if (int rc = lc.xchg.allreduce(lc.xchg.user, bd.x_send, bd.x_recv, n_x, 0, s)) return rc;
        k_shard_flags<<<1, 32, 0, s>>>(bd); LCHK("k_shard_flags");
        // the solve reads the window-wide sums
        bc.sred = bd.x_recv; bc.bkf = bd.x_recv + n_s; bc.cost_part_x = bd.x_recv + n_s + n_b + n_g; bc.cost_parts = bd.shard_cost_parts;
        if (n_g) { bc.gp_kfb = bd.x_recv + n_s + n_b; bc.gp_cost_x = bd.x_recv + n_s + n_b + 65LL * wh.n_kf; }
        k_sred_reduce<<<g_red, 256, 0, s>>>(bc, 2); LCHK("k_sred_reduce");
    } else if (bd.p_split > 1 || bd.solve_banded) {  // banded: A = -Sred by the whole GPU, not by stage 1's one CTA
        k_sred_reduce<<<g_red, 256, 0, s>>>(bd, 0); LCHK("k_sred_reduce");
    }
    if (bd.solve_tiled) {
        k_reduced_solve<true><<<B, 512, solve_tiled_smem(lc.plan.nr_cap_max), s>>>(bc, 0); LCHK("k_reduced_solve");
    } else if (!bd.solve_split) {
        k_reduced_solve<false><<<B, 512, solve_smem(lc.plan.nr_cap_max), s>>>(bc, 0); LCHK("k_reduced_solve");
    } else {  // few large windows, or any above kPanelMaxRows: the factorisation is spread over the GPU, one 32-column block at a time
        const bool banded = bd.solve_banded != 0;
        const size_t stage_smem = banded ? solve_stage_smem(lc.plan.nr_cap_max) : solve_smem(lc.plan.nr_cap_max);
        k_reduced_solve<false><<<B, 512, stage_smem, s>>>(bc, 1); LCHK("k_reduced_solve");
        const int strips = (lc.plan.nr_cap_max + 7) / 8;
        for (int kb = 0; kb < lc.plan.nr_cap_max; kb += kNB) {
            k_chol_diag<<<B, 32, 0, s>>>(bc, kb); LCHK("k_chol_diag");
            k_chol_panel<<<dim3((strips + 15) / 16, B), 512, 0, s>>>(bc, kb); LCHK("k_chol_panel");
            if (banded) k_chol_trail_band<<<dim3(bd.solve_split, B), 256, 0, s>>>(bc, kb);
            else k_chol_trail<<<dim3(bd.solve_split, B), 512, trail_smem(lc.plan.nr_cap_max), s>>>(bc, kb);
            LCHK("k_chol_trail");
        }
        k_reduced_solve<false><<<B, 512, stage_smem, s>>>(bc, 2); LCHK("k_reduced_solve");
    }
    if (bd.fused) {
        const int n_units = (bd.max_lm + 15) / 16;
        const int gx = strided_grid(lc.knobs.bs_grid, n_units, 1, 3, B, lc.sm_count, 2, 8);
        if (gx < n_units) k_backsub_v<true><<<dim3(gx, B), 256, 0, s>>>(bd, n_units);
        else k_backsub_v<false><<<dim3(n_units, B), 256, 0, s>>>(bd, n_units);
    }
    else k_backsub<<<dim3((bd.max_lm + 15) / 16, B), 256, 0, s>>>(bd);
    LCHK("k_backsub");
    launch_eval_obs<false>(bd, s);
    if (bd.tot_gp > 0) k_gp_eval<false><<<B, 256, 0, s>>>(bd);
    LCHK("k_gp_eval");
    if (bd.sharded) {  // model decrease / step norm / candidate cost over all ranks
        k_shard_scalars<<<1, 32, 0, s>>>(bd); LCHK("k_shard_scalars");
        // model decrease, step / state norms, candidate cost, failure flag (sums) and one gradient-max slot per rank
        if (int rc = lc.xchg.allreduce(lc.xchg.user, bd.xs, bd.xs, 16 + bd.shard_world, 0, s)) return rc;
    }
    k_lm_update<<<(B * 32 + 127) / 128, 128, 0, s>>>(bd); LCHK("k_lm_update");
    k_trim_eval<<<g_lm, 256, 0, s>>>(bd); LCHK("k_trim_eval");
    if (bd.sharded) {  // quantiles are taken over the landmarks of all ranks
        k_shard_trim_scatter<<<(bd.max_lm + 255) / 256, 256, 0, s>>>(bd); LCHK("k_shard_trim_scatter");
        if (int rc = lc.xchg.allreduce(lc.xchg.user, bd.trim_send, bd.trim_glob, 3LL * bd.lm_total, 0, s)) return rc;
    }
    k_trim_select<<<B, 512, 0, s>>>(bd); LCHK("k_trim_select");
    if (cnt) {
        const int gp = bd.tot_gp > 0 ? 1 : 0;
        const int prep = lin1 ? 1 : 2 + (bd.fused ? 1 : lc.max_rank + 1 + gp);  // pose blocks [, landmark blocks, V rows]
        cnt->launches_total += gp; cnt->launches_prep += gp;                       // k_gp_blocks
        if (bd.sharded && bd.shard_gp) cnt->launches_total += 1;                   // k_shard_planes
        const int split = (!bd.solve_tiled && bd.solve_split) ? 1 + 3 * ((lc.plan.nr_cap_max + kNB - 1) / kNB) : 0;
        cnt->launches_total += (bd.fused ? 0 : 1) + 1 + 1 + gp + prep + 1 + (bd.p_split > 1 || bd.solve_banded ? 1 : 0) + 1 + split + 1 + 1 + gp + 1 + 2;
        cnt->launches_jacobian += 1; cnt->launches_prep += prep + gp; cnt->launches_schur += 1; cnt->launches_solve += 2;
        cnt->launches_backsub += 1; cnt->launches_cost += 1 + gp; cnt->launches_update += 1; cnt->launches_trim += 2;
    }
    return 0;
}

void launch_count_active(const BatchDev& bd, cudaStream_t s) {
    cudaMemsetAsync(bd.n_active, 0, sizeof(int), s);
    k_count_active<<<(bd.n_win + 127) / 128, 128, 0, s>>>(bd); LCHK("k_count_active");
}

// Loop condition of the device-driven solve (kba_api.cu: the pass sequence is the body of a conditional WHILE node of a CUDA
// graph).  Last kernel of the body: any window not done and the pass cap not reached -> run the body again.  The host launches the
// graph once per solve and is not involved until every window has finished.
__global__ void __launch_bounds__(256) k_loop_cond(BatchDev bd, cudaGraphConditionalHandle handle, int* pass, int max_passes) {
    int active = 0;
    for (int w = threadIdx.x; w < bd.n_win; w += blockDim.x) active += (bd.state[w].phase != PH_DONE) ? 1 : 0;
    active = __syncthreads_count(active > 0);  // threads that saw an unfinished window (the host only tests for zero)
    if (threadIdx.x == 0) {
        const int p = *pass + 1;
        *pass = p;
        *bd.n_active = active;
        cudaGraphSetConditional(handle, (active > 0 && p < max_passes) ? 1u : 0u);
    }
}
void launch_loop_cond(const BatchDev& bd, unsigned long long handle, int* pass, int max_passes, cudaStream_t s) {
    k_loop_cond<<<1, 256, 0, s>>>(bd, (cudaGraphConditionalHandle)handle, pass, max_passes);
}

// stand-alone residual/Jacobian pass at the uploaded state (parity + roofline measurement)
__global__ void k_force_linearize(BatchDev bd) {
    const int w = blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= bd.n_win) return;
    WinState& st = bd.state[w];
    st.phase = PH_ITERATE; st.need_linearize = 1; st.iter0 = 1; st.cur = 0; st.eval_failed = 0; st.solve_failed = 0;
}
void launch_jacobian_only(const BatchDev& bd, cudaStream_t s) {
    launch_eval_obs<true>(bd, s);
}
// inspection entry point (kba_eval) on the fused path: J_l of every observation, formed exactly as the consumers of the
// linearisation form it -- translation columns of the materialised J_p times the staged rotation of the keyframe, in FP64
// whatever precision J_p is stored in (precision 1: FP32 J_p, widened, times the FP64 rotation; the product is not rounded)
template <typename TLin>
__global__ void k_expand_jl(BatchDev bd, double* out) {
    const WinDesc& wd = bd.desc[0];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= wd.n_obs) return;
    const size_t o = (size_t)wd.obs_off + i, T = (size_t)bd.tot_obs;
    const double* R = bd.rt[0] + kPoseStride * (size_t)(wd.kf_off + bd.obs_kf[o]);
    const TLin* jp = reinterpret_cast<const TLin*>(bd.jp);
    for (int r = 0; r < 3; ++r) {
        const double m0 = (double)jp[(6 * r + 3) * T + o], m1 = (double)jp[(6 * r + 4) * T + o], m2 = (double)jp[(6 * r + 5) * T + o];
        for (int c = 0; c < 3; ++c) out[(size_t)(3 * r + c) * T + o] = m0 * R[c] + m1 * R[3 + c] + m2 * R[6 + c];
    }
}
void launch_expand_jl(const BatchDev& bd, double* out, cudaStream_t s) {
    const int n = (int)bd.tot_obs;
    if (bd.precision) k_expand_jl<float><<<(n + 255) / 256, 256, 0, s>>>(bd, out);
    else k_expand_jl<double><<<(n + 255) / 256, 256, 0, s>>>(bd, out);
    LCHK("k_expand_jl");
}
void launch_force_linearize(const BatchDev& bd, cudaStream_t s) {
    k_solve_begin<<<bd.n_win, kBeginThreads, 0, s>>>(bd); LCHK("k_solve_begin");  // layout (off_pose) for the eval entry point
    k_force_linearize<<<(bd.n_win + 127) / 128, 128, 0, s>>>(bd); LCHK("k_force_linearize");
}

}  // namespace kba
