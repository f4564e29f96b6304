// kba_evaluate.cu -- evaluation of stored windows at the store's state (kba_track_evaluate / kba_track_group_evaluate): the raw
// residual rows, robust losses and trimming values of every observation and landmark, the trimming decisions, the attached
// ground-plane residuals and the cost parts.  The kernels read the window the gather of kba_pack.cu builds for a solve (its raw,
// caller-ordered CSR and the gathered poses, planes and positions), so the window is the solve's array for array; every value
// comes from the solver's own device functions (eval_observation, cauchy, gp_height, gp_huber, scale_regulariser,
// plane_chain_cost, trim_select_group).  Nothing is written back: the store stays as it is.
#include <cfloat>
#include <cmath>

#include "kba_device.cuh"
#include "kba_kernels.h"
#include "kba_regularisers.cuh"
#include "kba_controller.cuh"

namespace kba {

constexpr int kEvLmPerCta = 64;  // 8 warps x 8 landmarks: one cost partial per CTA

// One warp per landmark of window blockIdx.y, its lanes over the landmark's observations.  Per observation: the raw rows
// (eval_observation with unit weight and an infinite Cauchy scale, whose sqrt(rho') is exactly 1, so its rows are the residuals
// before any loss or weight), the scaled Cauchy losses of its reprojection and depth blocks at the options' scales, and its raw
// block norms; per landmark the maxima of those norms (k_trim_eval's values); per CTA the two cost sums and the failure flag.
__global__ void __launch_bounds__(256) k_ev_obs(BatchDev bd, PackRaw raw, const EvalWin* wins, EvalOut o) {
    const int w = blockIdx.y;
    const WinDesc& wd = bd.desc[w];
    if (wd.idle || blockIdx.x * kEvLmPerCta >= wd.n_lm) return;
    const EvalWin& ew = wins[w];
    const SolveParams& sp = bd.wsp[w];
    __shared__ double s_pose[kMaxKf * kPoseStride];
    __shared__ double s_cam[kMaxCam * kCamStride];
    __shared__ double s_red[8][3];
    stage_window(wd, bd.pose0, bd.cam, s_pose, s_cam);
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const double b_repr = sp.reprojection_thres * sp.reprojection_thres, b_depth = sp.depth_thres * sp.depth_thres;
    const int* lp = raw.lm_ptr + wd.lm_off + w;
    double c_repr = 0.0, c_depth = 0.0, failed = 0.0;
    for (int it = 0; it < 8; ++it) {
        const int j = (blockIdx.x * 8 + it) * 8 + warp;
        if (j >= wd.n_lm) break;
        const size_t L = (size_t)wd.lm_off + j;
        const double p[3] = {raw.lm_pos[3 * L], raw.lm_pos[3 * L + 1], raw.lm_pos[3 * L + 2]};
        const double wt = raw.lm_weight[L];
        double m_r = -1.0, m_d = -1.0;
        for (int q = lp[j] + lane; q < lp[j + 1]; q += 32) {
            const size_t oo = (size_t)wd.obs_off + q;
            const int k = raw.obs_kf[oo], c = raw.obs_cam[oo];
            const double d = (double)raw.obs_d[oo];
            double r[3], rb[2], hr;
            const bool ok = eval_observation<double, false, false>(s_pose + kPoseStride * k, s_cam + kCamStride * c, p,
                                                                   (double)raw.obs_u[oo], (double)raw.obs_v[oo], d, 1.0, HUGE_VAL,
                                                                   HUGE_VAL, r, nullptr, nullptr, hr, rb);
            const size_t e = (size_t)ew.obs0 + q;
            o.obs_lm[e] = j; o.obs_kf[e] = k; o.obs_cam[e] = c;
            if (!ok) {  // |z_cam| < 0.01: the solver's evaluation fails (cost_functors_ceres.hpp:78-83)
                failed = 1.0;
                for (int i = 0; i < 3; ++i) o.res[3 * e + i] = NAN;
                o.rho[2 * e] = NAN; o.rho[2 * e + 1] = NAN;
                continue;
            }
            double h_r, h_d = 0.0, sq;
            cauchy<double>(b_repr, wt, r[0] * r[0] + r[1] * r[1], h_r, sq);
            if (d > 0.0) cauchy<double>(b_depth, wt, r[2] * r[2], h_d, sq);
            for (int i = 0; i < 3; ++i) o.res[3 * e + i] = r[i];
            o.rho[2 * e] = 2.0 * h_r; o.rho[2 * e + 1] = 2.0 * h_d;
            c_repr += h_r; c_depth += h_d;
            m_r = fmax(m_r, rb[0]);
            m_d = fmax(m_d, rb[1]);
        }
        m_r = warp_max(m_r);
        m_d = warp_max(m_d);
        if (lane == 0) { o.trim[ew.lm0 + j] = m_r; o.trim[(size_t)ew.n_lm_total + ew.lm0 + j] = m_d; }
    }
    c_repr = warp_sum(c_repr); c_depth = warp_sum(c_depth); failed = warp_max(failed);
    if (lane == 0) { s_red[warp][0] = c_repr; s_red[warp][1] = c_depth; s_red[warp][2] = failed; }
    __syncthreads();
    if (threadIdx.x < 3) {  // fixed order over the warps: a window's partials do not depend on the batch it is evaluated in
        double s = 0.0;
        for (int q = 0; q < 8; ++q) s = threadIdx.x == 2 ? fmax(s, s_red[q][2]) : s + s_red[q][threadIdx.x];
        o.part[3 * ((size_t)ew.part0 + blockIdx.x) + threadIdx.x] = s;
    }
}

// One CTA per window: the attached ground-plane residuals, the regularisers, the cost parts and the quantile trimming of the
// reprojection and depth groups (TrimmerQuantile at the options' quantiles, ties broken by landmark index as k_trim_select does).
__global__ void __launch_bounds__(512) k_ev_finish(BatchDev bd, PackRaw raw, const EvalWin* wins, EvalOut o) {
    const int w = blockIdx.x;
    const WinDesc& wd = bd.desc[w];
    if (wd.idle) return;
    const EvalWin& ew = wins[w];
    const SolveParams& sp = bd.wsp[w];
    __shared__ TrimSmem s_trim;
    __shared__ double s_red[16];
    double c_gp = 0.0;
    for (int g = threadIdx.x; g < wd.n_gp; g += blockDim.x) {
        const size_t G = (size_t)wd.gp_off + g, e = (size_t)ew.gp0 + g;
        const int j = raw.gp_lm[G], k = bd.gp_kf[G];
        double R[9], a[3], px[3], rho, rho1;
        const double r = gp_height(bd.pose0 + 7 * ((size_t)wd.kf_off + k), bd.plane0 + 4 * ((size_t)wd.kf_off + k),
                                   raw.lm_pos + 3 * ((size_t)wd.lm_off + j), R, a, px);
        gp_huber(r * r, sp.gp_huber, rho, rho1);
        c_gp += 0.5 * bd.gp_weight[G] * rho;
        o.gp_lm[e] = j; o.gp_kf[e] = k; o.gp_w[e] = bd.gp_weight[G]; o.gp_r[e] = r;
    }
    c_gp = warp_sum(c_gp);
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = c_gp;
    // trimming: the decisions of each group start from "kept"
    const int n = wd.n_lm;
    unsigned char* rej_r = o.rej + ew.lm0, *rej_d = o.rej + (size_t)ew.n_lm_total + ew.lm0;
    for (int j = threadIdx.x; j < n; j += blockDim.x) { rej_r[j] = 0; rej_d[j] = 0; }
    __syncthreads();
    const double* t_r = o.trim + ew.lm0, *t_d = o.trim + (size_t)ew.n_lm_total + ew.lm0;
    auto oid = [](int j) { return j; };  // the window's landmarks are in the caller's order
    trim_select_group(s_trim, n, sp.depth_quantile, sp.min_residual_groups, [t_d](int j) { return t_d[j]; }, oid, rej_d);
    trim_select_group(s_trim, n, sp.reprojection_quantile, sp.min_residual_groups, [t_r](int j) { return t_r[j]; }, oid, rej_r);
    if (threadIdx.x != 0) return;
    double c_repr = 0.0, c_depth = 0.0, failed = 0.0, gp = 0.0;
    for (int q = 0; q < ew.n_part; ++q) {
        const double* p = o.part + 3 * ((size_t)ew.part0 + q);
        c_repr += p[0]; c_depth += p[1]; failed = fmax(failed, p[2]);
    }
    for (int q = 0; q < (int)(blockDim.x >> 5); ++q) gp += s_red[q];
    double scale = 0.0, chain = 0.0;
    if (wd.scale_weight > 0) {
        double r;
        scale_regulariser(bd.pose0 + 7 * (size_t)(wd.kf_off + wd.scale_kf1), bd.pose0 + 7 * (size_t)(wd.kf_off + wd.scale_kf0),
                          wd.scale_value, r, nullptr, nullptr);
        scale = 0.5 * wd.scale_weight * r * r;
    }
    if (wd.plane_reg_weight > 0 && wd.n_kf > 1) chain = plane_chain_cost(wd, bd.pose0, bd.plane0);
    EvalHead& hd = o.head[w];
    hd.n_obs = wd.n_obs; hd.n_gp = wd.n_gp; hd.failed = failed > 0.0 ? 1 : 0; hd.pad = 0;
    hd.cost[0] = c_repr; hd.cost[1] = c_depth; hd.cost[2] = gp; hd.cost[3] = scale; hd.cost[4] = chain;
    hd.cost[5] = c_repr + c_depth + gp + scale + chain;
}

void launch_evaluate(const BatchDev& bd, const PackRaw& raw, const EvalWin* wins, const EvalOut& o, int max_lm, cudaStream_t s) {
    const int B = bd.n_win;
    const int gx = (max_lm + kEvLmPerCta - 1) / kEvLmPerCta;
    k_ev_obs<<<dim3(gx > 0 ? gx : 1, B), 256, 0, s>>>(bd, raw, wins, o); LCHK("k_ev_obs");
    k_ev_finish<<<B, 512, 0, s>>>(bd, raw, wins, o); LCHK("k_ev_finish");
}

}  // namespace kba
