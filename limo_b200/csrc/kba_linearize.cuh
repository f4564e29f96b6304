// kba_linearize.cuh -- the whole linearisation of a small window in ONE kernel (fused path, FP64, one camera per keyframe):
//
//   k_linearize = residual / Jacobian evaluation (cost_functors_ceres.hpp:91-155,193-212, as k_eval_obs)
//               + landmark blocks C_j = sum J_l^T J_l, g_j = sum J_l^T r, LM damping, 3x3 Cholesky (as k_landmark_reduce)
//               + V_i = (J_p^T J_l) L^-T of every observation (as k_obs_v2)
//
// Round 1 / early round 2 ran these as three kernels around a materialised J_p (168 B per observation written, then read
// twice).  Here nothing of the Jacobian reaches
// memory: a lane evaluates its observation in factored form (kba_device.cuh: eval_factored), parks M = m^T m and a = R p in
// the warp's shared-memory strip (9 doubles, where J_p took 18 registers: this is what fits three CTAs per SM), forms V from
// them and writes only what the Schur kernel and the back substitution consume -- V_i (144 B per observation) and the
// landmark's L^-1, z, g, lambda.  A rejected LM step (new radius, same x) simply runs the kernel again: re-evaluating is
// cheaper than re-reading.
//
// Work split: lane = observation, WARP = tile.  k_solve_begin cuts the window's landmark-major observation stream into
// tiles of whole, consecutive landmarks with at most 32 observations together (a landmark has at most 32 on this path:
// <= 32 keyframes, one observation per keyframe; the lanes of trimmed landmarks idle, so the tiling -- and with it the
// cost-partial slots -- does not change inside a solve), so everything a landmark needs is inside one warp: the lanes
// leave their block contributions in the warp's shared-memory strip, lane (landmark, component) sums its segment in
// observation order (the order of the CPU oracle; fixed -> bit-reproducible), every lane then factors its landmark's
// damped block redundantly (it needs L^-1 anyway) -- no CTA barrier between evaluation and V.  A first version with CTA-wide tiles and one thread per landmark for the block sums stalled 256
// threads on two barriers around a serial sqrt / divide chain.
#pragma once
#include <type_traits>
#include "kba_device.cuh"

namespace kba {

constexpr int kLinThreads = 256;
constexpr int kLinWarps = kLinThreads / 32;

// tiles of window w: at most n_obs / 16 + n_lm / 32 + 4 (two consecutive tiles of a chunk hold more than 32 observations; every
// chunk of >= 64 landmarks may end with a short one), stored at BatchDev::lin_tile + lin_tile_offset as {first observation
// (window-local), observations}
__host__ __device__ __forceinline__ int lin_tile_bound(int n_obs, int n_lm) { return n_obs / 16 + n_lm / 32 + 4; }
__device__ __forceinline__ size_t lin_tile_offset(const WinDesc& wd, int w) {
    return (size_t)(wd.obs_off / 16) + (size_t)(wd.lm_off / 32) + 4 * (size_t)w;
}

// Tried and dropped: a descriptor that also carries the first landmark and a segment-start mask,
// so that a lane requests its landmark's data together with its observation's (no obs_lm -> lm_ptr round first), made the kernel
// slower -- the bit arithmetic costs more than the dependent loads, which mostly hit L2.
// called by k_solve_begin (one CTA per window).  The tiling depends on the CSR only.  Greedy packing is sequential, so the
// landmarks are cut into <= 512 chunks that are packed independently by one thread each (pass 1 counts, a scan places the
// chunks, pass 2 writes): one thread walking thousands of landmarks would be a long serial chain in every solve begin.
__device__ inline void build_lin_tiles(const BatchDev& bd, const WinDesc& wd, WinState& st, int w, int* s_chunk /* [513] */) {
    const int* lm_ptr = bd.lm_ptr + wd.lm_off + w;
    int2* tiles = bd.lin_tile + lin_tile_offset(wd, w);
    const int per = max(64, (wd.n_lm + 511) / 512);
    const int n_chunks = (wd.n_lm + per - 1) / per;
    for (int pass = 0; pass < 2; ++pass) {
        for (int c = threadIdx.x; c < n_chunks; c += blockDim.x) {
            const int j0 = c * per, j1 = min(wd.n_lm, j0 + per);
            int n = 0, t_start = 0, t_cnt = 0;
            int2* out = tiles + (pass ? s_chunk[c] : 0);
            int o0 = lm_ptr[j0];
            for (int j = j0; j < j1; ++j) {
                const int o1 = lm_ptr[j + 1], k = o1 - o0;
                if (k > 0) {
                    const bool over = k > 32;  // oversized (never on this path): ends the tile, is skipped
                    if (t_cnt > 0 && (over || t_cnt + k > 32)) { if (pass) out[n] = make_int2(t_start, t_cnt); ++n; t_cnt = 0; }
                    if (!over) { if (t_cnt == 0) t_start = o0; t_cnt += k; }
                }
                o0 = o1;
            }
            if (t_cnt > 0) { if (pass) out[n] = make_int2(t_start, t_cnt); ++n; }
            if (!pass) s_chunk[c] = n;
        }
        __syncthreads();
        if (!pass) {
            if (threadIdx.x == 0) {
                int acc = 0;
                for (int c = 0; c < n_chunks; ++c) { const int t = s_chunk[c]; s_chunk[c] = acc; acc += t; }
                // windows this path does not serve (several observations per landmark and keyframe: more tile breaks than the
                // bound allows for) get no tiles -- k_linearize is not launched for them (BatchDev::lin1)
                if (acc > lin_tile_bound(wd.n_obs, wd.n_lm)) acc = 0;
                st.n_lin_tiles = acc;
                s_chunk[512] = acc;
            }
            __syncthreads();
            if (s_chunk[512] == 0) return;
        }
    }
}

// Three CTAs (24 warps) per SM: at most 80 registers per thread.  The kernel is bound by instruction latency, so the occupancy
// pays (DESIGN.md section 9).  The FP64 division / square-root slow paths are calls: whatever is live across the evaluation is
// saved around them, so what a lane needs later is parked in shared memory (s_ma, s_ix) or re-read where it is used.  The
// form without the unit loop compiles to 78 registers without spills; the striding form keeps 8 B of spill stores.
// n_units = ceil(lin_tile_bound / kLinWarps): a unit is 8 consecutive warp tiles and owns cost slot `unit`.  The CTAs of a window
// stride over the units (grid.x <= n_units; grid.x == n_units: one unit per CTA, the original launch): the tile bound is 1.7x the
// tiles a window really has and every pass is launched for every window, so a smaller grid saves the CTAs that would only find out
// that they have nothing to do and stages the poses once for several units.
// kLoop = false: grid.x == n_units, compiled without the loop (no loop-carried registers: the loop form spills more).
constexpr int kLinMinBlocks = 3;
// k_linearize's static shared memory (the arrays declared in the kernel, below): it has to stay within the 48 KB a kernel may
// declare statically; a larger kFusedMaxKf or kMaxCam means dynamic shared memory (or thinner per-lane strips)
constexpr size_t kLinStaticSmem = sizeof(double) * (kFusedMaxKf * kPoseStride + kMaxCam * kCamStride + kLinWarps * 9 * 33 +
                                                    kLinWarps * 32 * 9 + kLinWarps + 4) +
                                  sizeof(int) * (kLinWarps * 6 * 32 + kLinWarps) + sizeof(uint64_t);
static_assert(kLinStaticSmem <= 48 * 1024, "k_linearize: static shared memory over 48 KB");
template <bool kLoop>
__global__ void __launch_bounds__(kLinThreads, kLinMinBlocks) k_linearize(BatchDev bd, int n_units) {
    const int w = blockIdx.y;
    WinState& st = bd.state[w];
    if (st.phase != PH_ITERATE) return;
    const WinDesc& wd = bd.desc[w];
    // The flags of the pass are read from the window state where they are used (volatile): carried in registers across the
    // evaluation, they would be spilled at 80 registers.  lin: x changed.  want_cost: the cost at x is evaluated at iteration
    // zero of a solve only -- afterwards x is an accepted candidate whose cost the candidate pass (k_eval_obs<false>) has
    // already summed, and k_lm_update carries it over (as ceres does): two FP64 logarithms per observation less in every
    // later pass.
    const volatile WinState& vst = st;
    const auto n_tiles = [&] { return vst.n_lin_tiles; };
    const auto lin = [&] { return vst.need_linearize != 0; };
    const auto want_cost = [&] { return vst.need_linearize != 0 && vst.iter0 != 0; };
    if (wd.landmarks_fixed && !want_cost()) return;     // motion-only window past iteration zero: the landmark blocks are constant
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    __shared__ __align__(16) double s_pose[kFusedMaxKf * kPoseStride];
    __shared__ __align__(16) double s_cam[kMaxCam * kCamStride];
    __shared__ __align__(8) uint64_t s_bar;
    __shared__ double s_cg[kLinWarps][9][33];           // per warp: block contributions of its 32 observations; then, in place at the
                                                        // landmark's first lane, their sums
    __shared__ double s_ma[kLinWarps][32][9];           // per lane: M (sym3 layout) and a of its observation, written as they are
                                                        // formed and read back for V: in registers they would be live across the
                                                        // FP64 division calls, the segment sums and the Cholesky (9 doubles per
                                                        // lane, odd: conflict-free)
    __shared__ int s_ix[kLinWarps][6][32];              // per lane: keyframe, pose row, first observation of the landmark (batch
                                                        // index), its observation count, landmark, flags (1: lane holds an
                                                        // observation, 2: of an active landmark; bits 2-6: the landmark's first
                                                        // lane; 128: evaluated) -- parked across the evaluation, whose FP64
                                                        // division calls would spill them
    __shared__ double s_red[kLinWarps];
    __shared__ int s_cnt[kLinWarps];
    __shared__ double s_prm[4];                         // the window's options (BatchDev::wsp): squared Cauchy scales of the
                                                        // reprojection and depth rows, LM diagonal bounds -- staged with the
                                                        // poses, read where they are used (no register is live for them)
    for (int unit = blockIdx.x; unit < n_units; unit += gridDim.x) {
    asm volatile("" ::: "memory");  // the window's values are re-read per unit: hoisted out of the loop, they would be spilled
    if (unit * kLinWarps >= n_tiles()) {                  // no tile in this unit: its cost slot still has to read zero
        if (tid == 0 && want_cost()) bd.cost_part_x[(size_t)w * bd.cost_parts + unit] = 0.0;
        if constexpr (!kLoop) return;
        continue;
    }
    const size_t base = (size_t)wd.obs_off;
    const int* lm_ptr = bd.lm_ptr + wd.lm_off + w;
    // my observation: the loads are issued before the staging barrier so that their latency overlaps the bulk copy
    const int t = unit * kLinWarps + warp;
    int2 tile = make_int2(0, 0);
    if (t < n_tiles()) tile = bd.lin_tile[lin_tile_offset(wd, w) + t];
    const bool have = lane < tile.y;
    const int o = tile.x + lane;
    int j = 0, kf = 0, cam = 0, row0 = -1, p0 = 0, p1 = 0;
    float mu = 0.f, mv = 0.f, md = 0.f;
    double p[3] = {0, 0, 0}, wgt = 0.0;
    bool act = false;
    if (have) {
        const size_t oo = base + o;
        j = bd.obs_lm[oo];
        kf = bd.obs_kf[oo]; cam = bd.obs_cam[oo]; row0 = bd.obs_row[oo];
        mu = bd.obs_u[oo]; mv = bd.obs_v[oo]; md = bd.obs_d[oo];
        p0 = lm_ptr[j]; p1 = lm_ptr[j + 1];
        act = bd.lm_active[wd.lm_off + j] != 0;         // lanes of trimmed landmarks idle
        const double* lmp = bd.lm[st.cur] + 3 * (size_t)(wd.lm_off + j);
        p[0] = lmp[0]; p[1] = lmp[1]; p[2] = lmp[2];
        wgt = bd.lm_weight[wd.lm_off + j];
    }
    int (*six)[32] = s_ix[warp];
    // once, in the CTA's first unit (the poses do not change within a pass): units are taken in increasing order, so when the
    // first one holds no tile, none does
    if (unit == (int)blockIdx.x) {
        if (tid == 0) {
            const SolveParams& sp = bd.wsp[w];
            s_prm[0] = sp.reprojection_thres * sp.reprojection_thres; s_prm[1] = sp.depth_thres * sp.depth_thres;
            s_prm[2] = sp.min_lm_diagonal; s_prm[3] = sp.max_lm_diagonal;
        }
        stage_window_bulk(wd, bd.rt[st.cur], bd.cam, s_pose, s_cam, &s_bar);  // its barrier publishes s_prm
    }
    six[0][lane] = kf; six[1][lane] = row0; six[2][lane] = wd.obs_off + p0; six[3][lane] = p1 - p0; six[4][lane] = wd.lm_off + j;
    six[5][lane] = have ? 1 | (act ? 2 : 0) | ((p0 - tile.x) << 2) : 0;
    // ---- evaluate my observation; contributions to its landmark block
    double* sma = s_ma[warp][lane];
    bool ok = false;                                    // my observation is active and evaluated
    double hr = 0.0;
    double cg[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    if (act) {
        // the contributions are formed inside each of the two instantiations (with / without the cost terms): merged after
        // them, m and r would be live across the join and spilled
        const auto evaluate = [&](auto with_cost) {
            double r[3], m[9], raw[2];
            const double br = s_prm[0], bdp = s_prm[1];
            ok = eval_factored<double, true, decltype(with_cost)::value>(s_pose + kPoseStride * kf, s_cam + kCamStride * cam, p,
                                                                          (double)mu, (double)mv, (double)md, wgt, br, bdp, r, m,
                                                                          sma + 6, hr, raw);
            if (!ok) return;
            {   // the flag word's address from a fresh read of the thread index: kept from before the evaluation, it would be spilled
                unsigned t;
                asm volatile("mov.u32 %0, %%tid.x;" : "=r"(t));
                s_ix[t >> 5][5][t & 31] |= 128;
            }
            gram_factored(m, sma);
            // C and g from J_l = m R, as the three-kernel path forms them.  R^T M R rounds no worse, but a landmark seen with
            // almost no parallax (condition ~1e10) amplifies any change of rounding: in the parity tests' evaluation-failure
            // window one then ended 17 cm from the oracle's solution (this form: 5 cm).  The keyframe is re-read from the
            // strip: kept in a register, it would be spilled across the evaluation
            const double* R = s_pose + kPoseStride * reinterpret_cast<volatile int*>(six[0])[lane];
            double jl[9];
#pragma unroll
            for (int i = 0; i < 3; ++i) {
#pragma unroll
                for (int c = 0; c < 3; ++c) jl[3 * i + c] = m[3 * i] * R[c] + m[3 * i + 1] * R[3 + c] + m[3 * i + 2] * R[6 + c];
            }
            cg[0] = jl[0] * jl[0] + jl[3] * jl[3] + jl[6] * jl[6];
            cg[1] = jl[0] * jl[1] + jl[3] * jl[4] + jl[6] * jl[7];
            cg[2] = jl[0] * jl[2] + jl[3] * jl[5] + jl[6] * jl[8];
            cg[3] = jl[1] * jl[1] + jl[4] * jl[4] + jl[7] * jl[7];
            cg[4] = jl[1] * jl[2] + jl[4] * jl[5] + jl[7] * jl[8];
            cg[5] = jl[2] * jl[2] + jl[5] * jl[5] + jl[8] * jl[8];
#pragma unroll
            for (int c = 0; c < 3; ++c) cg[6 + c] = jl[c] * r[0] + jl[3 + c] * r[1] + jl[6 + c] * r[2];
        };
        if (want_cost()) evaluate(std::true_type{});
        else evaluate(std::false_type{});
        if (!ok) {
            hr = 0.0;
            if (lin()) st.eval_failed = 1;  // benign race
        }
    }
    {   // cost partial of the CTA (fixed-shape reduction; the barrier is at the very end) and the observation count of the roofline report
        const double cs = warp_sum(hr);
        const int dn = __reduce_add_sync(0xffffffffu, ok ? 1 : 0);
        if (lane == 0) { s_red[warp] = cs; s_cnt[warp] = dn; }
    }
    if (!wd.landmarks_fixed) {  // (uniform per window) motion-only: the landmark blocks are constant, only the cost at x was needed
        // ---- landmark blocks.  Lanes seg0 .. seg0 + klen - 1 of the warp hold my landmark.
        double (*sw)[33] = s_cg[warp];  // row stride 33: the lanes summing different components below hit different banks
#pragma unroll
        for (int q = 0; q < 9; ++q) sw[q][lane] = cg[q];
        __syncwarp();
        const int L = six[4][lane];
        const bool in_tile = six[5][lane] & 1, active = six[5][lane] & 2;  // have, act of the loads above
        const int seg0 = (six[5][lane] >> 2) & 31;
        const int klen = six[3][lane];
        // the stored Jacobi scaling of my landmark (past iteration zero): requested here, consumed after the segment sums
        double tt_ld[3] = {0.0, 0.0, 0.0};
        if (active && !st.iter0) {
#pragma unroll
            for (int e = 0; e < 3; ++e) tt_ld[e] = bd.lm_scale[3 * (size_t)L + e];
        }
        // lane seg0 + q of a landmark sums component q of its block in lane order (landmarks with fewer than 9 observations: several
        // components per lane) and leaves the sum at [q][first lane of the landmark] -- in place: component q of a landmark is read
        // and written by this one lane only
        if (in_tile) {
            for (int q = lane - seg0; q < 9; q += klen) {
                double sacc = 0.0;
                for (int l = seg0; l < seg0 + klen; ++l) sacc += sw[q][l];
                sw[q][seg0] = sacc;
            }
        }
        __syncwarp();
        if (active) {
            double c[6], g[3];
#pragma unroll
            for (int q = 0; q < 6; ++q) c[q] = sw[q][seg0];
#pragma unroll
            for (int q = 0; q < 3; ++q) g[q] = sw[6 + q][seg0];
            const bool first = lane == seg0;  // writes the landmark's outputs
            // the landmark's ground-plane height residual (at most one) is one more row of its Jacobian
            const int gl = (wd.n_gp > 0) ? bd.gp_of_lm[L] : -1;
            const size_t TG = (size_t)bd.tot_gp, G = (size_t)wd.gp_off + (gl >= 0 ? gl : 0);
            double gjl[3] = {0, 0, 0};
            if (gl >= 0) {
                gjl[0] = bd.gp_lin[11 * TG + G]; gjl[1] = bd.gp_lin[12 * TG + G]; gjl[2] = bd.gp_lin[13 * TG + G];
                const double gr = bd.gp_lin[G];
                c[0] += gjl[0] * gjl[0]; c[1] += gjl[0] * gjl[1]; c[2] += gjl[0] * gjl[2];
                c[3] += gjl[1] * gjl[1]; c[4] += gjl[1] * gjl[2]; c[5] += gjl[2] * gjl[2];
                g[0] += gjl[0] * gr; g[1] += gjl[1] * gr; g[2] += gjl[2] * gr;
            }
            // Jacobi scaling (fixed at iteration zero of the solve) and LM damping of the three landmark columns
            // BatchDev::lm_scale holds t = 1 / scale = 1 + sqrt(C_ee) on this path, so that the Jacobi-scaled damping
            // clamp(C_ee s^2, lo, hi) / (radius s^2) = clamp(C_ee, lo t^2, hi t^2) / radius needs no division per column
            const double cd[3] = {c[0], c[3], c[5]};
            const double inv_radius = 1.0 / st.radius;
            double tt[3], lam[3];
#pragma unroll
            for (int e = 0; e < 3; ++e) {
                tt[e] = st.iter0 ? 1.0 + sqrt(cd[e]) : tt_ld[e];
                const double t2 = tt[e] * tt[e];
                lam[e] = fmin(fmax(cd[e], s_prm[2] * t2), s_prm[3] * t2) * inv_radius;
            }
            // Cholesky of C + diag(lam) through the reciprocal square roots of the pivots: L^-1 is what every consumer wants
            // (V = E L^-T, z = L^-1 g, the back substitution), L itself is never needed
            const double a00 = c[0] + lam[0], a11 = c[3] + lam[1], a22 = c[5] + lam[2];
            const double i00 = rsqrt(a00);
            const double l10 = c[1] * i00, l20 = c[2] * i00;
            const double d11 = a11 - l10 * l10;
            const double i11 = rsqrt(d11);
            const double l21 = (c[4] - l20 * l10) * i11;
            const double d22 = a22 - l20 * l20 - l21 * l21;
            const double i22 = rsqrt(d22);
            if (!((a00 > 0.0) && (d11 > 0.0) && (d22 > 0.0))) {
                st.solve_failed = 1;  // benign race; V of this landmark is not written, the step is invalid anyway
            } else {
                const double i10 = -l10 * i00 * i11;
                const double i21 = -l21 * i11 * i22;
                const double i20 = -(l20 * i00 + l21 * i10) * i22;
                if (first) {
                    double* li = bd.lm_linv + 6 * (size_t)L;
                    li[0] = i00; li[1] = i10; li[2] = i11; li[3] = i20; li[4] = i21; li[5] = i22;
                    double* zz = bd.lm_z + 3 * (size_t)L;
                    zz[0] = i00 * g[0]; zz[1] = i10 * g[0] + i11 * g[1]; zz[2] = i20 * g[0] + i21 * g[1] + i22 * g[2];
#pragma unroll
                    for (int e = 0; e < 3; ++e) {
                        bd.lm_g[3 * (size_t)L + e] = g[e];
                        bd.lm_lambda[3 * (size_t)L + e] = lam[e];
                        if (st.iter0) bd.lm_scale[3 * (size_t)L + e] = tt[e];
                    }
                    if (gl >= 0) {  // V rows of the gp block: E = J_f^T J_l is 10 x 3 (rank one)
                        for (int rr = 0; rr < 10; ++rr) {
                            const double jf_ = bd.gp_lin[(1 + rr) * TG + G];
                            const double e0 = jf_ * gjl[0], e1 = jf_ * gjl[1], e2 = jf_ * gjl[2];
                            bd.vgp[(3 * rr + 0) * TG + G] = e0 * i00;
                            bd.vgp[(3 * rr + 1) * TG + G] = e0 * i10 + e1 * i11;
                            bd.vgp[(3 * rr + 2) * TG + G] = e0 * i20 + e1 * i21 + e2 * i22;
                        }
                    }
                }
                // ---- V_i = (J_p^T J_l) L^-T = [K^T ; I] W with W = M R L^-T: the translation rows are W, the rotation rows
                //      K^T W_c = 2 a x W_c (K = -2 [a]x)
                if ((six[5][lane] & 128) && six[1][lane] >= 0) {
                    const double* R = s_pose + kPoseStride * six[0][lane];
                    const int g0 = six[2][lane];
                    double wm[9];
#pragma unroll
                    for (int r = 0; r < 3; ++r) {
                        const double m0 = sma[sym3(r, 0)], m1 = sma[sym3(r, 1)], m2 = sma[sym3(r, 2)];
                        const double l0 = m0 * R[0] + m1 * R[3] + m2 * R[6], l1 = m0 * R[1] + m1 * R[4] + m2 * R[7], l2 = m0 * R[2] + m1 * R[5] + m2 * R[8];
                        wm[3 * r + 0] = l0 * i00;
                        wm[3 * r + 1] = l0 * i10 + l1 * i11;
                        wm[3 * r + 2] = l0 * i20 + l1 * i21 + l2 * i22;
                    }
#pragma unroll
                    for (int cc = 0; cc < 3; ++cc) {  // 48 contiguous bytes per column; consecutive lanes = consecutive observations of the landmark
                        double2* out = reinterpret_cast<double2*>(bd.vobs + vobs_index(0, g0, g0 + klen, g0 + lane - seg0, cc));
                        const double w0 = wm[cc], w1 = wm[3 + cc], w2 = wm[6 + cc];
                        const double a0 = sma[6], a1 = sma[7], a2 = sma[8];
                        out[0] = make_double2(2.0 * (a1 * w2 - a2 * w1), 2.0 * (a2 * w0 - a0 * w2));
                        out[1] = make_double2(2.0 * (a0 * w1 - a1 * w0), w0);
                        out[2] = make_double2(w1, w2);
                    }
                }
            }
        }
    }
    __syncthreads();  // only the cost partial crosses warps
    if (tid == 0) {
        double s = 0.0;
        int cnt = 0;
        for (int q = 0; q < kLinWarps; ++q) { s += s_red[q]; cnt += s_cnt[q]; }
        if (want_cost()) bd.cost_part_x[(size_t)w * bd.cost_parts + unit] = s;
        if (cnt) atomicAdd(bd.jac_obs, (unsigned long long)cnt);
    }
    if constexpr (!kLoop) break;
    if (unit + (int)gridDim.x < n_units) __syncthreads();  // s_red / s_cnt are rewritten by the next unit
    }  // units
}

}  // namespace kba
