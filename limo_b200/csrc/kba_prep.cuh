// kba_prep.cuh -- per-landmark preparation of one LM step, split by access pattern:
//   k_landmark_reduce : 16 lanes per landmark -> C_j = sum J_l^T J_l, g_j = sum J_l^T r (shuffle tree), Jacobi-scaled LM
//                       damping, 3x3 Cholesky, L^-1, z_j = L^-1 g_j, V rows of the landmark's ground-plane block
//   k_obs_v           : one thread per observation (fully coalesced SoA loads) -> V_i = (J_p^T J_l) L^-T, written either
//                       into the dense column-major chunk panel the Schur kernels load
//   k_gp_panel        : ground-plane V rows into the panel (added onto an observation's pose rows when they coincide)
#pragma once
#include "kba_device.cuh"

namespace kba {

__device__ __forceinline__ int gp_row(const BatchDev& bd, const WinDesc& wd, int k, int r);

// kFused: J_l is not materialised; it is formed here as (translation columns of J_p) R(keyframe), the rotations staged by
// one bulk copy, and the z row goes to global memory only (lm_z) -- the fused Schur kernel builds its panels itself.
template <bool kFused>
__global__ void __launch_bounds__(256, 4) k_landmark_reduce(BatchDev bd) {
    const int w = blockIdx.y;
    const SolveParams& sp = bd.wsp[w];
    WinState& st = bd.state[w];
    if (st.phase != PH_ITERATE) return;
    const WinDesc& wd = bd.desc[w];
    if (wd.landmarks_fixed) return;
    __shared__ __align__(16) double s_pose[kFused ? kFusedMaxKf * kPoseStride : 2];
    __shared__ __align__(8) uint64_t s_bar;
    if (kFused) {
        if (threadIdx.x == 0) {
            mbar_init(&s_bar, 1);
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            const uint32_t bytes = (uint32_t)(wd.n_kf * kPoseStride * sizeof(double));
            mbar_expect_tx(&s_bar, bytes);
            tma_load_1d(s_pose, bd.rt[st.cur] + (size_t)kPoseStride * wd.kf_off, bytes, &s_bar);
        }
    }
    const int sl = threadIdx.x & 15;                       // lane inside the 16-lane group
    const int j = blockIdx.x * 16 + (threadIdx.x >> 4);    // one landmark per half warp
    const int L = wd.lm_off + min(j, wd.n_lm - 1);
    const int* lm_ptr = bd.lm_ptr + wd.lm_off + w;
    int o0 = 0, o1 = 0;
    bool valid = j < wd.n_lm && bd.lm_active[L];
    if (valid) { o0 = lm_ptr[j]; o1 = lm_ptr[j + 1]; valid = o1 > o0; }
    const size_t T = (size_t)bd.tot_obs, base = (size_t)wd.obs_off;
    double c[6] = {0, 0, 0, 0, 0, 0}, g[3] = {0, 0, 0};
    if (kFused) mbar_wait(&s_bar, 0);
    if (valid) {
        for (int o = o0 + sl; o < o1; o += 16) {
            double jl[9], r[3];
            if (kFused) {
                const double* R = s_pose + kPoseStride * bd.obs_kf[base + o];
#pragma unroll
                for (int i = 0; i < 3; ++i) {
                    const double m0 = lin_load(bd.jp, (6 * i + 3) * T + base + o, bd.precision);
                    const double m1 = lin_load(bd.jp, (6 * i + 4) * T + base + o, bd.precision);
                    const double m2 = lin_load(bd.jp, (6 * i + 5) * T + base + o, bd.precision);
#pragma unroll
                    for (int c = 0; c < 3; ++c) jl[3 * i + c] = m0 * R[c] + m1 * R[3 + c] + m2 * R[6 + c];
                }
            } else {
#pragma unroll
                for (int q = 0; q < 9; ++q) jl[q] = lin_load(bd.jl, q * T + base + o, bd.precision);
            }
#pragma unroll
            for (int q = 0; q < 3; ++q) r[q] = lin_load(bd.res, q * T + base + o, bd.precision);
            c[0] += jl[0] * jl[0] + jl[3] * jl[3] + jl[6] * jl[6];
            c[1] += jl[0] * jl[1] + jl[3] * jl[4] + jl[6] * jl[7];
            c[2] += jl[0] * jl[2] + jl[3] * jl[5] + jl[6] * jl[8];
            c[3] += jl[1] * jl[1] + jl[4] * jl[4] + jl[7] * jl[7];
            c[4] += jl[1] * jl[2] + jl[4] * jl[5] + jl[7] * jl[8];
            c[5] += jl[2] * jl[2] + jl[5] * jl[5] + jl[8] * jl[8];
#pragma unroll
            for (int a = 0; a < 3; ++a) g[a] += jl[a] * r[0] + jl[3 + a] * r[1] + jl[6 + a] * r[2];
        }
    }
    // the landmark's ground-plane height residual (at most one) is one more row of its Jacobian
    const int gl = (valid && wd.n_gp > 0) ? bd.gp_of_lm[L] : -1;
    const size_t TG = (size_t)bd.tot_gp, G = (size_t)wd.gp_off + (gl >= 0 ? gl : 0);
    double gjl[3] = {0, 0, 0};
    if (gl >= 0) {
        gjl[0] = bd.gp_lin[11 * TG + G]; gjl[1] = bd.gp_lin[12 * TG + G]; gjl[2] = bd.gp_lin[13 * TG + G];
        if (sl == 0) {
            const double gr = bd.gp_lin[G];
            c[0] += gjl[0] * gjl[0]; c[1] += gjl[0] * gjl[1]; c[2] += gjl[0] * gjl[2];
            c[3] += gjl[1] * gjl[1]; c[4] += gjl[1] * gjl[2]; c[5] += gjl[2] * gjl[2];
            g[0] += gjl[0] * gr; g[1] += gjl[1] * gr; g[2] += gjl[2] * gr;
        }
    }
    // fixed-shape butterfly inside the 16-lane group (xor offsets < 16 never cross the half-warp boundary)
#pragma unroll
    for (int q = 0; q < 6; ++q)
#pragma unroll
        for (int o = 8; o > 0; o >>= 1) c[q] += __shfl_xor_sync(0xffffffffu, c[q], o);
#pragma unroll
    for (int q = 0; q < 3; ++q)
#pragma unroll
        for (int o = 8; o > 0; o >>= 1) g[q] += __shfl_xor_sync(0xffffffffu, g[q], o);
    if (!valid) return;
    // Jacobi scaling (fixed at iteration zero of the solve) and LM damping of the three landmark columns
    const double cd[3] = {c[0], c[3], c[5]};
    double sc[3], lam[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        sc[a] = st.iter0 ? 1.0 / (1.0 + sqrt(cd[a])) : bd.lm_scale[3 * (size_t)L + a];
        const double s2 = sc[a] * sc[a];
        lam[a] = fmin(fmax(cd[a] * s2, sp.min_lm_diagonal), sp.max_lm_diagonal) / (st.radius * s2);
    }
    // Cholesky of C + diag(lam) and the inverse of its factor
    const double a00 = c[0] + lam[0], a11 = c[3] + lam[1], a22 = c[5] + lam[2];
    const double l00 = sqrt(a00);
    const double l10 = c[1] / l00, l20 = c[2] / l00;
    const double d11 = a11 - l10 * l10;
    const double l11 = sqrt(d11);
    const double l21 = (c[4] - l20 * l10) / l11;
    const double d22 = a22 - l20 * l20 - l21 * l21;
    const double l22 = sqrt(d22);
    if (!(a00 > 0.0) || !(d11 > 0.0) || !(d22 > 0.0)) {
        if (sl == 0) st.solve_failed = 1;
        return;
    }
    const double i00 = 1.0 / l00, i11 = 1.0 / l11, i22 = 1.0 / l22;
    const double i10 = -l10 * i00 * i11;
    const double i21 = -l21 * i11 * i22;
    const double i20 = -(l20 * i00 + l21 * i10) * i22;
    const double z0 = i00 * g[0], z1 = i10 * g[0] + i11 * g[1], z2 = i20 * g[0] + i21 * g[1] + i22 * g[2];
    if (sl == 0) {
        double* li = bd.lm_linv + 6 * (size_t)L;
        li[0] = i00; li[1] = i10; li[2] = i11; li[3] = i20; li[4] = i21; li[5] = i22;
        double* zz = bd.lm_z + 3 * (size_t)L;
        zz[0] = z0; zz[1] = z1; zz[2] = z2;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            bd.lm_g[3 * (size_t)L + a] = g[a];
            bd.lm_lambda[3 * (size_t)L + a] = lam[a];
            if (st.iter0) bd.lm_scale[3 * (size_t)L + a] = sc[a];
        }
        if (!kFused) {  // right-hand-side row z_j of the chunk panel
            const int ch = wd.chunk_off + (j >> 5);
            const int prs = bd.chunk_rs[ch];
            if (prs > 0) {
                const int t0 = bd.chunk_t0[ch], t1 = bd.chunk_t1[ch], trhs = st.n_f >> 3;
                const int rl = (trhs >= t0 && trhs < t1) ? st.n_f - 8 * t0 : 8 * (t1 - t0) + (st.n_f - 8 * trhs);
                double* pcol = bd.vpanel + wd.panel_off + bd.chunk_poff[ch] + (size_t)(3 * (j & 31)) * prs;
                pcol[rl] = z0; pcol[prs + rl] = z1; pcol[2 * prs + rl] = z2;
            }
        }
    }
    if (gl >= 0 && sl < 10) {  // V rows of the gp block: E = J_f^T J_l is 10 x 3 (rank one), row `sl`
        const double jf = bd.gp_lin[(1 + sl) * TG + G];
        const double e0 = jf * gjl[0], e1 = jf * gjl[1], e2 = jf * gjl[2];
        bd.vgp[(3 * sl + 0) * TG + G] = e0 * i00;
        bd.vgp[(3 * sl + 1) * TG + G] = e0 * i10 + e1 * i11;
        bd.vgp[(3 * sl + 2) * TG + G] = e0 * i20 + e1 * i21 + e2 * i22;
    }
}

// V_i = E_i L^-T with E_i = J_p^T J_l (6x3): one thread per observation.  `round` selects the observation rank: rank 0
// writes, rank r > 0 (further cameras of a rig seeing the landmark in the same keyframe) adds onto the same panel rows.
__global__ void __launch_bounds__(256) k_obs_v(BatchDev bd, int round) {
    const int w = blockIdx.y;
    const WinState& st = bd.state[w];
    if (st.phase != PH_ITERATE || st.solve_failed) return;
    const WinDesc& wd = bd.desc[w];
    if (wd.landmarks_fixed || round > wd.max_rank) return;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= wd.n_obs) return;
    const size_t o = (size_t)wd.obs_off + i, T = (size_t)bd.tot_obs;
    const int row0 = bd.obs_row[o];  // -1: constant pose or trimmed landmark
    if (row0 < 0 || bd.obs_rank[o] != round) return;
    const int j = bd.obs_lm[o];
    const double* li = bd.lm_linv + 6 * (size_t)(wd.lm_off + j);
    const double i00 = li[0], i10 = li[1], i11 = li[2], i20 = li[3], i21 = li[4], i22 = li[5];
    double jl[9], jp[18];
#pragma unroll
    for (int q = 0; q < 9; ++q) jl[q] = lin_load(bd.jl, q * T + o, bd.precision);
#pragma unroll
    for (int q = 0; q < 18; ++q) jp[q] = lin_load(bd.jp, q * T + o, bd.precision);
    double vv[3][6];  // [column][row]
#pragma unroll
    for (int r = 0; r < 6; ++r) {
        const double e0 = jp[r] * jl[0] + jp[6 + r] * jl[3] + jp[12 + r] * jl[6];
        const double e1 = jp[r] * jl[1] + jp[6 + r] * jl[4] + jp[12 + r] * jl[7];
        const double e2 = jp[r] * jl[2] + jp[6 + r] * jl[5] + jp[12 + r] * jl[8];
        vv[0][r] = e0 * i00; vv[1][r] = e0 * i10 + e1 * i11; vv[2][r] = e0 * i20 + e1 * i21 + e2 * i22;
    }
    const int ch = wd.chunk_off + (j >> 5);
    const int prs = bd.chunk_rs[ch];
    const int rl = row0 - 8 * bd.chunk_t0[ch];
    double* pcol = bd.vpanel + wd.panel_off + bd.chunk_poff[ch] + (size_t)(3 * (j & 31)) * prs + rl;
    // six consecutive rows of one column = 48 contiguous bytes; 16-byte aligned unless the row is odd
    // (plane blocks without the distance parameter): three 128-bit stores per column
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        double* qs = pcol + (size_t)c * prs;
        if (rl & 1) {
#pragma unroll
            for (int r = 0; r < 6; ++r) qs[r] = (round == 0) ? vv[c][r] : qs[r] + vv[c][r];
        } else {
            double2* q = reinterpret_cast<double2*>(qs);
#pragma unroll
            for (int h = 0; h < 3; ++h) {
                double2 t = make_double2(vv[c][2 * h], vv[c][2 * h + 1]);
                if (round != 0) { const double2 old = q[h]; t.x += old.x; t.y += old.y; }
                q[h] = t;
            }
        }
    }
}

// Fused path: V_i = (J_p^T J_l) L^-T per observation, written compactly (18 doubles: 3 columns x 6 rows; layout: BatchDev::vobs,
// column-major per landmark) -- the fused Schur kernel copies whole landmark columns straight into its shared-memory panels
// and the back substitution reads them again.  J_l is formed
// as (translation columns of J_p) R(keyframe) from the staged rotations; W = J_l L^-T first keeps the dependency chains short.
// HBM per observation: 144 B of J_p read + 144 B written.
__global__ void __launch_bounds__(256) k_obs_v2(BatchDev bd) {
    const int w = blockIdx.y;
    const WinState& st = bd.state[w];
    if (st.phase != PH_ITERATE || st.solve_failed) return;
    const WinDesc& wd = bd.desc[w];
    if (wd.landmarks_fixed) return;
    if ((int)(blockIdx.x * blockDim.x) >= wd.n_obs) return;
    __shared__ __align__(16) double s_pose[kFusedMaxKf * kPoseStride];
    __shared__ __align__(8) uint64_t s_bar;
    if (threadIdx.x == 0) {
        mbar_init(&s_bar, 1);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        const uint32_t bytes = (uint32_t)(wd.n_kf * kPoseStride * sizeof(double));
        mbar_expect_tx(&s_bar, bytes);
        tma_load_1d(s_pose, bd.rt[st.cur] + (size_t)kPoseStride * wd.kf_off, bytes, &s_bar);
    }
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const bool have = i < wd.n_obs;
    const size_t o = (size_t)wd.obs_off + (have ? i : 0), T = (size_t)bd.tot_obs;
    const int row0 = have ? bd.obs_row[o] : -1;  // -1: constant pose or trimmed landmark
    double jp[18], li[6];
    int kf = 0, p0 = 0, p1 = 0;
    if (row0 >= 0) {
        kf = bd.obs_kf[o];
        const int j = bd.obs_lm[o];
        const int* lm_ptr = bd.lm_ptr + wd.lm_off + w;
        p0 = lm_ptr[j]; p1 = lm_ptr[j + 1];
        const double* lp = bd.lm_linv + 6 * (size_t)(wd.lm_off + j);
#pragma unroll
        for (int q = 0; q < 6; ++q) li[q] = lp[q];
#pragma unroll
        for (int q = 0; q < 18; ++q) jp[q] = lin_load(bd.jp, q * T + o, bd.precision);
    }
    mbar_wait(&s_bar, 0);
    if (row0 < 0) return;
    const double* R = s_pose + kPoseStride * kf;
    double wm[9];  // W = J_l L^-T, J_l = M R with M = J_p[:, 3:6];  L^-1 = [i00; i10 i11; i20 i21 i22]
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        const double m0 = jp[6 * r + 3], m1 = jp[6 * r + 4], m2 = jp[6 * r + 5];
        const double l0 = m0 * R[0] + m1 * R[3] + m2 * R[6], l1 = m0 * R[1] + m1 * R[4] + m2 * R[7], l2 = m0 * R[2] + m1 * R[5] + m2 * R[8];
        wm[3 * r + 0] = l0 * li[0];
        wm[3 * r + 1] = l0 * li[1] + l1 * li[2];
        wm[3 * r + 2] = l0 * li[3] + l1 * li[4] + l2 * li[5];
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {  // 48 contiguous bytes per column; consecutive threads = consecutive observations of the landmark
        double2* out = reinterpret_cast<double2*>(bd.vobs + vobs_index((size_t)wd.obs_off, p0, p1, i, c));
#pragma unroll
        for (int h = 0; h < 3; ++h) {
            const int r0 = 2 * h, r1 = 2 * h + 1;  // V[r][c] = sum_k J_p[k][r] W[k][c]
            out[h] = make_double2(jp[r0] * wm[c] + jp[6 + r0] * wm[3 + c] + jp[12 + r0] * wm[6 + c],
                                  jp[r1] * wm[c] + jp[6 + r1] * wm[3 + c] + jp[12 + r1] * wm[6 + c]);
        }
    }
}

// ground-plane V rows into the chunk panels: one thread per (gp residual, row of its 10 x 3 block)
__global__ void __launch_bounds__(256) k_gp_panel(BatchDev bd) {
    const int w = blockIdx.y;
    const WinState& st = bd.state[w];
    if (st.phase != PH_ITERATE || st.solve_failed) return;
    const WinDesc& wd = bd.desc[w];
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= wd.n_gp * 10) return;
    const int gi = idx / 10, r = idx - 10 * gi;
    const size_t G = (size_t)wd.gp_off + gi, TG = (size_t)bd.tot_gp;
    const int j = bd.gp_lm[G];
    const int* lm_ptr = bd.lm_ptr + wd.lm_off + w;
    if (!bd.lm_active[wd.lm_off + j] || lm_ptr[j + 1] <= lm_ptr[j]) return;
    const int row = gp_row(bd, wd, bd.gp_kf[G], r);
    if (row < 0) return;
    const int ch = wd.chunk_off + (j >> 5);
    const int prs = bd.chunk_rs[ch];
    double* q = bd.vpanel + wd.panel_off + bd.chunk_poff[ch] + (size_t)(3 * (j & 31)) * prs + (row - 8 * bd.chunk_t0[ch]);
    const double a0 = bd.vgp[(3 * r + 0) * TG + G], a1 = bd.vgp[(3 * r + 1) * TG + G], a2 = bd.vgp[(3 * r + 2) * TG + G];
    if (r < 6 && bd.gp_shared[G]) { q[0] += a0; q[prs] += a1; q[2 * prs] += a2; }  // an observation wrote these rows
    else { q[0] = a0; q[prs] = a1; q[2 * prs] = a2; }
}

}  // namespace kba
