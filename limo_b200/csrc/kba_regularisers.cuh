// kba_regularisers.cuh -- the f-only residual blocks of the window problem (no landmark involved): ground-plane
// regularisation chain (reference bundle_adjuster_keyframes.cpp:769-818, cost_functors_ceres.hpp:394-438,507-555) and the
// warp-cooperative accumulation of a small residual block into the reduced normal equations.
#pragma once
#include <cfloat>

#include "kba_device.cuh"

namespace kba {

// (I - n n^T / |n|^2) / |n| : Jacobian of FixScaleVectorPlus at delta = 0 (reference local_parameterizations.hpp:146-162)
__device__ inline void dir_plus_jacobian(const double* n, double* P) {
    const double nn = n[0] * n[0] + n[1] * n[1] + n[2] * n[2], inv = 1.0 / sqrt(nn);
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) P[3 * i + j] = ((i == j ? 1.0 : 0.0) - n[i] * n[j] / nn) * inv;
}

__device__ inline void dir_plus(const double* n, const double* d, double* o) {
    const double a = n[0] + d[0], b = n[1] + d[1], c = n[2] + d[2];
    const double f = 1.0 / sqrt(a * a + b * b + c * c);
    o[0] = a * f; o[1] = b * f; o[2] = c * f;
}

// d = t_a - R_a R_b^T t_b = (T_a T_b^-1).t ; Ja, Jb: 3x6 local Jacobians (rot | trans) of d w.r.t. poses a and b
__device__ inline void rel_translation(const double* pa, const double* pb, double* d, double* Ja, double* Jb) {
    double Ra[9], Rb[9], c[3], rac[3];
    quat_to_rot<double>(pa, Ra);
    quat_to_rot<double>(pb, Rb);
    const double* tb = pb + 4;
    for (int i = 0; i < 3; ++i) c[i] = Rb[i] * tb[0] + Rb[3 + i] * tb[1] + Rb[6 + i] * tb[2];
    for (int i = 0; i < 3; ++i) rac[i] = Ra[3 * i] * c[0] + Ra[3 * i + 1] * c[1] + Ra[3 * i + 2] * c[2];
    for (int i = 0; i < 3; ++i) d[i] = pa[4 + i] - rac[i];
    if (!Ja) return;
    double Rab[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j)
            Rab[3 * i + j] = Ra[3 * i] * Rb[3 * j] + Ra[3 * i + 1] * Rb[3 * j + 1] + Ra[3 * i + 2] * Rb[3 * j + 2];
    const double X[9] = {0, -rac[2], rac[1], rac[2], 0, -rac[0], -rac[1], rac[0], 0};
    const double Tm[9] = {0, -tb[2], tb[1], tb[2], 0, -tb[0], -tb[1], tb[0], 0};
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            Ja[6 * i + j] = 2.0 * X[3 * i + j];
            Ja[6 * i + 3 + j] = (i == j) ? 1.0 : 0.0;
            double s = 0.0;
            for (int k = 0; k < 3; ++k) s += Rab[3 * i + k] * Tm[3 * k + j];
            Jb[6 * i + j] = -2.0 * s;
            Jb[6 * i + 3 + j] = -Rab[3 * i + j];
        }
}

// GroundPlaneMotionRegularization (reference cost_functors_ceres.hpp:528-555): r = n0 . normalize((T0 T1^-1).t)
__device__ inline double plane_motion(const double* p0, const double* p1, const double* n0, double* j0, double* j1,
                                      double* jd) {
    double d[3], J0[18], J1[18];
    rel_translation(p0, p1, d, j0 ? J0 : nullptr, J1);
    const double nrm = sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
    const double u[3] = {d[0] / nrm, d[1] / nrm, d[2] / nrm};
    const double r = n0[0] * u[0] + n0[1] * u[1] + n0[2] * u[2];
    if (j0) {
        const double gq[3] = {(n0[0] - r * u[0]) / nrm, (n0[1] - r * u[1]) / nrm, (n0[2] - r * u[2]) / nrm};
        for (int j = 0; j < 6; ++j) {
            j0[j] = gq[0] * J0[j] + gq[1] * J0[6 + j] + gq[2] * J0[12 + j];
            j1[j] = gq[0] * J1[j] + gq[1] * J1[6 + j] + gq[2] * J1[12 + j];
        }
        double P[9];
        dir_plus_jacobian(n0, P);
        for (int j = 0; j < 3; ++j) jd[j] = u[0] * P[j] + u[1] * P[3 + j] + u[2] * P[6 + j];
    }
    return r;
}

// PoseRegularization residual |(T1 T0^-1).t| - s0 with local Jacobians (reference cost_functors_ceres.hpp:224-250).
__device__ inline void scale_regulariser(const double* p1, const double* p0, double s0, double& r, double* j1, double* j0) {
    double R1[9], R0[9];
    quat_to_rot<double>(p1, R1);
    quat_to_rot<double>(p0, R0);
    const double* t1 = p1 + 4, *t0 = p0 + 4;
    double c[3], rc[3], d[3];
    for (int i = 0; i < 3; ++i) c[i] = R0[i] * t0[0] + R0[3 + i] * t0[1] + R0[6 + i] * t0[2];          // R0^T t0
    for (int i = 0; i < 3; ++i) rc[i] = R1[3 * i] * c[0] + R1[3 * i + 1] * c[1] + R1[3 * i + 2] * c[2];  // R1 c
    for (int i = 0; i < 3; ++i) d[i] = t1[i] - rc[i];
    const double nrm = sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
    r = nrm - s0;
    if (!j1) return;
    const double u[3] = {d[0] / nrm, d[1] / nrm, d[2] / nrm};
    // dd/d(dr1) = 2 [R1 c]x -> u^T 2 [rc]x = 2 (u x rc)^T ... (u^T [a]x = (u x a)^T)
    j1[0] = 2.0 * (u[1] * rc[2] - u[2] * rc[1]);
    j1[1] = 2.0 * (u[2] * rc[0] - u[0] * rc[2]);
    j1[2] = 2.0 * (u[0] * rc[1] - u[1] * rc[0]);
    j1[3] = u[0]; j1[4] = u[1]; j1[5] = u[2];
    // dd/d(dt0) = -R1 R0^T ;  dd/d(dr0) = -2 R1 R0^T [t0]x
    double ur[3];  // u^T R1 R0^T  = (R0 R1^T u)^T
    double tmp[3];
    for (int i = 0; i < 3; ++i) tmp[i] = R1[i] * u[0] + R1[3 + i] * u[1] + R1[6 + i] * u[2];               // R1^T u
    for (int i = 0; i < 3; ++i) ur[i] = R0[3 * i] * tmp[0] + R0[3 * i + 1] * tmp[1] + R0[3 * i + 2] * tmp[2];  // R0 R1^T u
    j0[3] = -ur[0]; j0[4] = -ur[1]; j0[5] = -ur[2];
    j0[0] = -2.0 * (ur[1] * t0[2] - ur[2] * t0[1]);
    j0[1] = -2.0 * (ur[2] * t0[0] - ur[0] * t0[2]);
    j0[2] = -2.0 * (ur[0] * t0[1] - ur[1] * t0[0]);
}

// Ground-plane height residual r = n . (R(q) p + t) + dist of landmark p against keyframe pose ps (7-vector) and plane pl
// (reference cost_functors_ceres.hpp:355-392); R, a = R p and px = a + t are kept for the Jacobian.
__device__ inline double gp_height(const double* ps, const double* pl, const double* p, double R[9], double a[3], double px[3]) {
    quat_to_rot<double>(ps, R);
    a[0] = R[0] * p[0] + R[1] * p[1] + R[2] * p[2];
    a[1] = R[3] * p[0] + R[4] * p[1] + R[5] * p[2];
    a[2] = R[6] * p[0] + R[7] * p[1] + R[8] * p[2];
    px[0] = a[0] + ps[4]; px[1] = a[1] + ps[5]; px[2] = a[2] + ps[6];
    return pl[0] * px[0] + pl[1] * px[1] + pl[2] * px[2] + pl[3];
}

// HuberLoss(ah) of a squared residual s (bundle_adjuster_keyframes.cpp:549): rho and rho'
__device__ inline void gp_huber(double s, double ah, double& rho, double& rho1) {
    if (s > ah * ah) { const double q = sqrt(s); rho = 2.0 * ah * q - ah * ah; rho1 = fmax(DBL_MIN, ah / q); }
    else { rho = s; rho1 = 1.0; }
}

// SpeedRegularizationVector2 (reference cost_functors_ceres.hpp:300-353): r = (R t_ob + t) / dt - v_before on one pose p;
// T_ob = the frozen speed_T_origin_before (7-vector), J (3x6, may be NULL) = local Jacobian (rot | trans).
__device__ inline void speed_regulariser(const double* p, const double* T_ob, const double* v_before, double dt, double r[3],
                                         double* J) {
    double R[9];
    quat_to_rot<double>(p, R);
    const double* tob = T_ob + 4;
    double a[3];
    for (int i = 0; i < 3; ++i) a[i] = R[3 * i] * tob[0] + R[3 * i + 1] * tob[1] + R[3 * i + 2] * tob[2];
    const double idt = 1.0 / dt;
    for (int i = 0; i < 3; ++i) r[i] = (a[i] + p[4 + i]) * idt - v_before[i];
    if (!J) return;
    // d/d(delta_rot) = -2 [a]x / dt, d/d(delta_t) = I / dt
    const double X[9] = {0, -a[2], a[1], a[2], 0, -a[0], -a[1], a[0], 0};
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            J[6 * i + j] = -2.0 * X[3 * i + j] * idt;
            J[6 * i + 3 + j] = (i == j) ? idt : 0.0;
        }
}

// Warp-cooperative J^T J / J^T r accumulation of one residual block (all 32 lanes pass identical arguments).
// parts: column offsets (or -1 for constant blocks) and sizes; J row-major nres x (sum of sizes), already times sqrt(rho').
template <typename Mat>
__device__ inline void warp_add_block(const Mat& A, double* fdiag, double* g, int nres, const double* r, int nparts,
                                      const int* off, const int* sz, const double* J, int lane) {
    int cols[16];
    double Jc[3][16];
    int m = 0, pos = 0, width = 0;
    for (int a = 0; a < nparts; ++a) width += sz[a];
    for (int a = 0; a < nparts; ++a) {
        for (int c = 0; c < sz[a]; ++c) {
            if (off[a] >= 0) {
                cols[m] = off[a] + c;
                for (int i = 0; i < nres; ++i) Jc[i][m] = J[i * width + pos + c];
                ++m;
            }
        }
        pos += sz[a];
    }
    for (int idx = lane; idx < m * m; idx += 32) {
        const int a = idx / m, b = idx - a * m;
        if (cols[b] > cols[a]) continue;
        double s = 0.0;
        for (int i = 0; i < nres; ++i) s += Jc[i][a] * Jc[i][b];
        A(cols[a], cols[b]) += s;
        if (a == b) {
            fdiag[cols[a]] += s;
            double t = 0.0;
            for (int i = 0; i < nres; ++i) t += Jc[i][a] * r[i];
            g[cols[a]] += t;
        }
    }
    __syncwarp();
}

// Robustified cost of the ground-plane regularisation chain at the given state (TrivialLoss * weight), for windows with
// plane_reg_weight > 0; single thread (called from the LM controller for the candidate, from warp 0 lane 0 at x).
__device__ inline double plane_chain_cost(const WinDesc& wd, const double* pose, const double* plane) {
    const double w = wd.plane_reg_weight;
    double c = 0.0;
    for (int k0 = 0; k0 + 1 < wd.n_kf; ++k0) {
        const double* n0 = plane + 4 * (size_t)(wd.kf_off + k0), *n1 = n0 + 4;
        const double dn[3] = {n1[0] - n0[0], n1[1] - n0[1], n1[2] - n0[2]};
        c += 0.5 * 3.0 * w * (dn[0] * dn[0] + dn[1] * dn[1] + dn[2] * dn[2]);
        const double dd = n1[3] - n0[3];
        c += 0.5 * w * dd * dd;
        const double rm = plane_motion(pose + 7 * (size_t)(wd.kf_off + k0), pose + 7 * (size_t)(wd.kf_off + k0 + 1), n0,
                                       nullptr, nullptr, nullptr);
        c += 0.5 * 2.0 * w * rm * rm;
    }
    for (int k = 0; k < wd.n_kf; ++k) {
        const double* n = plane + 4 * (size_t)(wd.kf_off + k);
        const double e[3] = {0.0 - n[0], 0.0 - n[1], 1.0 - n[2]};
        c += 0.5 * w * (e[0] * e[0] + e[1] * e[1] + e[2] * e[2]);
    }
    return c;
}

}  // namespace kba
