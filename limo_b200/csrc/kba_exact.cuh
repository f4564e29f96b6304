// kba_exact.cuh -- the facade's host arithmetic (internal/mini_eigen.hpp, g++ -O2 without FMA) as explicit round-to-nearest
// double operations, for the kernels whose results must equal the host's bit for bit (kba_select.cu, kba_create.cu).  Include it
// only from files compiled with -fmad=false.
#pragma once

namespace kba {
namespace exact {

__device__ __forceinline__ double dm(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double da(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double ds(double a, double b) { return __dsub_rn(a, b); }

// convert(Pose) of the facade (definitions.cpp: Identity().translate(t).rotate(q), Eigen's un-normalised toRotationMatrix) as
// R (row-major) and t in T[0..12); the products with the identity are kept, as in k_track_ground
__device__ inline void iso_of_pose7(const double* q, double* T) {
    const double qw = q[0], qx = q[1], qy = q[2], qz = q[3];
    const double tx = dm(2.0, qx), ty = dm(2.0, qy), tz = dm(2.0, qz);
    const double twx = dm(tx, qw), twy = dm(ty, qw), twz = dm(tz, qw);
    const double txx = dm(tx, qx), txy = dm(ty, qx), txz = dm(tz, qx);
    const double tyy = dm(ty, qy), tyz = dm(tz, qy), tzz = dm(tz, qz);
    const double Rq[9] = {ds(1.0, da(tyy, tzz)), ds(txy, twz), da(txz, twy),
                          da(txy, twz), ds(1.0, da(txx, tzz)), ds(tyz, twx),
                          ds(txz, twy), da(tyz, twx), ds(1.0, da(txx, tyy))};
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) {
            double s = 0.0;
            for (int k = 0; k < 3; ++k) s = da(s, dm(i == k ? 1.0 : 0.0, Rq[3 * k + j]));
            T[3 * i + j] = s;
        }
        const double Iv = da(da(dm(i == 0 ? 1.0 : 0.0, q[4]), dm(i == 1 ? 1.0 : 0.0, q[5])), dm(i == 2 ? 1.0 : 0.0, q[6]));
        T[9 + i] = da(0.0, Iv);
    }
}

// Isometry3d * Vector3d: R * p + t, each row ((r0 p0 + r1 p1) + r2 p2) + t
__device__ __forceinline__ double iso_row(const double* T, int i, double px, double py, double pz) {
    return da(da(da(dm(T[3 * i], px), dm(T[3 * i + 1], py)), dm(T[3 * i + 2], pz)), T[9 + i]);
}

}  // namespace exact
}  // namespace kba
