// kba_depth_cost.cuh -- limo's AddDepth sorter on the device: std::max(-DBL_MAX, double(float(|kf * pos|))) (mono_lidar.cpp:418-429
// with the scheme's fold over a keyframe's cameras, landmark_selection_scheme_add_depth.cpp:16-75).  Round-to-nearest intrinsics in
// mini_eigen's order for Isometry3d * Vector3d and norm(); the including files are compiled with -fmad=false.  Shared by
// kba_track_depth_costs (kba_upkeep.cu) and the ranked selection (kba_rank.cu), so that both give the same bits.
#pragma once
#include <cfloat>

#include "kba_exact.cuh"

namespace kba {

// T: the keyframe's transform (iso_of_pose7), p: the landmark's position.  A NaN norm leaves -DBL_MAX.
__device__ __forceinline__ double depth_cost(const double* T, const double* p) {
    using namespace exact;
    const double x = iso_row(T, 0, p[0], p[1], p[2]), y = iso_row(T, 1, p[0], p[1], p[2]), z = iso_row(T, 2, p[0], p[1], p[2]);
    const double v = (double)__double2float_rn(__dsqrt_rn(da(da(dm(x, x), dm(y, y)), dm(z, z))));
    return -DBL_MAX < v ? v : -DBL_MAX;
}

}  // namespace kba
