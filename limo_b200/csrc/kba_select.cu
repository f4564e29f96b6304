// kba_select.cu -- landmark selection on the device-resident store (kba_track_select_landmarks, include/kba_b200.h): the
// per-landmark quantities of limo's production chain (LandmarkRejectionSchemeCheirality, then the steps 1-5 of
// LandmarkSparsificationSchemeVoxel, facade/landmark_selection.cpp) from the keyframe poses, the measurement arena and the
// landmark positions the store already holds.  The host keeps the ranking (partial sorts, the std::rand shuffle, the caps).
//
// Exactness: every floating-point operation is an explicit round-to-nearest intrinsic in the order of the facade's host code
// (internal/mini_eigen.hpp, g++ -O2 without FMA), and the file is compiled with -fmad=false, so that each quantity equals the
// host's bit for bit.  Only integer atomics; every order-dependent step (voxel centroids, the near order, flow sums) runs in
// a fixed order.
//
// Windows: one launch sequence serves W requests (a track group's, kba_track_group_select_landmarks; a single call is W = 1),
// window w = blockIdx.z.  Grids are sized from the maxima over the windows and threads beyond their own window's sizes exit.
// A window's counters live in its output block and its bounds, slot map and the rest of its scratch in its track's buffers:
// no two windows share a word (a group lists a track once).
#include <cfloat>
#include <cstdint>

#include "kba_exact.cuh"
#include "kba_kernels.h"

namespace kba {

namespace {

using namespace exact;

__device__ __forceinline__ double sq3(double x, double y, double z) { return da(da(dm(x, x), dm(y, y)), dm(z, z)); }

// distance_to_path of the voxel scheme (boost::geometry::distance(point, linestring) as the facade restates it)
__device__ double path_distance(double qx, double qy, double qz, const double* path, int n) {
    if (n == 1) return __dsqrt_rn(sq3(ds(qx, path[0]), ds(qy, path[1]), ds(qz, path[2])));
    double best = DBL_MAX;
    for (int i = 0; i + 1 < n; ++i) {
        const double* a = path + 3 * i, *b = a + 3;
        const double vx = ds(b[0], a[0]), vy = ds(b[1], a[1]), vz = ds(b[2], a[2]);
        const double wx = ds(qx, a[0]), wy = ds(qy, a[1]), wz = ds(qz, a[2]);
        const double c1 = da(da(dm(wx, vx), dm(wy, vy)), dm(wz, vz)), c2 = da(da(dm(vx, vx), dm(vy, vy)), dm(vz, vz));
        double d2;
        if (c1 <= 0.) d2 = sq3(wx, wy, wz);
        else if (c2 <= c1) d2 = sq3(ds(qx, b[0]), ds(qy, b[1]), ds(qz, b[2]));
        else {
            const double t = __ddiv_rn(c1, c2);
            d2 = sq3(ds(qx, da(a[0], dm(vx, t))), ds(qy, da(a[1], dm(vy, t))), ds(qz, da(a[2], dm(vz, t))));
        }
        best = d2 < best ? d2 : best;  // std::min(best, d2)
    }
    return __dsqrt_rn(best);
}

// float <-> unsigned with the order of the floats (integer atomics for the cloud's bounding box)
__device__ __forceinline__ unsigned f2o(float f) {
    const unsigned u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float o2f(unsigned o) { return __uint_as_float((o & 0x80000000u) ? (o & 0x7fffffffu) : ~o); }

// the voxel grid's per-axis constants (voxel_grid of the facade: float leaf inverse, floor of the scaled bounds)
struct Grid {
    float inv[3];
    int min_b[3];
    long long mul[3];
};
__device__ Grid grid_of(const SelectArgs& a) {
    Grid g;
    int div_b[3];
    for (int q = 0; q < 3; ++q) {
        g.inv[q] = __fdiv_rn(1.0f, __double2float_rn(a.leaf[q]));
        g.min_b[q] = __float2int_rz(floorf(__fmul_rn(o2f(a.bounds[q]), g.inv[q])));
        div_b[q] = __float2int_rz(floorf(__fmul_rn(o2f(a.bounds[3 + q]), g.inv[q]))) - g.min_b[q] + 1;
    }
    g.mul[0] = 1; g.mul[1] = div_b[0]; g.mul[2] = (long long)div_b[0] * div_b[1];
    return g;
}

// the arguments of this block's window (the launch parameters are __grid_constant__, so window 0's are read in place)
__device__ __forceinline__ const SelectArgs& win(const SelectLaunch& l) {
    return l.all ? l.all[blockIdx.z] : (blockIdx.z == 0 ? l.w0 : l.rest[blockIdx.z - 1]);
}

}  // namespace

// slot -> candidate map, output defaults, keyframe and camera transforms, the keyframe path seen from the newest keyframe
__global__ void __launch_bounds__(256) k_sel_init(const __grid_constant__ SelectLaunch l) {
    const SelectArgs& a = win(l);
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < a.n_cand) {
        a.cand_of[a.lm_slot[i]] = i;
        a.cheiral[i] = 1; a.bin[i] = -1; a.flow[i] = __longlong_as_double(0x7ff8000000000000LL); a.seen[i] = 0;
        a.near_order[i] = -1; a.cnt[i] = 0; a.cursor[i] = 0;
    }
    if (i < a.n_kf) {
        double* T = a.kf_T + 12 * (size_t)i;
        iso_of_pose7(a.td.kf_pose + 7 * (size_t)a.kf_slot[i], T);
        double C[12];
        iso_of_pose7(a.td.kf_pose + 7 * (size_t)a.kf_slot[a.n_kf - 1], C);
        // cur * kf.inverse().translation(): inverse t = -(R^T t)
        double it[3];
        for (int r = 0; r < 3; ++r) it[r] = -da(da(dm(T[r], T[9]), dm(T[3 + r], T[10])), dm(T[6 + r], T[11]));
        for (int r = 0; r < 3; ++r) a.path[3 * (size_t)i + r] = iso_row(C, r, it[0], it[1], it[2]);
    }
    if (i < a.n_cam) iso_of_pose7(a.cam_pose7 + 7 * i, a.cam_T + 12 * i);
    if (i == 0) {
        for (int q = 0; q < 3; ++q) { a.bounds[q] = 0xffffffffu; a.bounds[3 + q] = 0u; }
        a.counters[0] = 0; a.counters[1] = 0; a.counters[2] = 0;
    }
}

// Cheirality (landmark_selection.cpp:17-31): every arena entry of an active keyframe that measures a candidate, one thread per
// entry: z of cam * (kf * pos) < 0 clears the flag.  Also the candidate's observation count (flow gather) and, on the first entry
// of its run in the keyframe (entries come in landmark-id order), one more keyframe that measures it (chooseFarLmIds).
__global__ void __launch_bounds__(256) k_sel_cheiral(const __grid_constant__ SelectLaunch l) {
    const SelectArgs& a = win(l);
    const int k = blockIdx.y;
    if (k >= a.n_kf) return;
    const int slot = a.kf_slot[k];
    const int n = a.td.m_cnt[slot], m0 = a.td.m_off[slot];
    const double* T = a.kf_T + 12 * (size_t)k;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int lm = a.td.m_lm[m0 + i];
        const int c = a.cand_of[lm];
        if (c < 0) continue;
        const double* p = a.td.lm_pos + 3 * (size_t)lm;
        const double vx = iso_row(T, 0, p[0], p[1], p[2]), vy = iso_row(T, 1, p[0], p[1], p[2]), vz = iso_row(T, 2, p[0], p[1], p[2]);
        const double z = iso_row(a.cam_T + 12 * a.td.m_cam[m0 + i], 2, vx, vy, vz);
        if (z < 0.) a.cheiral[c] = 0;
        atomicAdd(&a.cnt[c], 1);
        if (i == 0 || a.td.m_lm[m0 + i - 1] != lm) atomicAdd(&a.seen[c], 1);
    }
}

// Voxel scheme steps 1-3 on the survivors: into the newest keyframe's frame (double, rounded to float), PassThrough z in
// [-20, 100], far bin = not closer than roi_far to the path.  The rest joins the voxel cloud: its bounding box by integer
// atomics on order-preserving bit patterns, its list in any order (the rank sort fixes the order).
__global__ void __launch_bounds__(256) k_sel_points(const __grid_constant__ SelectLaunch l) {
    const SelectArgs& a = win(l);
    if ((int)(blockIdx.x * blockDim.x) >= a.n_cand) return;  // whole blocks only: every warp below takes part in the reductions
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    bool inside = false;
    float f[3] = {0.f, 0.f, 0.f};
    if (c < a.n_cand && a.cheiral[c]) {
        const double* p = a.td.lm_pos + 3 * (size_t)a.lm_slot[c];
        const double* C = a.kf_T + 12 * (size_t)(a.n_kf - 1);
        for (int r = 0; r < 3; ++r) f[r] = __double2float_rn(iso_row(C, r, p[0], p[1], p[2]));
        if (isfinite(f[2]) && f[2] >= -20.f && f[2] <= 100.f) {
            const double d = path_distance((double)f[0], (double)f[1], (double)f[2], a.path, a.n_kf);
            if (d < a.roi_far) {
                inside = true;
                const int r = atomicAdd(&a.counters[0], 1);
                a.in_list[r] = c;
                for (int q = 0; q < 3; ++q) a.pt[3 * (size_t)c + q] = f[q];
            } else {
                a.bin[c] = 2;
            }
        }
    }
    for (int q = 0; q < 3; ++q) {
        const unsigned lo = __reduce_min_sync(0xffffffffu, inside ? f2o(f[q]) : 0xffffffffu);
        const unsigned hi = __reduce_max_sync(0xffffffffu, inside ? f2o(f[q]) : 0u);
        if ((threadIdx.x & 31) == 0 && lo != 0xffffffffu) { atomicMin(&a.bounds[q], lo); atomicMax(&a.bounds[3 + q], hi); }
    }
}

// voxel index of every cloud point, relative to the cloud's minimum (voxel_grid: float floor, truncation to int)
__global__ void __launch_bounds__(256) k_sel_vkey(const __grid_constant__ SelectLaunch l) {
    const SelectArgs& a = win(l);
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= a.counters[0]) return;
    const Grid g = grid_of(a);
    const int c = a.in_list[r];
    long long idx = 0;
    for (int q = 0; q < 3; ++q) {
        const float t = __fsub_rn(floorf(__fmul_rn(a.pt[3 * (size_t)c + q], g.inv[q])), __int2float_rn(g.min_b[q]));
        idx += (long long)__float2int_rz(t) * g.mul[q];
    }
    a.vkey[r] = idx;
}

// std::sort of the (voxel index, label) pairs, as a rank: each point counts the points ordered before it (labels are unique and
// ascend with the candidate index).  O(n^2) comparisons from shared-memory tiles -- a few dozen microseconds for 20k points.
__global__ void __launch_bounds__(256) k_sel_rank(const __grid_constant__ SelectLaunch l) {
    const SelectArgs& a = win(l);
    __shared__ long long s_key[256];
    __shared__ int s_lab[256];
    const int n = a.counters[0];
    if ((int)(blockIdx.x * blockDim.x) >= n) return;
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    const long long key = r < n ? a.vkey[r] : 0;
    const int lab = r < n ? a.in_list[r] : 0;
    int rank = 0;
    for (int t0 = 0; t0 < n; t0 += 256) {
        const int j = t0 + threadIdx.x;
        s_key[threadIdx.x] = j < n ? a.vkey[j] : LLONG_MAX;
        s_lab[threadIdx.x] = j < n ? a.in_list[j] : INT_MAX;
        __syncthreads();
        const int m = n - t0 < 256 ? n - t0 : 256;
        for (int q = 0; q < m; ++q) {
            const long long kq = s_key[q];
            rank += (kq < key) | ((kq == key) & (s_lab[q] < lab));
        }
        __syncthreads();
    }
    if (r < n) a.sorted[rank] = r;
}

// one point per voxel (step 4): the first point of each run of equal voxel indices sums its run in sorted order (float), its
// label is the run's smallest; step 5: middle bin = centroid not closer than roi_middle to the path, near bin = the others
__global__ void __launch_bounds__(256) k_sel_voxels(const __grid_constant__ SelectLaunch l) {
    const SelectArgs& a = win(l);
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    const int n = a.counters[0];
    if (r >= n) return;
    const long long key = a.vkey[a.sorted[r]];
    a.near_flag[r] = 0;
    if (r > 0 && a.vkey[a.sorted[r - 1]] == key) return;
    float sx = 0.f, sy = 0.f, sz = 0.f;
    int b = r;
    for (; b < n && a.vkey[a.sorted[b]] == key; ++b) {
        const float* p = a.pt + 3 * (size_t)a.in_list[a.sorted[b]];
        sx = __fadd_rn(sx, p[0]); sy = __fadd_rn(sy, p[1]); sz = __fadd_rn(sz, p[2]);
    }
    const float cnt = __int2float_rn(b - r);
    const float cx = __fdiv_rn(sx, cnt), cy = __fdiv_rn(sy, cnt), cz = __fdiv_rn(sz, cnt);
    const int c = a.in_list[a.sorted[r]];
    if (path_distance((double)cx, (double)cy, (double)cz, a.path, a.n_kf) < a.roi_middle) {
        a.bin[c] = 0;
        a.near_flag[r] = 1;
        a.obs_off[c] = atomicAdd(&a.counters[2], a.cnt[c]);  // its observations' place in the flow gather (any order)
    } else {
        a.bin[c] = 1;
    }
}

// the near bin in ascending voxel index: an ordered compaction of the near flags, one CTA per window
__global__ void __launch_bounds__(1024) k_sel_near_order(const __grid_constant__ SelectLaunch l) {
    const SelectArgs& a = win(l);
    __shared__ int s_scan[1024];
    const int n = a.counters[0], tid = threadIdx.x;
    int carry = 0;
    for (int c0 = 0; c0 < n; c0 += 1024) {
        const int r = c0 + tid;
        const int f = r < n ? a.near_flag[r] : 0;
        s_scan[tid] = f;
        __syncthreads();
        for (int off = 1; off < 1024; off <<= 1) {
            const int v = tid >= off ? s_scan[tid - off] : 0;
            __syncthreads();
            s_scan[tid] += v;
            __syncthreads();
        }
        if (f) a.near_order[carry + s_scan[tid] - 1] = a.in_list[a.sorted[r]];
        const int tot = s_scan[1023];
        __syncthreads();
        carry += tot;
    }
    if (tid == 0) a.counters[1] = carry;
}

// the observations of every near landmark, (keyframe position, arena index) keys behind its offset
__global__ void __launch_bounds__(256) k_sel_gather(const __grid_constant__ SelectLaunch l) {
    const SelectArgs& a = win(l);
    const int k = blockIdx.y;
    if (k >= a.n_kf) return;
    const int slot = a.kf_slot[k];
    const int n = a.td.m_cnt[slot], m0 = a.td.m_off[slot];
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int c = a.cand_of[a.td.m_lm[m0 + i]];
        if (c < 0 || a.bin[c] != 0) continue;
        a.okey[a.obs_off[c] + atomicAdd(&a.cursor[c], 1)] = ((long long)k << 32) | (long long)(m0 + i);
    }
}

// calcFlow(use_mean = false) of a near landmark: its observations in time order (insertion sort of a few dozen keys), per camera
// the sum of the double norms between consecutive observations, the maximum over the cameras in index order (max_element with
// `<`); NaN when no camera saw it twice.  Then the slot -> candidate map goes back to all -1.
__global__ void __launch_bounds__(256) k_sel_flow(const __grid_constant__ SelectLaunch l) {
    const SelectArgs& a = win(l);
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= a.n_cand) return;
    if (a.bin[c] == 0) {
        long long* key = a.okey + a.obs_off[c];
        const int m = a.cnt[c];
        for (int i = 1; i < m; ++i) {
            const long long v = key[i];
            int j = i - 1;
            while (j >= 0 && key[j] > v) { key[j + 1] = key[j]; --j; }
            key[j + 1] = v;
        }
        bool any = false;
        double best = 0.;
        for (int cam = 0; cam < a.n_cam; ++cam) {
            bool has_last = false, has_flow = false;
            float lu = 0.f, lv = 0.f;
            double sum = 0.;
            for (int i = 0; i < m; ++i) {
                const int e = (int)(key[i] & 0xffffffffLL);
                if (a.td.m_cam[e] != cam) continue;
                const float u = a.td.m_u[e], v = a.td.m_v[e];
                if (has_last) {
                    const double du = ds((double)lu, (double)u), dv = ds((double)lv, (double)v);
                    sum = da(sum, __dsqrt_rn(da(dm(du, du), dm(dv, dv))));
                    has_flow = true;
                }
                lu = u; lv = v; has_last = true;
            }
            if (!has_flow) continue;
            if (!any || best < sum) best = sum;
            any = true;
        }
        if (any) a.flow[c] = best;
    }
    a.cand_of[a.lm_slot[c]] = -1;
}

void launch_select(const SelectLaunch& l, const SelectGrid& g, cudaStream_t s) {
    const unsigned W = (unsigned)l.n_win;
    const dim3 gi((g.max_init + 255) / 256, 1, W);
    const dim3 gc((g.max_cand > 0 ? g.max_cand + 255 : 256) / 256, 1, W);
    const dim3 gm((g.max_meas + 255) / 256 > 0 ? (g.max_meas + 255) / 256 : 1, g.max_kf, W);
    k_sel_init<<<gi, 256, 0, s>>>(l); LCHK("k_sel_init");
    k_sel_cheiral<<<gm, 256, 0, s>>>(l); LCHK("k_sel_cheiral");
    k_sel_points<<<gc, 256, 0, s>>>(l); LCHK("k_sel_points");
    k_sel_vkey<<<gc, 256, 0, s>>>(l); LCHK("k_sel_vkey");
    k_sel_rank<<<gc, 256, 0, s>>>(l); LCHK("k_sel_rank");
    k_sel_voxels<<<gc, 256, 0, s>>>(l); LCHK("k_sel_voxels");
    k_sel_near_order<<<dim3(1, 1, W), 1024, 0, s>>>(l); LCHK("k_sel_near_order");
    k_sel_gather<<<gm, 256, 0, s>>>(l); LCHK("k_sel_gather");
    k_sel_flow<<<gc, 256, 0, s>>>(l); LCHK("k_sel_flow");
}

}  // namespace kba
