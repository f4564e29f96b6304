// kba_create.cu -- landmark creation of push() on the device-resident store (kba_track_create_landmarks, include/kba_b200.h):
// for every landmark the pushed keyframe measures for the first time, the back-projection of its first measurement with a lidar
// depth (calculateLandmark(kf, id), facade/bundle_adjuster_keyframes.cpp) or, without one, the triangulation of the rays of every
// listed keyframe and camera that measure it (calculateLandmark(id), triangulate_rays), from the keyframe poses, the measurement
// arena and the cameras the store already holds.  Created landmarks are written into the store with weight 1.
//
// Exactness: every floating-point operation is an explicit round-to-nearest intrinsic in the order of the facade's host code
// (internal/mini_eigen.hpp, g++ -O2 without FMA), and the file is compiled with -fmad=false, so that each position equals the
// host's bit for bit (a degenerate triangulation gives the host's inf or NaN).  A landmark's rays are visited in the host's
// order: keyframes in list order, entries of a keyframe in arena order (the caller's camera order).
//
// Windows: one launch sequence serves W requests (a track group's, kba_track_group_create_landmarks; a single call is W = 1),
// window w = blockIdx.z, as in kba_select.cu: grids from the maxima over the windows, threads beyond their window's sizes exit,
// every window's scratch is its own track's.
#include <cstdint>

#include "kba_exact.cuh"
#include "kba_kernels.h"

namespace kba {

namespace {

using namespace exact;

__device__ __forceinline__ const CreateArgs& win(const CreateLaunch& l) { return blockIdx.z == 0 ? l.w0 : l.rest[blockIdx.z - 1]; }

// Matrix3d::inverse() of mini_eigen: the cofactors over the determinant (row-major m, r)
__device__ void inverse3(const double* m, double* r) {
    const double d = da(ds(dm(m[0], ds(dm(m[4], m[8]), dm(m[5], m[7]))), dm(m[1], ds(dm(m[3], m[8]), dm(m[5], m[6])))),
                        dm(m[2], ds(dm(m[3], m[7]), dm(m[4], m[6]))));
    r[0] = __ddiv_rn(ds(dm(m[4], m[8]), dm(m[5], m[7])), d); r[1] = __ddiv_rn(ds(dm(m[2], m[7]), dm(m[1], m[8])), d);
    r[2] = __ddiv_rn(ds(dm(m[1], m[5]), dm(m[2], m[4])), d);
    r[3] = __ddiv_rn(ds(dm(m[5], m[6]), dm(m[3], m[8])), d); r[4] = __ddiv_rn(ds(dm(m[0], m[8]), dm(m[2], m[6])), d);
    r[5] = __ddiv_rn(ds(dm(m[2], m[3]), dm(m[0], m[5])), d);
    r[6] = __ddiv_rn(ds(dm(m[3], m[7]), dm(m[4], m[6])), d); r[7] = __ddiv_rn(ds(dm(m[1], m[6]), dm(m[0], m[7])), d);
    r[8] = __ddiv_rn(ds(dm(m[0], m[4]), dm(m[1], m[3])), d);
}

// Matrix3d * Vector3d: row i is (m0 p0 + m1 p1) + m2 p2
__device__ __forceinline__ double mv_row(const double* m, int i, double p0, double p1, double p2) {
    return da(da(dm(m[3 * i], p0), dm(m[3 * i + 1], p1)), dm(m[3 * i + 2], p2));
}

}  // namespace

// slot -> request map and counters; (cam * kf).inverse() of every listed keyframe and camera; intrin_inv of every camera
__global__ void __launch_bounds__(256) k_cr_init(const __grid_constant__ CreateLaunch l) {
    const CreateArgs& a = win(l);
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < a.n_new) {
        a.req_of[a.lm_slot[i]] = i;
        a.cnt[i] = 0; a.cursor[i] = 0;
    }
    if (i < a.n_kf * a.n_cam) {
        const int k = i / a.n_cam, c = i % a.n_cam;
        double C[12], K[12];
        iso_of_pose7(a.cam_pose7 + 7 * (size_t)c, C);
        iso_of_pose7(a.td.kf_pose + 7 * (size_t)a.kf_slot[k], K);
        // Isometry3d product: R = Rc Rk (each entry summed from 0), t = Rc tk + tc
        double R[9], t[3];
        for (int r = 0; r < 3; ++r) {
            for (int j = 0; j < 3; ++j) {
                double s = 0.0;
                for (int q = 0; q < 3; ++q) s = da(s, dm(C[3 * r + q], K[3 * q + j]));
                R[3 * r + j] = s;
            }
            t[r] = iso_row(C, r, K[9], K[10], K[11]);
        }
        // inverse: R^T, -(R^T t)
        double* T = a.ray_T + 12 * (size_t)i;
        for (int r = 0; r < 3; ++r) {
            for (int j = 0; j < 3; ++j) T[3 * r + j] = R[3 * j + r];
            T[9 + r] = -da(da(dm(R[r], t[0]), dm(R[3 + r], t[1])), dm(R[6 + r], t[2]));
        }
    }
    if (i < a.n_cam) {  // getIntrinsicMatrix(): Zero() with f, cx, f, cy, 1 set; then its inverse
        const double* in = a.cam_intr + 3 * (size_t)i;
        const double K[9] = {in[0], 0.0, in[1], 0.0, in[0], in[2], 0.0, 0.0, 1.0};
        inverse3(K, a.intr_inv + 9 * (size_t)i);
    }
    if (i == 0) *a.total = 0;
}

// arena entries of the requested landmarks in the listed keyframes, one thread per (entry, keyframe)
__global__ void __launch_bounds__(256) k_cr_count(const __grid_constant__ CreateLaunch l) {
    const CreateArgs& a = win(l);
    const int k = blockIdx.y;
    if (k >= a.n_kf) return;
    const int slot = a.kf_slot[k];
    const int n = a.td.m_cnt[slot], m0 = a.td.m_off[slot];
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int c = a.req_of[a.td.m_lm[m0 + i]];
        if (c >= 0) atomicAdd(&a.cnt[c], 1);
    }
}

// each request's place in the key array (any order)
__global__ void __launch_bounds__(256) k_cr_offsets(const __grid_constant__ CreateLaunch l) {
    const CreateArgs& a = win(l);
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c < a.n_new) a.off[c] = atomicAdd(a.total, a.cnt[c]);
}

// (keyframe position, arena index) keys of every request's entries behind its offset
__global__ void __launch_bounds__(256) k_cr_gather(const __grid_constant__ CreateLaunch l) {
    const CreateArgs& a = win(l);
    const int k = blockIdx.y;
    if (k >= a.n_kf) return;
    const int slot = a.kf_slot[k];
    const int n = a.td.m_cnt[slot], m0 = a.td.m_off[slot];
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int c = a.req_of[a.td.m_lm[m0 + i]];
        if (c >= 0) a.key[a.off[c] + atomicAdd(&a.cursor[c], 1)] = ((long long)k << 32) | (long long)(m0 + i);
    }
}

// one thread per requested landmark: its entries in host order (insertion sort of a few dozen keys), containsDepth on the pushed
// keyframe's entries, then the back-projection or the triangulation, the store write and the output.  Then the slot -> request
// map goes back to all -1 (k_cr_init filled it; the map is all -1 between calls, and create_run clears it if the sequence fails).
__global__ void __launch_bounds__(256) k_cr_land(const __grid_constant__ CreateLaunch l) {
    const CreateArgs& a = win(l);
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= a.n_new) return;
    long long* key = a.key + a.off[c];
    const int m = a.cnt[c];
    for (int i = 1; i < m; ++i) {
        const long long v = key[i];
        int j = i - 1;
        while (j >= 0 && key[j] > v) { key[j + 1] = key[j]; --j; }
        key[j + 1] = v;
    }
    // containsDepth: some entry of the pushed keyframe has d >= 0 (a NaN is no depth).  Then calculateLandmark(kf, id) takes the
    // first entry that is not skipped by its `d < 0` test: a NaN depth before the valid one is taken (and gives a NaN position),
    // exactly as on the host.
    bool has_depth = false;
    int depth_e = -1;
    for (int i = 0; i < m; ++i) {
        if ((int)(key[i] >> 32) != a.kf_new) continue;
        const int e = (int)(key[i] & 0xffffffffLL);
        const float d = a.td.m_d[e];
        has_depth |= d >= 0.f;
        if (depth_e < 0 && !(d < 0.f)) depth_e = e;
    }
    if (!has_depth) depth_e = -1;
    double p[3];
    unsigned char flags = 0;
    if (depth_e >= 0) {
        const int cam = a.td.m_cam[depth_e];
        const double* in = a.cam_intr + 3 * (size_t)cam;
        const double z = (double)a.td.m_d[depth_e];
        const double x = __ddiv_rn(dm(ds((double)a.td.m_u[depth_e], in[1]), z), in[0]);
        const double y = __ddiv_rn(dm(ds((double)a.td.m_v[depth_e], in[2]), z), in[0]);
        const double* T = a.ray_T + 12 * ((size_t)a.kf_new * a.n_cam + cam);
        for (int r = 0; r < 3; ++r) p[r] = iso_row(T, r, x, y, z);
        flags = 3;
    } else if (m >= 2) {  // calculateLandmark(id) with triangulate_rays: sum (I - r r^T), sum (I - r r^T) t, in ray order
        double S[9], rhs[3] = {0.0, 0.0, 0.0};
        for (int q = 0; q < 9; ++q) S[q] = 0.0;
        for (int i = 0; i < m; ++i) {
            const int k = (int)(key[i] >> 32), e = (int)(key[i] & 0xffffffffLL);
            const int cam = a.td.m_cam[e];
            const double* Ki = a.intr_inv + 9 * (size_t)cam;
            const double u = (double)a.td.m_u[e], v = (double)a.td.m_v[e];
            double ray[3];
            for (int r = 0; r < 3; ++r) ray[r] = mv_row(Ki, r, u, v, 1.0);
            const double nrm = __dsqrt_rn(da(da(dm(ray[0], ray[0]), dm(ray[1], ray[1])), dm(ray[2], ray[2])));
            for (int r = 0; r < 3; ++r) ray[r] = __ddiv_rn(ray[r], nrm);
            const double* T = a.ray_T + 12 * ((size_t)k * a.n_cam + cam);
            double rv[3], cur[9];
            for (int r = 0; r < 3; ++r) rv[r] = mv_row(T, r, ray[0], ray[1], ray[2]);
            for (int r = 0; r < 3; ++r)
                for (int j = 0; j < 3; ++j) cur[3 * r + j] = ds(r == j ? 1.0 : 0.0, dm(rv[r], rv[j]));
            for (int q = 0; q < 9; ++q) S[q] = da(S[q], cur[q]);
            for (int r = 0; r < 3; ++r) rhs[r] = da(rhs[r], mv_row(cur, r, T[9], T[10], T[11]));
        }
        double Si[9];
        inverse3(S, Si);
        for (int r = 0; r < 3; ++r) p[r] = mv_row(Si, r, rhs[0], rhs[1], rhs[2]);
        flags = 1;
    } else {
        for (int r = 0; r < 3; ++r) p[r] = __longlong_as_double(0x7ff8000000000000LL);
    }
    const int slot = a.lm_slot[c];
    if (flags & 1) {
        for (int r = 0; r < 3; ++r) a.td.lm_pos[3 * (size_t)slot + r] = p[r];
        a.td.lm_weight[slot] = 1.0;  // Landmark::weight's default
    }
    for (int r = 0; r < 3; ++r) a.pos[3 * (size_t)c + r] = p[r];
    a.flags[c] = flags;
    a.req_of[slot] = -1;
}

void launch_create(const CreateLaunch& l, const CreateGrid& g, cudaStream_t s) {
    const unsigned W = (unsigned)l.n_win;
    auto blocks = [](int n) { return (unsigned)(n > 0 ? (n + 255) / 256 : 1); };
    const dim3 gi(blocks(g.max_init), 1, W), gc(blocks(g.max_new), 1, W);
    const dim3 gm(blocks(g.max_meas), g.max_kf, W);
    k_cr_init<<<gi, 256, 0, s>>>(l); LCHK("k_cr_init");
    k_cr_count<<<gm, 256, 0, s>>>(l); LCHK("k_cr_count");
    k_cr_offsets<<<gc, 256, 0, s>>>(l); LCHK("k_cr_offsets");
    k_cr_gather<<<gm, 256, 0, s>>>(l); LCHK("k_cr_gather");
    k_cr_land<<<gc, 256, 0, s>>>(l); LCHK("k_cr_land");
}

}  // namespace kba
