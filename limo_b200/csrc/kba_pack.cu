// kba_pack.cu -- window packing on the device (SURVEY 8(f) row 3; replaces the host loops of fill_window in kba_api.cu for
// batches on the fused small-window path and for the large-window solver of a track).  The caller's window arrives as it is -- landmark-major CSR in the caller's landmark
// order (what addKeyframeToProblem enumerates, reference bundle_adjuster_keyframes.cpp:564-627) -- with ONE copy per array;
// everything the solver derives from it is built here:
//   k_pack_sort      : landmarks ordered by (first, last) observing keyframe (32-bit keys: 8 + 8 bits keyframes, 15 bits
//                      index -> stable and unique), bitonic sort in shared memory, one CTA per window; new CSR pointers by a
//                      block scan; the inverse permutation
//   k_pack_obs       : observations copied into the new landmark-major order (+ landmark index, rank inside a rig, origin)
//   k_pack_kf_count / k_pack_kf_fill : the keyframe-major copy read by k_pose_hessian, in landmark-major order inside each
//                      keyframe (deterministic reductions), by a block-wide ordered compaction per (keyframe, window)
//   k_pack_gp        : ground-plane residuals follow their landmark; shared-row flags
//   k_pack_ranges    : keyframe range of every 8-landmark group (fused path) or 32-landmark chunk (large-window path)
// Integer work only; every kernel is a streaming pass over 4-byte words (a config-2 window: 40k observations x ~50 B).
#include <cfloat>
#include <cstdint>

#include <cuda_runtime.h>

#include "kba_device.cuh"
#include "kba_kernels.h"

namespace kba {

__global__ void __launch_bounds__(1024) k_pack_sort(BatchDev bd, PackRaw raw) {
    const int w = blockIdx.x;
    const WinDesc& wd = bd.desc[w];
    extern __shared__ unsigned s_key[];  // [n_pow2]
    __shared__ int s_scan[1024];
    const int n = wd.n_lm, tid = threadIdx.x, nth = blockDim.x;
    int np = 1;
    while (np < n) np <<= 1;
    const int* rp = raw.lm_ptr + wd.lm_off + w;
    const int* rkf = raw.obs_kf + wd.obs_off;
    for (int j = tid; j < np; j += nth) {
        unsigned key = 0xffffffffu;  // padding sorts last
        if (j < n) {
            const int o0 = rp[j], o1 = rp[j + 1];
            const unsigned k0 = o1 > o0 ? (unsigned)rkf[o0] : (unsigned)wd.n_kf, k1 = o1 > o0 ? (unsigned)rkf[o1 - 1] : (unsigned)wd.n_kf;
            key = (k0 << 23) | (k1 << 15) | (unsigned)j;
        }
        s_key[j] = key;
    }
    __syncthreads();
    for (int k = 2; k <= np; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = tid; i < np; i += nth) {
                const int l = i ^ j;
                if (l > i) {
                    const unsigned a = s_key[i], b = s_key[l];
                    const bool up = (i & k) == 0;
                    if ((a > b) == up) { s_key[i] = b; s_key[l] = a; }
                }
            }
            __syncthreads();
        }
    // new order: position jn holds caller landmark orig; CSR pointers by a chunked block scan of the track lengths
    int* lp = bd.lm_ptr + wd.lm_off + w;
    int carry = 0;
    for (int c0 = 0; c0 < n; c0 += nth) {
        const int jn = c0 + tid;
        int len = 0, orig = 0;
        if (jn < n) {
            orig = (int)(s_key[jn] & 0x7fffu);
            len = rp[orig + 1] - rp[orig];
            bd.lm_orig[wd.lm_off + jn] = orig;
            raw.lm_inv[wd.lm_off + orig] = jn;
            bd.lm0[3 * (size_t)(wd.lm_off + jn) + 0] = raw.lm_pos[3 * (size_t)(wd.lm_off + orig) + 0];
            bd.lm0[3 * (size_t)(wd.lm_off + jn) + 1] = raw.lm_pos[3 * (size_t)(wd.lm_off + orig) + 1];
            bd.lm0[3 * (size_t)(wd.lm_off + jn) + 2] = raw.lm_pos[3 * (size_t)(wd.lm_off + orig) + 2];
            bd.lm_weight[wd.lm_off + jn] = raw.lm_weight[wd.lm_off + orig];
            bd.gp_of_lm[wd.lm_off + jn] = -1;
        }
        s_scan[tid] = len;
        __syncthreads();
        for (int off = 1; off < nth; off <<= 1) {  // Hillis-Steele inclusive scan
            const int v = tid >= off ? s_scan[tid - off] : 0;
            __syncthreads();
            s_scan[tid] += v;
            __syncthreads();
        }
        if (jn < n) lp[jn + 1] = carry + s_scan[tid];
        const int tot = s_scan[nth - 1];
        __syncthreads();
        carry += tot;
    }
    if (tid == 0) lp[0] = 0;
}

// one warp per landmark (new order): its observations keep their order (keyframe, then camera)
__global__ void __launch_bounds__(256) k_pack_obs(BatchDev bd, PackRaw raw) {
    const int w = blockIdx.y;
    const WinDesc& wd = bd.desc[w];
    const int lane = threadIdx.x & 31, jn = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (jn >= wd.n_lm) return;
    const int orig = bd.lm_orig[wd.lm_off + jn];
    const int* rp = raw.lm_ptr + wd.lm_off + w;
    const int s0 = rp[orig], s1 = rp[orig + 1];
    const int d0 = (bd.lm_ptr + wd.lm_off + w)[jn];
    const size_t ob = (size_t)wd.obs_off;
    for (int i = lane; i < s1 - s0; i += 32) {
        const size_t src = ob + s0 + i, dst = ob + d0 + i;
        const int kf = raw.obs_kf[src];
        bd.obs_kf[dst] = kf;
        bd.obs_cam[dst] = raw.obs_cam[src];
        bd.obs_lm[dst] = jn;
        bd.obs_u[dst] = raw.obs_u[src]; bd.obs_v[dst] = raw.obs_v[src]; bd.obs_d[dst] = raw.obs_d[src];
        int rank = 0;  // position among the landmark's observations in the same keyframe (rigs)
        for (int q = i - 1; q >= 0 && raw.obs_kf[ob + s0 + q] == kf; --q) ++rank;
        bd.obs_rank[dst] = rank;
        if (raw.obs_orig) raw.obs_orig[dst] = s0 + i;
    }
}

__global__ void __launch_bounds__(256) k_pack_kf_count(BatchDev bd) {
    const int w = blockIdx.x;
    const WinDesc& wd = bd.desc[w];
    __shared__ int s_cnt[kMaxKf + 1];
    for (int k = threadIdx.x; k <= kMaxKf; k += blockDim.x) s_cnt[k] = 0;
    __syncthreads();
    for (int o = threadIdx.x; o < wd.n_obs; o += blockDim.x) atomicAdd(&s_cnt[bd.obs_kf[(size_t)wd.obs_off + o]], 1);
    __syncthreads();
    if (threadIdx.x == 0) {
        int* kp = bd.kf_ptr + wd.kf_off + w;
        int acc = 0;
        for (int k = 0; k < wd.n_kf; ++k) { kp[k] = acc; acc += s_cnt[k]; }
        kp[wd.n_kf] = acc;
    }
}

// keyframe-major copy: CTA (k, w) walks the window's observations in landmark-major order and keeps those of keyframe k
__global__ void __launch_bounds__(256) k_pack_kf_fill(BatchDev bd) {
    const int w = blockIdx.y, k = blockIdx.x;
    const WinDesc& wd = bd.desc[w];
    if (k >= wd.n_kf) return;
    __shared__ int s_warp[8];
    __shared__ int s_base;
    const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
    const size_t ob = (size_t)wd.obs_off;
    if (threadIdx.x == 0) s_base = (bd.kf_ptr + wd.kf_off + w)[k];
    __syncthreads();
    for (int o0 = 0; o0 < wd.n_obs; o0 += 256) {
        const int o = o0 + threadIdx.x;
        const bool mine = o < wd.n_obs && bd.obs_kf[ob + o] == k;
        const unsigned m = __ballot_sync(0xffffffffu, mine);
        if (lane == 0) s_warp[wp] = __popc(m);
        __syncthreads();
        int before = 0, total = 0;
        for (int q = 0; q < 8; ++q) { const int c = s_warp[q]; if (q < wp) before += c; total += c; }
        if (mine) {
            const size_t e = ob + s_base + before + __popc(m & ((1u << lane) - 1));
            bd.pm_lm[e] = bd.obs_lm[ob + o];
            bd.pm_cam[e] = bd.obs_cam[ob + o];
            bd.pm_u[e] = bd.obs_u[ob + o]; bd.pm_v[e] = bd.obs_v[ob + o]; bd.pm_d[e] = bd.obs_d[ob + o];
        }
        __syncthreads();
        if (threadIdx.x == 0) s_base += total;
        __syncthreads();
    }
}

__global__ void __launch_bounds__(256) k_pack_gp(BatchDev bd, PackRaw raw) {
    const int w = blockIdx.y;
    const WinDesc& wd = bd.desc[w];
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= wd.n_gp) return;
    const size_t G = (size_t)wd.gp_off + g;
    const int jn = raw.lm_inv[wd.lm_off + raw.gp_lm[G]];
    bd.gp_lm[G] = jn;
    bd.gp_of_lm[wd.lm_off + jn] = g;
    const int* lp = bd.lm_ptr + wd.lm_off + w;
    int shared = 0;
    for (int o = lp[jn]; o < lp[jn + 1]; ++o) shared |= (bd.obs_kf[(size_t)wd.obs_off + o] == bd.gp_kf[G]);
    bd.gp_shared[G] = shared;
}

// keyframe range [k0, k1] of every kWidth-landmark unit (observations + the ground-plane keyframes of its landmarks): the 8-landmark
// groups of the fused Schur kernel, or the 32-landmark chunks of the large-window path (k_solve_begin, k_schur_syrk), which also get
// their landmark range.  Runs after k_pack_gp (gp_of_lm).
template <int kWidth>
__global__ void __launch_bounds__(256) k_pack_ranges(BatchDev bd) {
    const int w = blockIdx.y;
    const WinDesc& wd = bd.desc[w];
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= (kWidth == 8 ? wd.n_groups : wd.n_chunks)) return;
    const int* lp = bd.lm_ptr + wd.lm_off + w;
    const int j0 = c * kWidth, j1 = min(wd.n_lm, j0 + kWidth);
    int k0 = wd.n_kf, k1 = -1;
    for (int o = lp[j0]; o < lp[j1]; ++o) {
        const int k = bd.obs_kf[(size_t)wd.obs_off + o];
        k0 = min(k0, k); k1 = max(k1, k);
    }
    if (wd.n_gp > 0)
        for (int j = j0; j < j1; ++j) {
            const int g = bd.gp_of_lm[wd.lm_off + j];
            if (g >= 0) { const int k = bd.gp_kf[wd.gp_off + g]; k0 = min(k0, k); k1 = max(k1, k); }
        }
    if (kWidth == 8) {
        bd.grp_k0[wd.grp_off + c] = k0;
        bd.grp_k1[wd.grp_off + c] = k1;
    } else {
        const size_t C = (size_t)wd.chunk_off + c;
        bd.chunk_lm0[C] = j0; bd.chunk_lm1[C] = j1;
        bd.chunk_k0[C] = k0; bd.chunk_k1[C] = k1;
    }
}

// landmark results back into the caller's order, so that the download is one plain copy per array
__global__ void __launch_bounds__(256) k_unpack_landmarks(BatchDev bd, double* lm_user, unsigned char* rejected_user) {
    const int w = blockIdx.y;
    const WinDesc& wd = bd.desc[w];
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= wd.n_lm) return;
    const int L = wd.lm_off + j, U = wd.lm_off + bd.lm_orig[L];
    const double* p = bd.lm[bd.state[w].cur] + 3 * (size_t)L;
    lm_user[3 * (size_t)U] = p[0]; lm_user[3 * (size_t)U + 1] = p[1]; lm_user[3 * (size_t)U + 2] = p[2];
    rejected_user[U] = !bd.lm_active[L];
}

// =====================================================================================================================
// persistent window (kba_track_*): the window's raw CSR is gathered on the device from the measurement arena
// =====================================================================================================================
// Every kernel takes window w of the batch from its grid (blockIdx.y, or .z where .y is taken) and that window's track store
// tds[w] and selection sels[w]: one window for kba_track_solve, one per track for kba_track_group_solve.  Writes go through
// desc[w]'s offsets; the per-track scratch (sel_index, cursor, key, n_depth) is indexed window-locally -- a track is in a batch
// at most once, so no two windows share it.  An idle window (a track sitting a group solve out) has empty selections.
__global__ void __launch_bounds__(256) k_track_begin(BatchDev bd, const TrackDev* tds, const TrackSel* sels, double* r_lm_pos,
                                                     double* r_lm_weight, int* r_cnt) {
    const int w = blockIdx.y;
    const WinDesc& wd = bd.desc[w];
    if (wd.idle) return;
    const TrackDev& td = tds[w];
    const TrackSel& sel = sels[w];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < sel.n_kf) {
        const int slot = sel.kf_slot[i];
        const size_t k = (size_t)wd.kf_off + i;
        for (int q = 0; q < 7; ++q) bd.pose0[7 * k + q] = td.kf_pose[7 * (size_t)slot + q];
        for (int q = 0; q < 4; ++q) bd.plane0[4 * k + q] = td.kf_plane[4 * (size_t)slot + q];
        bd.kf_fixed[k] = sel.kf_fixed[i];
    }
    if (i < sel.n_lm) {
        const int slot = sel.lm_slot[i];
        const size_t L = (size_t)wd.lm_off + i;
        td.sel_index[slot] = i;
        for (int q = 0; q < 3; ++q) r_lm_pos[3 * L + q] = td.lm_pos[3 * (size_t)slot + q];
        r_lm_weight[L] = td.lm_weight[slot];
        r_cnt[L] = 0;
        td.cursor[i] = 0;
    }
    if (i == 0) *td.n_depth = 0;
}

// Ground points attached on the device: addGroundPlaneResiduals (reference bundle_adjuster_keyframes.cpp:517-562) on the gathered
// window, for a window whose request lists candidate ground landmarks (TrackSel::gp_cand) instead of host-built lists.  One CTA per
// window, after k_track_begin (poses, planes, positions gathered) and before k_track_scan (the scale rule reads n_gp).  A candidate
// goes to the first keyframe, in window order, of strictly smallest distance |R(q) p + t| among those whose plane distance is not
// below -10, and is kept iff that distance is under 25 m, with weight 10 (1 - d / 25).  The kept ones are compacted in candidate
// order by an ordered block scan.  The arithmetic is the facade's host code operation for operation (mini_eigen.hpp: convert()
// of the 7-vector, Eigen's un-normalised toRotationMatrix, R * p + t, the square root of the squared norm; g++ -O2 without FMA):
// explicit round-to-nearest intrinsics, so that nothing is contracted and the lists equal the host's bit for bit.
__device__ __forceinline__ double gp_mul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double gp_add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double gp_sub(double a, double b) { return __dsub_rn(a, b); }

__global__ void __launch_bounds__(256) k_track_ground(BatchDev bd, const TrackSel* sels, const double* r_lm_pos, int* r_gp_lm) {
    const int w = blockIdx.x;
    const TrackSel& sel = sels[w];
    if (sel.n_cand == 0) return;  // idle, plane-free or host lists: untouched
    WinDesc& d = bd.desc[w];
    __shared__ double s_T[kMaxKf][12];  // R row-major, t (every keyframe a window may have; a track's ground window has at most 63)
    __shared__ int s_use[kMaxKf];
    __shared__ int s_warp[8];
    __shared__ int s_base;
    const int tid = threadIdx.x, lane = tid & 31, wp = tid >> 5, n_kf = sel.n_kf;
    if (tid < n_kf) {
        const double* q = bd.pose0 + 7 * ((size_t)d.kf_off + tid);
        const double qw = q[0], qx = q[1], qy = q[2], qz = q[3];
        const double tx = gp_mul(2.0, qx), ty = gp_mul(2.0, qy), tz = gp_mul(2.0, qz);
        const double twx = gp_mul(tx, qw), twy = gp_mul(ty, qw), twz = gp_mul(tz, qw);
        const double txx = gp_mul(tx, qx), txy = gp_mul(ty, qx), txz = gp_mul(tz, qx);
        const double tyy = gp_mul(ty, qy), tyz = gp_mul(tz, qy), tzz = gp_mul(tz, qz);
        const double Rq[9] = {gp_sub(1.0, gp_add(tyy, tzz)), gp_sub(txy, twz), gp_add(txz, twy),
                              gp_add(txy, twz), gp_sub(1.0, gp_add(txx, tzz)), gp_sub(tyz, twx),
                              gp_sub(txz, twy), gp_add(tyz, twx), gp_sub(1.0, gp_add(txx, tyy))};
        // convert(): Identity().translate(t).rotate(q); the products with the identity are kept (they decide the inf / NaN cases)
        double* T = s_T[tid];
        for (int i = 0; i < 3; ++i) {
            for (int j = 0; j < 3; ++j) {
                double s = 0.0;
                for (int k = 0; k < 3; ++k) s = gp_add(s, gp_mul(i == k ? 1.0 : 0.0, Rq[3 * k + j]));
                T[3 * i + j] = s;
            }
            const double Iv = gp_add(gp_add(gp_mul(i == 0 ? 1.0 : 0.0, q[4]), gp_mul(i == 1 ? 1.0 : 0.0, q[5])), gp_mul(i == 2 ? 1.0 : 0.0, q[6]));
            T[9 + i] = gp_add(0.0, Iv);
        }
        s_use[tid] = !(bd.plane0[4 * ((size_t)d.kf_off + tid) + 3] < -10.0);
    }
    if (tid == 0) s_base = 0;
    __syncthreads();
    const size_t go = (size_t)d.gp_off;
    for (int c0 = 0; c0 < sel.n_cand; c0 += 256) {
        const int c = c0 + tid;
        int j = 0, best = 0;
        double md = DBL_MAX;
        if (c < sel.n_cand) {
            j = sel.gp_cand[c];
            const double* p = r_lm_pos + 3 * ((size_t)d.lm_off + j);
            const double px = p[0], py = p[1], pz = p[2];
            for (int k = 0; k < n_kf; ++k) {
                if (!s_use[k]) continue;
                const double* T = s_T[k];
                const double x = gp_add(gp_add(gp_add(gp_mul(T[0], px), gp_mul(T[1], py)), gp_mul(T[2], pz)), T[9]);
                const double y = gp_add(gp_add(gp_add(gp_mul(T[3], px), gp_mul(T[4], py)), gp_mul(T[5], pz)), T[10]);
                const double z = gp_add(gp_add(gp_add(gp_mul(T[6], px), gp_mul(T[7], py)), gp_mul(T[8], pz)), T[11]);
                const double dist = __dsqrt_rn(gp_add(gp_add(gp_mul(x, x), gp_mul(y, y)), gp_mul(z, z)));
                if (dist < md) { md = dist; best = k; }  // first strict minimum; a NaN never is one
            }
        }
        const bool keep = md < 25.0;  // false past the list and when no keyframe qualified
        const unsigned m = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) s_warp[wp] = __popc(m);
        __syncthreads();
        int before = 0, total = 0;
        for (int q = 0; q < 8; ++q) { const int n = s_warp[q]; if (q < wp) before += n; total += n; }
        if (keep) {
            const size_t G = go + s_base + before + __popc(m & ((1u << lane) - 1));
            r_gp_lm[G] = j;
            bd.gp_kf[G] = best;
            bd.gp_weight[G] = gp_mul(10.0, gp_sub(1.0, __ddiv_rn(md, 25.0)));
        }
        __syncthreads();
        if (tid == 0) s_base += total;
        __syncthreads();
    }
    if (tid == 0) {
        d.n_gp = s_base;
        if (d.plane_reg_weight < 0) d.plane_reg_weight = s_base > 0 ? 10.0 : 0.0;  // cpp:717-719
    }
}

// pass 0: observations per selected landmark; pass 1: scatter behind the CSR pointers (order fixed afterwards by k_track_sort)
template <int kPass>
__global__ void __launch_bounds__(256) k_track_scatter(BatchDev bd, PackRaw raw, const TrackDev* tds, const TrackSel* sels, int* r_cnt,
                                                       int* r_kf, int* r_cam, float* r_u, float* r_v, float* r_d) {
    const int w = blockIdx.z, k = blockIdx.y;
    const TrackSel& sel = sels[w];
    if (k >= sel.n_kf) return;
    const TrackDev& td = tds[w];
    const WinDesc& wd = bd.desc[w];
    const int* lp = raw.lm_ptr + wd.lm_off + w;
    int* cnt = r_cnt + wd.lm_off;
    const size_t ob = (size_t)wd.obs_off;
    const int slot = sel.kf_slot[k];
    const int n = td.m_cnt[slot], m0 = td.m_off[slot];
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int j = td.sel_index[td.m_lm[m0 + i]];
        if (j < 0) continue;
        if (kPass == 0) {
            atomicAdd(&cnt[j], 1);
            if (td.m_d[m0 + i] > 0.0f) atomicAdd(td.n_depth, 1);
            continue;
        }
        const int pos = lp[j] + atomicAdd(&td.cursor[j], 1);
        r_kf[ob + pos] = k; r_cam[ob + pos] = td.m_cam[m0 + i];
        r_u[ob + pos] = td.m_u[m0 + i]; r_v[ob + pos] = td.m_v[m0 + i]; r_d[ob + pos] = td.m_d[m0 + i];
        td.key[pos] = ((long long)k << 32) | (long long)(m0 + i);
    }
}

// one CTA per window: CSR pointers of the gathered window, its observation count and, when asked, the scale-regulariser rule
__global__ void __launch_bounds__(1024) k_track_scan(BatchDev bd, const TrackDev* tds, const TrackSel* sels, const int* r_cnt, int* r_lm_ptr) {
    const int w = blockIdx.x;
    WinDesc& d = bd.desc[w];
    if (d.idle) return;
    __shared__ int s_scan[1024];
    const TrackSel& sel = sels[w];
    const int* cnt = r_cnt + d.lm_off;
    int* lp = r_lm_ptr + d.lm_off + w;
    const int tid = threadIdx.x, nth = blockDim.x, n = sel.n_lm;
    int carry = 0;
    for (int c0 = 0; c0 < n; c0 += nth) {
        const int j = c0 + tid;
        s_scan[tid] = j < n ? cnt[j] : 0;
        __syncthreads();
        for (int off = 1; off < nth; off <<= 1) {
            const int v = tid >= off ? s_scan[tid - off] : 0;
            __syncthreads();
            s_scan[tid] += v;
            __syncthreads();
        }
        if (j < n) lp[j + 1] = carry + s_scan[tid];
        const int tot = s_scan[nth - 1];
        __syncthreads();
        carry += tot;
    }
    if (tid == 0) {
        lp[0] = 0;
        d.n_obs = carry;
        if (sel.auto_scale) {  // addScaleRegularization's weight (bundle_adjuster_keyframes.cpp:703-716) and the plane-distance rule (:722-728)
            const int n_depth = *tds[w].n_depth, n_gp = d.n_gp;
            double wgt = 1000.0;
            if (n_depth > 10 || n_gp > 10) wgt = (n_gp < 30) ? 1000.0 / ((double)n_depth + (double)n_gp) : 0.0;
            d.scale_weight = wgt;
            d.plane_dist_fixed = n_depth < 10;
        }
    }
}

// a landmark's observations in (keyframe, arena) order = (keyframe, camera id) order of the caller: insertion sort, <= a few dozen
__global__ void __launch_bounds__(256) k_track_sort(BatchDev bd, const TrackDev* tds, const TrackSel* sels, const int* r_lm_ptr, int* r_kf,
                                                    int* r_cam, float* r_u, float* r_v, float* r_d) {
    const int w = blockIdx.y;
    const TrackSel& sel = sels[w];
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= sel.n_lm) return;
    const TrackDev& td = tds[w];
    const WinDesc& wd = bd.desc[w];
    const size_t ob = (size_t)wd.obs_off;
    r_kf += ob; r_cam += ob; r_u += ob; r_v += ob; r_d += ob;
    const int* lp = r_lm_ptr + wd.lm_off + w;
    const int o0 = lp[j], o1 = lp[j + 1];
    for (int a = o0 + 1; a < o1; ++a) {
        const long long key = td.key[a];
        const int kf = r_kf[a], cam = r_cam[a];
        const float u = r_u[a], v = r_v[a], d = r_d[a];
        int b = a - 1;
        while (b >= o0 && td.key[b] > key) {
            td.key[b + 1] = td.key[b]; r_kf[b + 1] = r_kf[b]; r_cam[b + 1] = r_cam[b];
            r_u[b + 1] = r_u[b]; r_v[b + 1] = r_v[b]; r_d[b + 1] = r_d[b];
            --b;
        }
        td.key[b + 1] = key; r_kf[b + 1] = kf; r_cam[b + 1] = cam; r_u[b + 1] = u; r_v[b + 1] = v; r_d[b + 1] = d;
    }
    td.sel_index[sel.lm_slot[j]] = -1;  // restore the all -1 state for the next solve
}

__global__ void __launch_bounds__(256) k_track_writeback(BatchDev bd, const TrackDev* tds, const TrackSel* sels) {
    const int w = blockIdx.y;
    const TrackSel& sel = sels[w];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= sel.n_kf && i >= sel.n_lm) return;
    const TrackDev& td = tds[w];
    const WinDesc& wd = bd.desc[w];
    const int cur = bd.state[w].cur;
    if (i < sel.n_kf) {
        const int slot = sel.kf_slot[i];
        const size_t k = (size_t)wd.kf_off + i;
        for (int q = 0; q < 7; ++q) td.kf_pose[7 * (size_t)slot + q] = bd.pose[cur][7 * k + q];
        for (int q = 0; q < 4; ++q) td.kf_plane[4 * (size_t)slot + q] = bd.plane[cur][4 * k + q];
    }
    if (i < sel.n_lm) {  // i: sorted position
        const size_t L = (size_t)wd.lm_off + i;
        const int slot = sel.lm_slot[bd.lm_orig[L]];
        for (int q = 0; q < 3; ++q) td.lm_pos[3 * (size_t)slot + q] = bd.lm[cur][3 * L + q];
    }
}

// dst[slot[i]][0..width) = src[i][0..width): host-staged rows into their store slots (poses, planes, landmark values)
// window blockIdx.y's rows
__global__ void __launch_bounds__(256) k_scatter_rows(const ScatterWin* wins, const int* slot, const double* val, int width) {
    const ScatterWin w = wins[blockIdx.y];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= w.n * width) return;
    const int r = i / width, c = i - r * width;
    w.dst[(size_t)slot[w.slot0 + r] * width + c] = val[(size_t)w.val0 * width + i];
}
void launch_scatter_rows(const ScatterWin* wins, int n_win, int max_rows, const int* slot, const double* val, int width, cudaStream_t s) {
    if (n_win > 0 && max_rows > 0) k_scatter_rows<<<dim3((max_rows * width + 255) / 256, n_win), 256, 0, s>>>(wins, slot, val, width);
    LCHK("k_scatter_rows");
}

void launch_track_gather(const BatchDev& bd, const PackRaw& raw, const TrackDev* tds, const TrackSel* sels, const TrackGrid& g,
                         cudaStream_t s) {
    // the PackRaw pointers are const views of buffers this batch owns: the gather is what fills them
    int* r_lm_ptr = const_cast<int*>(raw.lm_ptr);
    int* r_kf = const_cast<int*>(raw.obs_kf); int* r_cam = const_cast<int*>(raw.obs_cam);
    float* r_u = const_cast<float*>(raw.obs_u); float* r_v = const_cast<float*>(raw.obs_v); float* r_d = const_cast<float*>(raw.obs_d);
    double* r_pos = const_cast<double*>(raw.lm_pos); double* r_w = const_cast<double*>(raw.lm_weight);
    int* r_cnt = raw.lm_inv;  // scratch until the packing kernels overwrite it
    const int B = bd.n_win;
    const int n = g.max_kf > g.max_lm ? g.max_kf : g.max_lm;
    k_track_begin<<<dim3((n + 255) / 256 > 0 ? (n + 255) / 256 : 1, B), 256, 0, s>>>(bd, tds, sels, r_pos, r_w, r_cnt); LCHK("k_track_begin");
    if (g.any_cand) { k_track_ground<<<B, 256, 0, s>>>(bd, sels, r_pos, const_cast<int*>(raw.gp_lm)); LCHK("k_track_ground"); }
    const dim3 gm((g.max_meas + 255) / 256 > 0 ? (g.max_meas + 255) / 256 : 1, g.max_kf > 0 ? g.max_kf : 1, B);
    k_track_scatter<0><<<gm, 256, 0, s>>>(bd, raw, tds, sels, r_cnt, r_kf, r_cam, r_u, r_v, r_d); LCHK("k_track_scatter");
    k_track_scan<<<B, 1024, 0, s>>>(bd, tds, sels, r_cnt, r_lm_ptr); LCHK("k_track_scan");
    k_track_scatter<1><<<gm, 256, 0, s>>>(bd, raw, tds, sels, r_cnt, r_kf, r_cam, r_u, r_v, r_d); LCHK("k_track_scatter");
    k_track_sort<<<dim3((g.max_lm + 255) / 256 > 0 ? (g.max_lm + 255) / 256 : 1, B), 256, 0, s>>>(bd, tds, sels, r_lm_ptr, r_kf, r_cam, r_u,
                                                                                                r_v, r_d);
    LCHK("k_track_sort");
}

void launch_track_writeback(const BatchDev& bd, const TrackDev* tds, const TrackSel* sels, const TrackGrid& g, cudaStream_t s) {
    const int n = g.max_kf > g.max_lm ? g.max_kf : g.max_lm;
    k_track_writeback<<<dim3((n + 255) / 256 > 0 ? (n + 255) / 256 : 1, bd.n_win), 256, 0, s>>>(bd, tds, sels); LCHK("k_track_writeback");
}

cudaError_t configure_pack() {
    return cudaFuncSetAttribute(k_pack_sort, cudaFuncAttributeMaxDynamicSharedMemorySize, kPackMaxLandmarks * (int)sizeof(unsigned));
}


void launch_pack(const BatchDev& bd, const PackRaw& raw, cudaStream_t s) {
    const int B = bd.n_win;
    int np = 1;
    while (np < bd.max_lm) np <<= 1;
    k_pack_sort<<<B, 1024, (size_t)np * sizeof(unsigned), s>>>(bd, raw); LCHK("k_pack_sort");
    k_pack_obs<<<dim3((bd.max_lm + 7) / 8, B), 256, 0, s>>>(bd, raw); LCHK("k_pack_obs");
    k_pack_kf_count<<<B, 256, 0, s>>>(bd); LCHK("k_pack_kf_count");
    k_pack_kf_fill<<<dim3(bd.max_kf, B), 256, 0, s>>>(bd); LCHK("k_pack_kf_fill");
    if (bd.tot_gp > 0) k_pack_gp<<<dim3((bd.max_gp + 255) / 256, B), 256, 0, s>>>(bd, raw);
    LCHK("k_pack_gp");
    if (bd.fused) k_pack_ranges<8><<<dim3(((bd.max_lm + 7) / 8 + 255) / 256, B), 256, 0, s>>>(bd);
    else k_pack_ranges<32><<<dim3(((bd.max_lm + 31) / 32 + 255) / 256, B), 256, 0, s>>>(bd);
    LCHK("k_pack_ranges");
}

void launch_unpack_landmarks(const BatchDev& bd, double* lm_user, unsigned char* rejected_user, cudaStream_t s) {
    k_unpack_landmarks<<<dim3((bd.max_lm + 255) / 256, bd.n_win), 256, 0, s>>>(bd, lm_user, rejected_user); LCHK("k_unpack_landmarks");
}

}  // namespace kba
