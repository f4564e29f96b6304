// kba_upkeep.cu -- window upkeep on the device-resident store (include/kba_b200.h): deactivateKeyframes
// (kba_track_deactivate_keyframes) and the AddDepth scheme's per-keyframe costs (kba_track_depth_costs), from the keyframe poses,
// the measurement arena and the landmark positions the store already holds.
//
// Slot contract: a keyframe's arena entries come in landmark-id order, one run per landmark, so a keyframe's distinct landmarks
// are the first entries of its runs.  The track's slot map holds (stamp << 32) | payload; an entry counts only when its stamp is
// the call's, so the map is never cleared between calls.
//
// Exactness: deactivation is integer arithmetic.  The cost is float(|kf * pos|) as limo's sorter computes it (depth_cost,
// kba_depth_cost.cuh, shared with the ranked selection); the file is compiled with -fmad=false.
//
// Windows: one launch sequence serves W requests (a track group's; a single call is W = 1), window w = blockIdx.z, as in
// kba_select.cu: grids from the maxima over the windows, blocks beyond their window's sizes exit.
#include <cfloat>
#include <cstdint>

#include "kba_depth_cost.cuh"
#include "kba_exact.cuh"
#include "kba_kernels.h"

namespace kba {

namespace {

using namespace exact;

__device__ __forceinline__ const UpkeepArgs& win(const UpkeepLaunch& l) { return blockIdx.z == 0 ? l.w0 : l.rest[blockIdx.z - 1]; }

__device__ __forceinline__ unsigned long long stamped(unsigned stamp, unsigned payload) {
    return ((unsigned long long)stamp << 32) | payload;
}

// the first entry of a landmark's run in keyframe `slot` (arena index e = m0 + i)
__device__ __forceinline__ bool run_first(const TrackDev& td, int m0, int i) { return i == 0 || td.m_lm[m0 + i] != td.m_lm[m0 + i - 1]; }

}  // namespace

// ---- deactivateKeyframes ------------------------------------------------------------------------------------------------------
// the newest keyframe's landmark slots get the call's stamp
__global__ void __launch_bounds__(256) k_up_mark_newest(const __grid_constant__ UpkeepLaunch l) {
    const UpkeepArgs& a = win(l);
    const int slot = a.kf_slot[a.n_kf - 1];
    const int n = a.td.m_cnt[slot], m0 = a.td.m_off[slot];
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
        a.map[a.td.m_lm[m0 + i]] = stamped(a.stamp, 0);
}

// one block per listed keyframe: its distinct landmarks the newest one names (getCommonLandmarkIds), then the window rule
__global__ void __launch_bounds__(256) k_up_common(const __grid_constant__ UpkeepLaunch l) {
    const UpkeepArgs& a = win(l);
    const int k = blockIdx.x;
    if (k >= a.n_kf) return;
    __shared__ int total;
    if (threadIdx.x == 0) total = 0;
    __syncthreads();
    const int slot = a.kf_slot[k];
    const int n = a.td.m_cnt[slot], m0 = a.td.m_off[slot];
    const unsigned long long mark = stamped(a.stamp, 0);
    int c = 0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) c += run_first(a.td, m0, i) && a.map[a.td.m_lm[m0 + i]] == mark;
    for (int o = 16; o > 0; o >>= 1) c += __shfl_down_sync(0xffffffffu, c, o);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(&total, c);
    __syncthreads();
    if (threadIdx.x == 0) {
        const int age = a.n_kf - 1 - k;  // n of the facade's loop: 0 for the newest keyframe
        a.kf_common[k] = total;
        a.kf_active[k] = age > a.max_window - 1 ? 0 : (age < a.min_window - 1 ? 1 : (total > a.min_connecting ? 1 : 0));
    }
}

// the landmark slots of the surviving keyframes get the call's second stamp
__global__ void __launch_bounds__(256) k_up_mark_active(const __grid_constant__ UpkeepLaunch l) {
    const UpkeepArgs& a = win(l);
    const int k = blockIdx.y;
    if (k >= a.n_kf || !a.kf_active[k]) return;
    const int slot = a.kf_slot[k];
    const int n = a.td.m_cnt[slot], m0 = a.td.m_off[slot];
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
        a.map[a.td.m_lm[m0 + i]] = stamped(a.stamp + 1, 0);
}

// the listed landmarks that a surviving keyframe measures
__global__ void __launch_bounds__(256) k_up_flag(const __grid_constant__ UpkeepLaunch l) {
    const UpkeepArgs& a = win(l);
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < (a.n_lm_d ? *a.n_lm_d : a.n_lm)) a.lm_active[j] = a.map[a.lm_slot[j]] == stamped(a.stamp + 1, 0);
}

// ---- AddDepth costs -----------------------------------------------------------------------------------------------------------
// slot -> eligible index
__global__ void __launch_bounds__(256) k_up_elig(const __grid_constant__ UpkeepLaunch l) {
    const UpkeepArgs& a = win(l);
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < a.n_lm) a.map[a.lm_slot[j]] = stamped(a.stamp, (unsigned)j);
}

// one block per listed keyframe: the eligible run-first entries in arena order (a block scan per chunk of 256 entries keeps the
// order), each with its cost.  The keyframe's pairs start at base_k, the sum of the earlier keyframes' bounds.
__global__ void __launch_bounds__(256) k_up_depth(const __grid_constant__ UpkeepLaunch l) {
    const UpkeepArgs& a = win(l);
    const int k = blockIdx.x;
    if (k >= a.n_kf) return;
    __shared__ double T[12];
    __shared__ int warp_off[8], base, chunk;
    const int slot = a.kf_slot[k];
    if (threadIdx.x == 0) {
        iso_of_pose7(a.td.kf_pose + 7 * (size_t)slot, T);
        int b = 0;
        for (int q = 0; q < k; ++q) b += min(a.n_lm, a.td.m_cnt[a.kf_slot[q]]);
        base = b;
    }
    __syncthreads();
    const int n = a.td.m_cnt[slot], m0 = a.td.m_off[slot];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int done = 0;
    for (int i0 = 0; i0 < n; i0 += blockDim.x) {
        const int i = i0 + threadIdx.x;
        int j = -1;
        if (i < n && run_first(a.td, m0, i)) {
            const unsigned long long v = a.map[a.td.m_lm[m0 + i]];
            if ((unsigned)(v >> 32) == a.stamp) j = (int)(unsigned)v;
        }
        const unsigned hit = __ballot_sync(0xffffffffu, j >= 0);
        if (lane == 0) warp_off[warp] = __popc(hit);
        __syncthreads();
        if (threadIdx.x == 0) {
            int s = 0;
            for (int w = 0; w < (int)(blockDim.x >> 5); ++w) { const int c = warp_off[w]; warp_off[w] = s; s += c; }
            chunk = s;
        }
        __syncthreads();
        if (j >= 0) {
            const int at = base + done + warp_off[warp] + __popc(hit & ((1u << lane) - 1u));
            a.cand[at] = j;
            a.cost[at] = depth_cost(T, a.td.lm_pos + 3 * (size_t)a.td.m_lm[m0 + i]);
        }
        done += chunk;
        __syncthreads();
    }
    if (threadIdx.x == 0) a.cnt[k] = done;
}

void launch_deactivate(const UpkeepLaunch& l, const UpkeepGrid& g, cudaStream_t s) {
    const unsigned W = (unsigned)l.n_win;
    auto blocks = [](int n) { return (unsigned)(n > 0 ? (n + 255) / 256 : 1); };
    k_up_mark_newest<<<dim3(blocks(g.max_meas), 1, W), 256, 0, s>>>(l); LCHK("k_up_mark_newest");
    k_up_common<<<dim3((unsigned)g.max_kf, 1, W), 256, 0, s>>>(l); LCHK("k_up_common");
    k_up_mark_active<<<dim3(blocks(g.max_meas), (unsigned)g.max_kf, W), 256, 0, s>>>(l); LCHK("k_up_mark_active");
    k_up_flag<<<dim3(blocks(g.max_lm), 1, W), 256, 0, s>>>(l); LCHK("k_up_flag");
}

void launch_depth_costs(const UpkeepLaunch& l, const UpkeepGrid& g, cudaStream_t s) {
    const unsigned W = (unsigned)l.n_win;
    auto blocks = [](int n) { return (unsigned)(n > 0 ? (n + 255) / 256 : 1); };
    k_up_elig<<<dim3(blocks(g.max_lm), 1, W), 256, 0, s>>>(l); LCHK("k_up_elig");
    k_up_depth<<<dim3((unsigned)g.max_kf, 1, W), 256, 0, s>>>(l); LCHK("k_up_depth");
}

}  // namespace kba
