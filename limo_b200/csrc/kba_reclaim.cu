// kba_reclaim.cu -- free landmark slots of the device-resident store (include/kba_b200.h, kba_track_reclaim_landmarks): the slots
// of a range [lo, hi) that no arena entry of a live keyframe names, in ascending order, with their stored positions and weights
// on request.
//
// The slot map is the track's upkeep map ((stamp << 32) | payload, never cleared between calls, kba_upkeep.cu): every arena entry
// of a live keyframe gets the call's stamp, and a slot of the range is free iff its entry does not carry that stamp.  Liveness is
// the host's (kba_track_drop_keyframe leaves a dropped keyframe's entries in the arena until the next compaction), so the live
// keyframe slots come with the request.  Integer work only: the result does not depend on the launch order.
//
// Windows: one launch sequence serves W requests (a track group's; a single call is W = 1), window w = blockIdx.z, as in
// kba_upkeep.cu: grids from the maxima over the windows, blocks beyond their window's sizes exit.
#include <cstdint>

#include "kba_kernels.h"

namespace kba {

namespace {

__device__ __forceinline__ const ReclaimArgs& win(const ReclaimLaunch& l) { return blockIdx.z == 0 ? l.w0 : l.rest[blockIdx.z - 1]; }

__device__ __forceinline__ bool is_free(const ReclaimArgs& a, int s) {
    return s < a.hi && (unsigned)(a.map[s] >> 32) != a.stamp;
}

// the sum of v over the block's 256 threads, in every thread
__device__ __forceinline__ int block_sum(int v, int* red) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    int s = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += red[w];
    return s;
}

}  // namespace

// every arena entry of live keyframe blockIdx.y (and its strides) gets the call's stamp
__global__ void __launch_bounds__(256) k_rc_mark(const __grid_constant__ ReclaimLaunch l) {
    const ReclaimArgs& a = win(l);
    const unsigned long long mark = (unsigned long long)a.stamp << 32;
    for (int k = blockIdx.y; k < a.n_live; k += gridDim.y) {
        const int slot = a.kf_live[k];
        const int n = a.td.m_cnt[slot], m0 = a.td.m_off[slot];
        for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) a.map[a.td.m_lm[m0 + i]] = mark;
    }
}

// free slots of chunk blockIdx.x of the range
__global__ void __launch_bounds__(256) k_rc_count(const __grid_constant__ ReclaimLaunch l) {
    const ReclaimArgs& a = win(l);
    const int base = a.lo + blockIdx.x * kReclaimChunk;
    if (base >= a.hi) return;
    __shared__ int red[8];
    int c = 0;
    for (int r = 0; r < kReclaimChunk; r += blockDim.x) c += is_free(a, base + r + threadIdx.x);
    c = block_sum(c, red);
    if (threadIdx.x == 0) a.blk[blockIdx.x] = c;
}

// the free slots of chunk blockIdx.x at the sum of the earlier chunks' counts, in ascending order (a ballot / block scan per
// 256 slots), with the gather of positions and weights; the range's last chunk writes n_free
__global__ void __launch_bounds__(256) k_rc_write(const __grid_constant__ ReclaimLaunch l) {
    const ReclaimArgs& a = win(l);
    const int base = a.lo + blockIdx.x * kReclaimChunk;
    if (base >= a.hi) return;
    __shared__ int red[8], warp_off[8], chunk;
    int b = 0;
    for (int q = threadIdx.x; q < (int)blockIdx.x; q += blockDim.x) b += a.blk[q];
    int done = block_sum(b, red);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int r = 0; r < kReclaimChunk; r += blockDim.x) {
        const int s = base + r + threadIdx.x;
        const bool f = is_free(a, s);
        const unsigned hit = __ballot_sync(0xffffffffu, f);
        __syncthreads();
        if (lane == 0) warp_off[warp] = __popc(hit);
        __syncthreads();
        if (threadIdx.x == 0) {
            int t = 0;
            for (int w = 0; w < (int)(blockDim.x >> 5); ++w) { const int c = warp_off[w]; warp_off[w] = t; t += c; }
            chunk = t;
        }
        __syncthreads();
        if (f) {
            const int at = done + warp_off[warp] + __popc(hit & ((1u << lane) - 1u));
            a.free_slot[at] = s;
            if (a.pos) {
                const double* p = a.td.lm_pos + 3 * (size_t)s;
                a.pos[3 * (size_t)at] = p[0]; a.pos[3 * (size_t)at + 1] = p[1]; a.pos[3 * (size_t)at + 2] = p[2];
            }
            if (a.weight) a.weight[at] = a.td.lm_weight[s];
        }
        done += chunk;
    }
    if (threadIdx.x == 0 && base + kReclaimChunk >= a.hi) *a.n_free = done;
}

void launch_reclaim(const ReclaimLaunch& l, const ReclaimGrid& g, cudaStream_t s) {
    const unsigned W = (unsigned)l.n_win;
    const unsigned mb = (unsigned)(g.max_meas > 0 ? (g.max_meas + 255) / 256 : 1);
    const unsigned ky = (unsigned)(g.max_live > 0 ? (g.max_live < 65535 ? g.max_live : 65535) : 1);
    const unsigned cb = (unsigned)((g.max_range + kReclaimChunk - 1) / kReclaimChunk);
    k_rc_mark<<<dim3(mb, ky, W), 256, 0, s>>>(l); LCHK("k_rc_mark");
    k_rc_count<<<dim3(cb, 1, W), 256, 0, s>>>(l); LCHK("k_rc_count");
    k_rc_write<<<dim3(cb, 1, W), 256, 0, s>>>(l); LCHK("k_rc_write");
}

}  // namespace kba
