// kba_keyframe.cu -- the flow scheme of keyframe selection on the device-resident store (include/kba_b200.h,
// kba_track_frame_flow): KeyframeRejectionSchemeFlow::isUsable (keyframe_rejection_scheme_flow.cpp:17-74) of a new frame against
// the newest active keyframe, whose measurements the store already holds.
//
// Matching: kf_last's arena entries come in runs, one per landmark slot (the slot contract of the select / create / upkeep
// calls).  k_kf_mark stores each run's first entry in the track's stamped slot map ((stamp << 32) | run start; an entry counts only
// under the call's stamp, so the map is never cleared between calls); each frame entry then scans that short run for its camera.
//
// Exactness: the host adds sqrt(dx * dx + dy * dy) over the matched pairs in measurements_ order, then divides by their count and
// squares.  The terms are computed in parallel with explicit round-to-nearest intrinsics (the file is compiled with -fmad=false),
// the matched ones compacted in order by a ballot / block scan, and one thread adds them in that order: any tree reduction would
// round differently from the host.
//
// Windows: one launch sequence serves W requests (a track group's; a single call is W = 1), window w = blockIdx.z, as in
// kba_upkeep.cu.
#include <cstdint>

#include "kba_exact.cuh"
#include "kba_kernels.h"

namespace kba {

namespace {

using namespace exact;

constexpr int kFlowThreads = 1024;

__device__ __forceinline__ const FlowArgs& win(const FlowLaunch& l) { return blockIdx.z == 0 ? l.w0 : l.rest[blockIdx.z - 1]; }

}  // namespace

// kf_last's runs: slot -> (stamp, index of the run's first entry among kf_last's entries)
__global__ void __launch_bounds__(256) k_kf_mark(const __grid_constant__ FlowLaunch l) {
    const FlowArgs& a = win(l);
    const int n = a.td.m_cnt[a.kf_last], m0 = a.td.m_off[a.kf_last];
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
        if (i == 0 || a.td.m_lm[m0 + i] != a.td.m_lm[m0 + i - 1])
            a.map[a.td.m_lm[m0 + i]] = ((unsigned long long)a.stamp << 32) | (unsigned)i;
}

// one block per window: chunks of kFlowThreads frame entries, each matched and its term computed by its thread, the matched terms
// compacted in request order into shared memory and added there by thread 0
__global__ void __launch_bounds__(kFlowThreads) k_kf_flow(const __grid_constant__ FlowLaunch l) {
    const FlowArgs& a = win(l);
    __shared__ double term[kFlowThreads];
    __shared__ int warp_off[kFlowThreads / 32], chunk;
    const int n = a.n_meas, n_last = a.td.m_cnt[a.kf_last], m0 = a.td.m_off[a.kf_last];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    double sum = 0.;  // thread 0's
    int matched = 0;
    for (int i0 = 0; i0 < n; i0 += blockDim.x) {
        const int i = i0 + threadIdx.x;
        int e = -1;
        double t = 0.;
        if (i < n) {
            const int slot = a.lm_slot[i], cam = a.cam[i];
            const unsigned long long v = a.map[slot];
            if ((unsigned)(v >> 32) == a.stamp)
                for (int q = (int)(unsigned)v; q < n_last && a.td.m_lm[m0 + q] == slot; ++q)
                    if (a.td.m_cam[m0 + q] == cam) { e = q; break; }
            if (e >= 0) {  // Vector2d(u, v) - last.toEigen2d(), squaredNorm(), std::sqrt
                const double dx = ds((double)a.u[i], (double)a.td.m_u[m0 + e]), dy = ds((double)a.v[i], (double)a.td.m_v[m0 + e]);
                t = __dsqrt_rn(da(dm(dx, dx), dm(dy, dy)));
            }
            a.match[i] = e;
        }
        const unsigned hit = __ballot_sync(0xffffffffu, e >= 0);
        if (lane == 0) warp_off[warp] = __popc(hit);
        __syncthreads();
        if (threadIdx.x == 0) {
            int s = 0;
            for (int w = 0; w < (int)(blockDim.x >> 5); ++w) { const int c = warp_off[w]; warp_off[w] = s; s += c; }
            chunk = s;
        }
        __syncthreads();
        if (e >= 0) term[warp_off[warp] + __popc(hit & ((1u << lane) - 1u))] = t;
        __syncthreads();
        if (threadIdx.x == 0) {
            const int c = chunk;
            for (int q = 0; q < c; ++q) sum = da(sum, term[q]);  // sum += std::sqrt(el), in order
            matched += c;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const double s = __ddiv_rn(sum, (double)matched);  // sum /= flow_squared.size(); 0 / 0 without a match
        const double mean = dm(s, s);
        a.res->flow_sum = sum;
        a.res->mean_flow_sq = mean;
        a.res->n_matched = matched;
        a.res->usable = mean > dm(a.min_median_flow, a.min_median_flow) ? 1 : 0;  // a NaN compares false
    }
}

void launch_frame_flow(const FlowLaunch& l, const FlowGrid& g, cudaStream_t s) {
    const unsigned W = (unsigned)l.n_win;
    const unsigned mark_blocks = (unsigned)(g.max_last > 0 ? (g.max_last + 255) / 256 : 1);
    k_kf_mark<<<dim3(mark_blocks, 1, W), 256, 0, s>>>(l); LCHK("k_kf_mark");
    k_kf_flow<<<dim3(1, 1, W), kFlowThreads, 0, s>>>(l); LCHK("k_kf_flow");
}

}  // namespace kba
