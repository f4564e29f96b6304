// kba_framestep.cu -- limo's frame step on the device-resident store (kba_track_frame_step, include/kba_b200.h): the gather that
// turns the frame's one staged copy into the pose-only kernel's input, ahead of k_adjust_pose and the flow kernels of the same
// launch sequence.
//
// Windows: one CTA per window (a track group's request; a single call is W = 1).  Integer work and word copies only: the gathered
// rows keep their request order (block-wide compaction), so the adjustment reads exactly the rows kba_track_adjust_pose is given.
// -Xptxas -v (sm_90a): k_fs_gather uses no local memory (no spills).
#include "kba_kernels.h"

namespace kba {

namespace {

constexpr int kGatherThreads = 1024;

// the block's exclusive prefix of f over the threads, in thread order; *total gets the block's count.  Every thread calls it.
__device__ int block_prefix(bool f, int* total) {
    __shared__ int warp_sum[32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
    const unsigned m = __ballot_sync(0xffffffffu, f);
    if (lane == 0) warp_sum[wid] = __popc(m);
    __syncthreads();
    if (wid == 0) {
        int v = lane < n_warps ? warp_sum[lane] : 0;
        for (int o = 1; o < 32; o <<= 1) {
            const int u = __shfl_up_sync(0xffffffffu, v, o);
            if (lane >= o) v += u;
        }
        warp_sum[lane] = v;  // inclusive sums over the warps
    }
    __syncthreads();
    const int r = (wid ? warp_sum[wid - 1] : 0) + __popc(m & ((1u << lane) - 1u));
    *total = warp_sum[n_warps - 1];
    __syncthreads();
    return r;
}

}  // namespace

// window blockIdx.x: kf_last's pose into the download; for an adjusted frame, the measurements of its selected runs (in order) into
// the pose-only kernel's columns and their frame-local run starts, closed by the gathered count
__global__ void __launch_bounds__(kGatherThreads) k_fs_gather(StepLaunch l) {
    const StepArgs a = l.win[blockIdx.x];
    if (threadIdx.x < 7) a.last_pose[threadIdx.x] = a.kf_pose[threadIdx.x];
    if (!a.adjust) return;
    const unsigned* lm = l.cols + a.src;
    int run0 = 0, out0 = 0, start0 = 0;    // runs begun, rows gathered, runs gathered before this chunk
    for (int c0 = 0; c0 < a.n_meas; c0 += blockDim.x) {
        const int k = c0 + threadIdx.x;
        const bool in = k < a.n_meas;
        const bool starts = in && (k == 0 || lm[k] != lm[k - 1]);
        int n_start, n_keep, n_kept_start;
        const int run = run0 + block_prefix(starts, &n_start) + (starts ? 1 : 0) - 1;  // the run of row k
        const bool keep = in && l.run_sel[a.flag0 + run] != 0;
        const int o = out0 + block_prefix(keep, &n_keep);
        const int r = start0 + block_prefix(keep && starts, &n_kept_start);
        if (keep) {
            for (int q = 0; q < 5; ++q) l.dst[q][a.meas_off + o] = l.cols[(size_t)q * l.stride + a.src + k];
            if (starts) l.run_start[a.rs_off + r] = o;
        }
        run0 += n_start; out0 += n_keep; start0 += n_kept_start;
    }
    if (threadIdx.x == 0) l.run_start[a.rs_off + start0] = out0;
}

void launch_frame_step_gather(const StepLaunch& l, cudaStream_t s) {
    if (l.n_win <= 0) return;
    k_fs_gather<<<l.n_win, kGatherThreads, 0, s>>>(l);
    LCHK("k_fs_gather");
}

}  // namespace kba
