// kba_compact.cuh -- order-keeping block-wide compaction, shared by the solve block's lists (kba_kfsolve.cu) and the camera step's
// post-push landmark list (kba_camerastep.cu).
#pragma once

namespace kba {

// the positions of the elements of [0, n) for which keep(c) holds, in order: emit(c, position); returns how many.  Every thread of
// the block calls it (blockDim.x a multiple of 32, at most 1024).  keep(c) of a chunk runs before any emit of that chunk, and every
// emit of a chunk before the next chunk's keep: a compaction in place reads its element in keep and writes it in emit.
template <class Keep, class Emit>
__device__ int block_compact(int n, Keep keep, Emit emit) {
    __shared__ int warp_sum[32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
    int base = 0;
    for (int c0 = 0; c0 < n; c0 += blockDim.x) {
        const int c = c0 + threadIdx.x;
        const bool f = c < n && keep(c);
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
        if (f) emit(c, base + (wid ? warp_sum[wid - 1] : 0) + __popc(m & ((1u << lane) - 1u)));
        base += warp_sum[n_warps - 1];
        __syncthreads();
    }
    return base;
}

}  // namespace kba
