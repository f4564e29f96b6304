// kba_store.cu -- store writes of the device-resident window (include/kba_b200.h, kba_track_group_push_keyframes): the arena
// compaction and the append of pushed keyframes, for every track of a call in one launch each; and the copies of a snapshot
// (kba_track_save / kba_track_load / kba_track_clone), which move the live keyframes' runs with the same two kernels and
// everything else as spans of words (k_copy_spans).
//
// The host decides every offset from its mirror of the arena layout (kba_api.cu, push_run): a compaction copies each live
// keyframe's run, in slot order, from the current arena into the other one; an append copies a keyframe's staged rows into the
// arena at the end of what is in use.  The arena's five columns (landmark slot, camera, u, v, d) are 4-byte words copied as such,
// so floats move bit for bit.  The host places each staged segment so that its offset is congruent to its arena offset modulo 4
// entries, and the copies run on 16-byte vectors wherever source and destination are aligned alike.
#include <algorithm>
#include <cstdint>

#include "kba_kernels.h"

namespace kba {

namespace {

constexpr int kSlice = 4096;  // entries of one run copied by one block (blockIdx.z): a multiple of 4, alignment is kept

// n words from src to dst by the block; 16-byte vectors when both are aligned alike
__device__ __forceinline__ void copy_words(unsigned* dst, const unsigned* src, int n) {
    const int head = (int)((4 - (((uintptr_t)dst >> 2) & 3)) & 3);
    if (((((uintptr_t)dst ^ (uintptr_t)src) & 15) == 0) && n > head) {
        for (int i = threadIdx.x; i < head; i += blockDim.x) dst[i] = src[i];
        const int nv = (n - head) >> 2;
        const uint4* s4 = reinterpret_cast<const uint4*>(src + head);
        uint4* d4 = reinterpret_cast<uint4*>(dst + head);
        for (int i = threadIdx.x; i < nv; i += blockDim.x) d4[i] = s4[i];
        for (int i = head + 4 * nv + threadIdx.x; i < n; i += blockDim.x) dst[i] = src[i];
    } else {
        for (int i = threadIdx.x; i < n; i += blockDim.x) dst[i] = src[i];
    }
}

}  // namespace

// run blockIdx.x, column blockIdx.y, slice blockIdx.z of it
__global__ void __launch_bounds__(256) k_arena_compact(const CompactTrack* ct, const CompactRun* runs) {
    const CompactRun r = runs[blockIdx.x];
    const CompactTrack& t = ct[r.track];
    const int q = blockIdx.y, i0 = blockIdx.z * kSlice;
    if (t.m_off && q == 0 && i0 == 0 && threadIdx.x == 0) { t.m_off[r.slot] = r.dst; t.m_cnt[r.slot] = r.n; }
    if (i0 >= r.n) return;
    copy_words(t.dst[q] + r.dst + i0, t.src[q] + r.src + i0, min(kSlice, r.n - i0));
}

// span blockIdx.x, its slices blockIdx.y, blockIdx.y + gridDim.y, ..
__global__ void __launch_bounds__(256) k_copy_spans(const CopySpan* spans) {
    const CopySpan sp = spans[blockIdx.x];
    for (long long i0 = (long long)blockIdx.y * kSlice; i0 < sp.n; i0 += (long long)gridDim.y * kSlice)
        copy_words(sp.dst + i0, sp.src + i0, (int)min((long long)kSlice, sp.n - i0));
}

// segment blockIdx.x, column blockIdx.y, slice blockIdx.z of it; block (x, 0, 0) also writes the keyframe's layout, pose and plane
__global__ void __launch_bounds__(256) k_store_append(const StoreAppend* app, const unsigned* cols, int stride) {
    const StoreAppend& a = app[blockIdx.x];
    const int q = blockIdx.y, i0 = blockIdx.z * kSlice;
    if (q == 0 && i0 == 0) {
        if (threadIdx.x < 7) a.kf_pose[7 * (size_t)a.slot + threadIdx.x] = a.pose_src ? a.pose_src[threadIdx.x] : a.pose[threadIdx.x];
        else if (threadIdx.x < 11) a.kf_plane[4 * (size_t)a.slot + threadIdx.x - 7] = a.plane[threadIdx.x - 7];
        else if (threadIdx.x == 32) { a.m_off[a.slot] = a.off; a.m_cnt[a.slot] = a.cnt; }
    }
    if (i0 >= a.n) return;
    const int n = min(kSlice, a.n - i0);
    unsigned* dst = a.col[q] + a.off + a.seg + i0;
    if (q == 1 && a.cam_zero) {
        for (int i = threadIdx.x; i < n; i += blockDim.x) dst[i] = 0u;
        return;
    }
    copy_words(dst, cols + (size_t)q * stride + a.src + i0, n);
}

void launch_store_push(const CompactTrack* ct, const CompactRun* runs, int n_runs, int max_run, const StoreAppend* app, int n_app,
                       int max_rows, const unsigned* cols, int stride, cudaStream_t s) {
    if (n_runs > 0) {
        k_arena_compact<<<dim3(n_runs, 5, (std::max(max_run, 1) + kSlice - 1) / kSlice), 256, 0, s>>>(ct, runs);
        LCHK("k_arena_compact");
    }
    if (n_app > 0) {
        k_store_append<<<dim3(n_app, 5, (std::max(max_rows, 1) + kSlice - 1) / kSlice), 256, 0, s>>>(app, cols, stride);
        LCHK("k_store_append");
    }
}

void launch_copy_spans(const CopySpan* spans, int n_spans, long long max_words, cudaStream_t s) {
    if (n_spans <= 0 || max_words <= 0) return;
    const long long slices = std::min<long long>((max_words + kSlice - 1) / kSlice, 65535);
    k_copy_spans<<<dim3(n_spans, (unsigned)slices), 256, 0, s>>>(spans);
    LCHK("k_copy_spans");
}

}  // namespace kba
