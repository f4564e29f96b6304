// kba_rank.cu -- the ranked landmark selection on the device-resident store (kba_track_rank_landmarks, include/kba_b200.h): the
// ranking LandmarkSelector::select does over the chain's quantities (facade/landmark_selection.cpp: chooseNearLmIds,
// chooseMiddleLmIds, chooseFarLmIds, the AddDepth scheme with limo's sorter), after launch_select computed them on the same lists.
//
// Exactness: the three partial sorts replay libstdc++'s heap (std::__make_heap, std::__adjust_heap, std::__push_heap as
// __partial_sort_copy and __heap_select call them), so that the tied elements a heap keeps are the host's.  The replay is cheap
// because the heap's top only gets better: an element that does not strictly beat the current top never enters later, so a warp
// screens 32 elements against the top at once and one lane replays the survivors in order.  The AddDepth costs come from
// depth_cost (kba_depth_cost.cuh), the function kba_track_depth_costs uses; the file is compiled with -fmad=false.  The middle
// bin's shuffle is libstdc++'s random_shuffle over the caller's draws.  Everything else is integer work in a fixed order.
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

__device__ __forceinline__ const RankArgs& win(const RankLaunch& l) {
    return l.all ? l.all[blockIdx.z] : (blockIdx.z == 0 ? l.w0 : l.rest[blockIdx.z - 1]);
}

// ---- libstdc++'s heap on element ids, `less` the partial sort's comparator (the heap's top is its greatest element) ----------
template <class Less>
__device__ void heap_adjust(int* h, int hole, int len, int value, const Less& less) {  // std::__adjust_heap
    const int top = hole;
    int second = hole;
    while (second < (len - 1) / 2) {
        second = 2 * (second + 1);
        if (less(h[second], h[second - 1])) --second;
        h[hole] = h[second];
        hole = second;
    }
    if ((len & 1) == 0 && second == (len - 2) / 2) {
        second = 2 * (second + 1);
        h[hole] = h[second - 1];
        hole = second - 1;
    }
    int parent = (hole - 1) / 2;  // std::__push_heap
    while (hole > top && less(h[parent], value)) {
        h[hole] = h[parent];
        hole = parent;
        parent = (hole - 1) / 2;
    }
    h[hole] = value;
}

template <class Less>
__device__ void heap_make(int* h, int len, const Less& less) {  // std::__make_heap
    if (len < 2) return;
    for (int parent = (len - 2) / 2;; --parent) {
        heap_adjust(h, parent, len, h[parent], less);
        if (parent == 0) return;
    }
}

// The elements item(0 .. n) (id >= 0, or -1: not part of the sequence) through a partial sort that keeps cap of them: the first
// cap fill the heap, make_heap, then each later element that beats the top replaces it (__adjust_heap at the root).  One warp;
// lane 0 owns the heap, the other lanes screen.  Returns the heap's size; the kept ids are heap[0 .. size).
template <class Item, class Less>
__device__ int heap_replay(int* heap, int cap, int n, const Item& item, const Less& less) {
    __shared__ int stage[32];
    const int lane = threadIdx.x & 31;
    int size = 0;  // the same in every lane
    if (cap <= 0) return 0;
    for (int i0 = 0; i0 < n; i0 += 32) {
        const int i = i0 + lane;
        const int id = i < n ? item(i) : -1;
        const bool keep = id >= 0 && (size < cap || less(id, heap[0]));
        const unsigned m = __ballot_sync(0xffffffffu, keep);
        if (m == 0) continue;
        stage[lane] = id;
        __syncwarp();
        if (lane == 0) {
            for (unsigned b = m; b; b &= b - 1) {
                const int v = stage[__ffs(b) - 1];
                if (size < cap) {
                    heap[size++] = v;
                    if (size == cap) heap_make(heap, cap, less);
                } else if (less(v, heap[0])) {
                    heap_adjust(heap, 0, cap, v, less);
                }
            }
        }
        size = __shfl_sync(0xffffffffu, size, 0);
        __syncwarp();
    }
    return size;
}

}  // namespace

// slot -> candidate again (k_sel_flow cleared it), marks cleared, the middle bin counted
__global__ void __launch_bounds__(256) k_rk_prep(const __grid_constant__ RankLaunch l) {
    const RankArgs& a = win(l);
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    const bool mid = c < a.n_cand && a.bin[c] == 1;
    if (c < a.n_cand) {
        a.cand_of[a.lm_slot[c]] = c;
        a.mark[c] = 0;
    }
    const unsigned m = __ballot_sync(0xffffffffu, mid);
    if ((threadIdx.x & 31) == 0 && m) atomicAdd(&l.n_mid[blockIdx.z], __popc(m));
}

// One block per listed keyframe that an AddDepth entry names: its eligible landmarks (cheirality survivors with elig set, the
// run-first entries in arena order, compacted by a block scan per chunk of 256 entries) with their costs, into the keyframe's own
// arena range of the scratch.
__global__ void __launch_bounds__(256) k_rk_depth(const __grid_constant__ RankLaunch l) {
    const RankArgs& a = win(l);
    const int k = blockIdx.x;
    if (k >= a.n_kf) return;
    __shared__ double T[12];
    __shared__ int warp_off[8], chunk, named;
    if (threadIdx.x == 0) named = 0;
    __syncthreads();
    for (int e = threadIdx.x; e < a.n_depth; e += blockDim.x)
        if (a.depth[2 * e] == k && a.depth[2 * e + 1] > 0) named = 1;
    __syncthreads();
    if (!named) return;
    const int slot = a.kf_slot[k];
    if (threadIdx.x == 0) iso_of_pose7(a.td.kf_pose + 7 * (size_t)slot, T);
    __syncthreads();
    const int n = a.td.m_cnt[slot], m0 = a.td.m_off[slot];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int done = 0;
    for (int i0 = 0; i0 < n; i0 += blockDim.x) {
        const int i = i0 + threadIdx.x;
        int c = -1;
        if (i < n && (i == 0 || a.td.m_lm[m0 + i] != a.td.m_lm[m0 + i - 1])) {
            c = a.cand_of[a.td.m_lm[m0 + i]];
            if (c >= 0 && !(a.cheiral[c] && a.elig[c])) c = -1;
        }
        const unsigned hit = __ballot_sync(0xffffffffu, c >= 0);
        if (lane == 0) warp_off[warp] = __popc(hit);
        __syncthreads();
        if (threadIdx.x == 0) {
            int s = 0;
            for (int w = 0; w < (int)(blockDim.x >> 5); ++w) { const int q = warp_off[w]; warp_off[w] = s; s += q; }
            chunk = s;
        }
        __syncthreads();
        if (c >= 0) {
            const int at = m0 + done + warp_off[warp] + __popc(hit & ((1u << lane) - 1u));
            a.dcand[at] = c;
            a.dcost[at] = depth_cost(T, a.td.lm_pos + 3 * (size_t)a.td.m_lm[m0 + i]);
        }
        done += chunk;
        __syncthreads();
    }
    if (threadIdx.x == 0) a.dcnt[k] = done;
}

// One warp per job: 0 the middle bin, 1 the near bin, 2 the far bin, 3 + e AddDepth entry e; job = first_job + blockIdx.x.  The
// heap (or the middle bin) lives in dynamic shared memory, sized per launch: the middle bins go in a launch of their own, so that
// a large middle bin does not size the shared memory of every heap.  The kept candidates get their job's bit in mark.
__global__ void __launch_bounds__(32) k_rk_heap(const __grid_constant__ RankLaunch l, int first_job) {
    extern __shared__ int heap[];
    const RankArgs& a = win(l);
    const int job = first_job + (int)blockIdx.x, lane = threadIdx.x;
    if (job == 1) {  // chooseNearLmIds: near order, those with a flow, partial_sort_copy by flow descending
        const double* flow = a.flow;
        const int* order = a.near_order;
        const int cap = min(a.max_near, a.n_cand);
        const int n = heap_replay(heap, cap, *a.n_near, [&](int i) { const int c = order[i]; return isnan(flow[c]) ? -1 : c; },
                                  [&](int x, int y) { return flow[x] > flow[y]; });
        for (int r = lane; r < n; r += 32) atomicOr(&a.mark[heap[r]], 1);
    } else if (job == 0) {  // chooseMiddleLmIds: candidate order, libstdc++'s random_shuffle, the first max_middle
        int n = 0;
        for (int c0 = 0; c0 < a.n_cand; c0 += 32) {
            const int c = c0 + lane;
            const bool mid = c < a.n_cand && a.bin[c] == 1;
            const unsigned m = __ballot_sync(0xffffffffu, mid);
            if (mid) heap[n + __popc(m & ((1u << lane) - 1u))] = c;
            n += __popc(m);
        }
        __syncwarp();
        if (lane == 0 && n > 1) {
            const int* d = l.p2 + 2 * l.n_win + l.p2[2 * blockIdx.z];
            for (int i = 1; i < n; ++i) {
                const int j = (int)((unsigned long long)(long long)d[i - 1] % (unsigned long long)(i + 1));  // size_t(draw) % (i + 1)
                if (i != j) { const int t = heap[i]; heap[i] = heap[j]; heap[j] = t; }
            }
        }
        __syncwarp();
        const int keep = min(a.max_middle, n);
        for (int r = lane; r < keep; r += 32) atomicOr(&a.mark[heap[r]], 2);
    } else if (job == 2) {  // chooseFarLmIds: candidate order, partial_sort_copy by seen descending
        const signed char* bin = a.bin;
        const int* seen = a.seen;
        const int cap = min(a.max_far, a.n_cand);
        const int n = heap_replay(heap, cap, a.n_cand, [&](int c) { return bin[c] == 2 ? c : -1; },
                                  [&](int x, int y) { return (unsigned)seen[x] > (unsigned)seen[y]; });
        for (int r = lane; r < n; r += 32) atomicOr(&a.mark[heap[r]], 4);
    } else {  // AddDepth entry: the keyframe's eligible landmarks, std::partial_sort by cost ascending, the first min(wanted, n)
        const int e = job - 3;
        if (e >= a.n_depth) return;
        const int ind = a.depth[2 * e], wanted = a.depth[2 * e + 1];
        if (ind >= a.n_kf || wanted <= 0) return;
        const int base = a.td.m_off[a.kf_slot[ind]], cnt = a.dcnt[ind];
        const double* cost = a.dcost + base;
        const int n = heap_replay(heap, min(wanted, cnt), cnt, [&](int i) { return i; }, [&](int x, int y) { return cost[x] < cost[y]; });
        for (int r = lane; r < n; r += 32) atomicOr(&a.mark[a.dcand[base + heap[r]]], 8);
    }
}

// The union in ascending candidate order (an ordered block scan per chunk of 1024 candidates, one CTA per window): the track's
// ranked slots and ground candidates, the caller's candidate indices and categories; then slot -> candidate back to all -1.
__global__ void __launch_bounds__(1024) k_rk_union(const __grid_constant__ RankLaunch l) {
    const RankArgs& a = win(l);
    __shared__ int s_sel[32], s_gnd[32], s_tot[2];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int o = l.p2[2 * blockIdx.z + 1];
    int* out_cand = l.out_cand + o;
    signed char* out_cat = l.out_cat + o;
    int n_sel = 0, n_gnd = 0;
    for (int c0 = 0; c0 < a.n_cand; c0 += 1024) {
        const int c = c0 + tid;
        const int mk = c < a.n_cand ? a.mark[c] : 0;
        const bool sel = mk != 0, gnd = sel && a.elig[c];
        const unsigned bs = __ballot_sync(0xffffffffu, sel), bg = __ballot_sync(0xffffffffu, gnd);
        if (lane == 0) { s_sel[warp] = __popc(bs); s_gnd[warp] = __popc(bg); }
        __syncthreads();
        if (tid == 0) {
            int x = 0, y = 0;
            for (int w = 0; w < 32; ++w) {
                const int p = s_sel[w], q = s_gnd[w];
                s_sel[w] = x; s_gnd[w] = y; x += p; y += q;
            }
            s_tot[0] = x; s_tot[1] = y;
        }
        __syncthreads();
        const unsigned lt = (1u << lane) - 1u;
        if (sel) {
            const int r = n_sel + s_sel[warp] + __popc(bs & lt);
            a.sel_slot[r] = a.lm_slot[c];
            out_cand[r] = c;
            out_cat[r] = (mk & 1) ? 0 : (mk & 2) ? 1 : (mk & 4) ? 2 : 3;
            if (gnd) a.gp[n_gnd + s_gnd[warp] + __popc(bg & lt)] = r;
        }
        if (c < a.n_cand) a.cand_of[a.lm_slot[c]] = -1;
        n_sel += s_tot[0]; n_gnd += s_tot[1];
        __syncthreads();
    }
    if (tid == 0) { l.res[2 * blockIdx.z] = n_sel; l.res[2 * blockIdx.z + 1] = n_gnd; }
}

void launch_rank_prepare(const RankLaunch& l, const RankGrid& g, cudaStream_t s) {
    const unsigned W = (unsigned)l.n_win;
    k_rk_prep<<<dim3((unsigned)(g.max_cand > 0 ? (g.max_cand + 255) / 256 : 1), 1, W), 256, 0, s>>>(l); LCHK("k_rk_prep");
    if (g.max_depth > 0) { k_rk_depth<<<dim3((unsigned)g.max_kf, 1, W), 256, 0, s>>>(l); LCHK("k_rk_depth"); }
}

void launch_rank(const RankLaunch& l, const RankGrid& g, cudaStream_t s) {
    const unsigned W = (unsigned)l.n_win;
    const size_t shm_mid = sizeof(int) * (size_t)g.mid_ints, shm = sizeof(int) * (size_t)g.heap_ints;
    const size_t shm_max = shm_mid > shm ? shm_mid : shm;
    if (shm_max > 48 * 1024) cudaFuncSetAttribute(k_rk_heap, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm_max);
    k_rk_heap<<<dim3(1, 1, W), 32, shm_mid, s>>>(l, 0); LCHK("k_rk_heap");
    k_rk_heap<<<dim3((unsigned)(2 + g.max_depth), 1, W), 32, shm, s>>>(l, 1); LCHK("k_rk_heap");
    k_rk_union<<<dim3(1, 1, W), 1024, 0, s>>>(l); LCHK("k_rk_union");
}

}  // namespace kba
