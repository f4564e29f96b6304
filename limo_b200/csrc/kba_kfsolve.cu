// kba_kfsolve.cu -- limo's solve block on the device-resident store (kba_track_keyframe_solve, include/kba_b200.h): updateLabels
// and the post-deactivation lists between the deactivation (kba_upkeep.cu) and the ranking's chain (kba_select.cu, kba_rank.cu),
// in the same launch sequence, so that nothing comes down between them.
//
// Windows: one CTA per window (a track group's request; a single call is W = 1).  Everything is integer work in a fixed order:
// each list keeps its input order (block-wide compaction), and "the last tracklet of a slot decides" is an atomicMax over
// tracklet indices, whose result does not depend on scheduling.
#include "kba_compact.cuh"
#include "kba_kernels.h"

namespace kba {

namespace {

// updateLabels (bundle_adjuster_keyframes.cpp:388-431 as the facade states it) over the deactivation's outputs, then the
// post-deactivation keyframes (the oldest one fixed) and the ranking's candidates (still active, not outliers) with their
// eligibility (the ground flag).  The counts go into the window's selection and ranking records, which the chain's kernels of
// this sequence read.
__global__ void __launch_bounds__(1024) k_kfs_labels(const KfsArgs* args) {
    const KfsArgs& a = args[blockIdx.x];
    const int t = threadIdx.x, B = blockDim.x;
    const int n_lm = a.n_lm_d ? *a.n_lm_d : a.n_lm;
    for (int j = t; j < n_lm; j += B) {
        a.lm_at[a.lm_slot[j]] = j;
        a.lm_out[j] = 0;
        a.ground[j] = a.ground_in ? (a.ground_in[j] != 0) : 0;
        a.last[j] = -1;
    }
    __syncthreads();
    for (int i = t; i < a.n_out; i += B) {  // the retained outliers that are still active
        const int j = a.lm_at[a.out_slot[i]];
        if (j >= 0 && a.lm_active[j]) a.lm_out[j] = 1;
    }
    for (int i = t; i < a.n_trk; i += B) {
        const int s = a.trk_slot[i], j = s >= 0 ? a.lm_at[s] : -1;
        if (j < 0) continue;
        if (a.trk_cls[i] & kKfsMarked) a.lm_out[j] = 1;  // active or not: the facade inserts the id
        if (a.lm_active[j]) atomicMax(&a.last[j], i);
    }
    __syncthreads();
    for (int j = t; j < n_lm; j += B)
        if (a.last[j] >= 0) a.ground[j] = (a.trk_cls[a.last[j]] & kKfsGround) ? 1 : 0;
    for (int i = t; i < a.n_trk; i += B) {
        const int s = a.trk_slot[i], j = s >= 0 ? a.lm_at[s] : -1;
        const unsigned char c = a.trk_cls[i];
        a.trk_out[i] = ((c & kKfsMarked) || (j >= 0 && a.lm_out[j])) ? 1 : 0;
        a.shrub[i] = (j >= 0 && a.lm_active[j] && (c & kKfsShrub)) ? 1 : 0;
    }
    __syncthreads();
    const int K = block_compact(a.n_kf, [&](int k) { return a.kf_active[k] != 0; },
                                [&](int k, int o) { a.kf_post[o] = a.kf_slot[k]; a.fixed[o] = o == 0 ? 1 : 0; });
    const int N = block_compact(n_lm, [&](int j) { return a.lm_active[j] && !a.lm_out[j]; },
                                [&](int j, int o) { a.cand[o] = a.lm_slot[j]; a.elig[o] = a.ground[j]; });
    for (int j = t; j < n_lm; j += B) a.lm_at[a.lm_slot[j]] = -1;
    if (t == 0) {
        a.counts[0] = K; a.counts[1] = N;
        // no keyframe kept (the host refuses the request): the chain runs on the newest listed keyframe and no candidate, so that
        // no kernel sees an empty keyframe list
        if (K == 0) a.kf_post[0] = a.kf_slot[a.n_kf - 1];
        a.sel->n_kf = K > 0 ? K : 1; a.sel->n_cand = K > 0 ? N : 0;
        a.rank->n_kf = a.sel->n_kf; a.rank->n_cand = a.sel->n_cand;
    }
}

// the shrubbery weights of the tracklets k_kfs_labels flagged, into the store: launched once every check has passed
__global__ void k_kfs_weights(const KfsArgs* args) {
    const KfsArgs& a = args[blockIdx.y];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < a.n_trk && a.shrub[i]) a.lm_weight[a.trk_slot[i]] = a.shrub_weight;
}

}  // namespace

void launch_kfs_labels(const KfsArgs* args, int n_win, cudaStream_t s) {
    k_kfs_labels<<<(unsigned)n_win, 1024, 0, s>>>(args); LCHK("k_kfs_labels");
}

void launch_kfs_weights(const KfsArgs* args, int n_win, int max_trk, cudaStream_t s) {
    if (max_trk <= 0) return;
    k_kfs_weights<<<dim3((unsigned)((max_trk + 255) / 256), (unsigned)n_win), 256, 0, s>>>(args); LCHK("k_kfs_weights");
}

}  // namespace kba
