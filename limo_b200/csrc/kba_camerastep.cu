// kba_camerastep.cu -- limo's camera callback on the device-resident store (kba_track_camera_step, include/kba_b200.h): the solve
// block's landmark list after the push, built on the device from the creation's outcome, between the frame step's creation kernels
// and the solve block's deactivation in one launch sequence, so that nothing comes down between them.
//
// Windows: one CTA per solving window.  The compaction keeps list order (block-wide ballot scan) and is integer work only.
#include "kba_compact.cuh"
#include "kba_kernels.h"

namespace kba {

namespace {

// bundle_adjuster_keyframes.cpp:289-330 on the candidates: a landmark active before the frame stays listed; one the frame measures
// is listed again iff the frame was pushed; a new one iff it was pushed and its creation succeeded.  In place: each element is
// read in keep, before the scan, and written in emit, after it, at a position no larger than its own.
__global__ void __launch_bounds__(1024) k_cs_lists(const CsArgs* args) {
    const CsArgs& a = args[blockIdx.x];
    int slot = 0;
    unsigned char ground = 0;
    const int n = block_compact(
        a.n_cand,
        [&](int c) {
            const int tag = a.tag[c];
            const bool keep = tag == kCsActive || (a.selected && (tag == kCsMeasured || (tag >= 0 && (a.created[tag] & 1))));
            slot = a.lm_slot[c];
            ground = a.ground[c];
            if (!keep) a.index[c] = -1;
            return keep;
        },
        [&](int c, int o) {
            a.lm_slot[o] = slot;
            a.ground[o] = ground;
            a.index[c] = o;
        });
    if (threadIdx.x == 0) *a.n_lm = n;
}

}  // namespace

void launch_cs_lists(const CsArgs* args, int n_win, cudaStream_t s) {
    k_cs_lists<<<(unsigned)n_win, 1024, 0, s>>>(args); LCHK("k_cs_lists");
}

}  // namespace kba
