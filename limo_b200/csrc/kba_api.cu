// kba_api.cu -- host side of the C ABI declared in include/kba_b200.h: handle / batch lifetime, packing of caller
// windows into the batch-flat device layout, the pass loop, result download.  No numerical work happens on the host.
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <memory>
#include <string>
#include <thread>
#include <vector>

#include <cuda_runtime.h>

#include "kba_b200.h"
#include "kba_kernels.h"

using namespace kba;

static thread_local std::string g_last_error;
static int fail(int code, const std::string& msg) {
    g_last_error = msg;
    return code;
}
#define CU(call)                                                                                              \
    do {                                                                                                      \
        cudaError_t e_ = (call);                                                                              \
        if (e_ != cudaSuccess)                                                                                \
            return fail(KBA_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(e_));                    \
    } while (0)

struct kba_handle {
    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    Counters counters;
    bool kernel_timing = false;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    std::vector<cudaEvent_t> ev_pool;  // event pairs around every residual/Jacobian launch (kernel timing)
    int ev_used = 0;
    int sm_count = 132;
    cudaEvent_t ev_block = nullptr;  // blocking-sync event: waiting host threads sleep instead of spinning on a core
    bool blocking_sync = false;      // KBA_BLOCKING_SYNC=1 at kba_create
    // grow-only device workspace of the single-shot entry points (kba_lidar_depth): no cudaMalloc / cudaFree per call
    void* ws = nullptr;
    size_t ws_cap = 0;
};

// Wait for the handle's stream.  With KBA_BLOCKING_SYNC=1 (read at kba_create) the host thread sleeps on a blocking-sync
// event instead of spinning on a core (cudaStreamSynchronize spins under the default scheduling policy): for several
// handles per process / one process per GPU that share the box's cores with the packing threads.
static cudaError_t wait_event(kba_handle*, cudaEvent_t ev) { return cudaEventSynchronize(ev); }
static cudaError_t wait_stream(kba_handle* h) {
    if (!h->blocking_sync) return cudaStreamSynchronize(h->stream);  // lowest latency: the default for a lone handle
    if (!h->ev_block) {
        const cudaError_t e = cudaEventCreateWithFlags(&h->ev_block, cudaEventBlockingSync | cudaEventDisableTiming);
        if (e != cudaSuccess) return e;
    }
    const cudaError_t e = cudaEventRecord(h->ev_block, h->stream);
    if (e != cudaSuccess) return e;
    return cudaEventSynchronize(h->ev_block);
}

// ---- a device + pinned-host buffer pair, filled on the host and uploaded with one async copy ----------------------------
template <typename T>
struct Staged {
    T* h = nullptr;
    T* d = nullptr;
    size_t n = 0;
    int alloc(size_t count, bool host_copy) {
        n = count;
        const size_t bytes = std::max<size_t>(count, 1) * sizeof(T);
        if (cudaMalloc(&d, bytes) != cudaSuccess) return 1;
        if (host_copy && cudaMallocHost(&h, bytes) != cudaSuccess) return 1;
        return 0;
    }
    void release() {
        if (d) cudaFree(d);
        if (h) cudaFreeHost(h);
        d = nullptr; h = nullptr;
    }
    cudaError_t upload(cudaStream_t s) { return cudaMemcpyAsync(d, h, std::max<size_t>(n, 1) * sizeof(T), cudaMemcpyHostToDevice, s); }
    cudaError_t download(cudaStream_t s) { return cudaMemcpyAsync(h, d, std::max<size_t>(n, 1) * sizeof(T), cudaMemcpyDeviceToHost, s); }
};

struct kba_batch {
    kba_handle* h = nullptr;
    BatchDev bd{};
    std::vector<WinDesc> desc_h;
    // staged inputs
    Staged<WinDesc> desc;
    Staged<double> pose0, plane0, cam, lm0, lm_weight;
    Staged<uint8_t> kf_fixed;
    Staged<int> lm_ptr, obs_kf, obs_cam, obs_lm, kf_ptr, pm_lm, pm_cam, chunk_lm0, chunk_lm1, chunk_k0, chunk_k1, lm_orig, obs_orig;
    Staged<int> grp_k0, grp_k1;
    // device-side packing (kba_pack.cu, lc.plan.device_pack): the caller's arrays are uploaded as they are, the sorted layout is
    // built by kernels
    Staged<int> r_lm_ptr, r_obs_kf, r_obs_cam, r_gp_lm;
    Staged<float> r_obs_u, r_obs_v, r_obs_d;
    Staged<double> r_lm_pos, r_lm_weight;
    Staged<double> lm_user;            // landmark results in the caller's order (device + pinned)
    Staged<uint8_t> rej_user;
    PackRaw raw;
    Staged<int> obs_rank;
    Staged<float> obs_u, obs_v, obs_d, pm_u, pm_v, pm_d;
    // outputs
    Staged<WinState> state;
    Staged<IterRecord> log;
    Staged<double> pose_out[2], lm_out[2], plane_out[2];
    Staged<int> gp_lm, gp_kf, gp_of_lm, gp_shared;
    Staged<double> gp_weight;
    Staged<uint8_t> lm_active;
    Staged<int> n_active;
    Staged<unsigned long long> jac_obs;
    std::vector<void*> scratch;  // device-only allocations
    LaunchCfg lc;
    size_t h2d_bytes = 0, d2h_bytes = 0;
    float last_solve_ms = 0.f;
    cudaEvent_t ev_a = nullptr, ev_b = nullptr, ev_poll = nullptr, ev_poll2 = nullptr;
    // The pass sequence as a CUDA graph (kba_batch_solve): mode 2 = ONE launch per solve, the passes are the body of a conditional
    // WHILE node whose condition the device sets (k_loop_cond); mode 1 = a graph of `check_every` passes launched until the
    // downloaded active-window count is zero.  Rebuilt when anything a kernel receives by value changes (`key`); the solver options
    // are read from device memory (BatchDev::wsp), so a solve with other options launches the same graph.
    struct SolveGraph {
        cudaGraph_t graph = nullptr;
        cudaGraphExec_t exec = nullptr;
        std::vector<unsigned char> key;
        Counters per_pass;
        int mode = 0, passes_per_launch = 0;
        bool unusable = false;  // capture / instantiation failed once on this batch: the stream path is used from then on
        void destroy() {
            if (exec) cudaGraphExecDestroy(exec);
            if (graph) cudaGraphDestroy(graph);
            exec = nullptr; graph = nullptr; key.clear();
        }
    } sg;
    Staged<int> loop_pass;  // passes the WHILE node has run (device counter + pinned copy)
    long long solves_done = 0;
    // the solver options of every window (BatchDev::wsp): staged here, or at the front of a track solver's list upload
    // (track_solver_create re-points bd.wsp), and uploaded only when they differ from wsp_dev, what the device holds
    Staged<SolveParams> wsp;
    std::vector<SolveParams> wsp_dev;

    template <typename T>
    int dev_alloc(T** p, size_t count) {
        void* q = nullptr;
        if (cudaMalloc(&q, std::max<size_t>(count, 1) * sizeof(T)) != cudaSuccess) return 1;
        scratch.push_back(q);
        *p = (T*)q;
        return 0;
    }
    void dev_free(void* q) {
        scratch.erase(std::remove(scratch.begin(), scratch.end(), q), scratch.end());
        cudaFree(q);
    }
    void release() {
        desc.release(); pose0.release(); plane0.release(); cam.release(); lm0.release(); lm_weight.release();
        kf_fixed.release(); lm_ptr.release(); obs_kf.release(); obs_cam.release(); obs_lm.release(); kf_ptr.release();
        pm_lm.release(); pm_cam.release(); chunk_lm0.release(); chunk_lm1.release(); chunk_k0.release(); chunk_k1.release();
        lm_orig.release(); obs_orig.release(); obs_rank.release(); obs_u.release(); obs_v.release();
        grp_k0.release(); grp_k1.release();
        r_lm_ptr.release(); r_obs_kf.release(); r_obs_cam.release(); r_gp_lm.release(); r_obs_u.release(); r_obs_v.release();
        r_obs_d.release(); r_lm_pos.release(); r_lm_weight.release(); lm_user.release(); rej_user.release();
        obs_d.release(); pm_u.release(); pm_v.release(); pm_d.release(); state.release(); log.release();
        pose_out[0].release(); pose_out[1].release(); lm_out[0].release(); lm_out[1].release(); lm_active.release();
        n_active.release(); jac_obs.release(); plane_out[0].release(); plane_out[1].release();
        gp_lm.release(); gp_kf.release(); gp_of_lm.release(); gp_weight.release(); gp_shared.release();
        for (void* p : scratch) cudaFree(p);
        scratch.clear();
        if (ev_a) cudaEventDestroy(ev_a);
        if (ev_b) cudaEventDestroy(ev_b);
        if (ev_poll) cudaEventDestroy(ev_poll);
        if (ev_poll2) cudaEventDestroy(ev_poll2);
        sg.destroy();
        loop_pass.release();
        wsp.release();
    }
};

// buffers of kba_track_adjust_pose / kba_track_group_adjust_pose (k_adjust_pose): allocated at the first call, for the capacities of
// the track(s), then reused: a call makes one upload, one launch, one download and one synchronisation
struct MotionBufs {
    Staged<unsigned char> up;    // frame descriptors, solver options, run starts and measurements of one call (pinned + device)
    Staged<unsigned char> out;   // FrameRes per frame, iteration records, rejections (device + pinned)
    double* run_pw = nullptr, *trim_val = nullptr;
    unsigned char* run_active = nullptr, *run_rej = nullptr;
    IterRecord* log = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    int frames_cap = 0, runs_cap = 0, meas_cap = 0;
    static size_t al(size_t b) { return (b + 15) & ~(size_t)15; }
    static size_t up_bytes(int frames, int runs, int meas) {
        return al(sizeof(FrameDesc) * (size_t)frames) + al(sizeof(SolveParams) * (size_t)frames) + al(4 * ((size_t)runs + frames)) +
               5 * al(4 * (size_t)meas);
    }
    static size_t out_bytes(int frames, int log_cap, int runs) {
        return al(sizeof(FrameRes) * (size_t)frames) + al(sizeof(IterRecord) * (size_t)frames * log_cap) + al((size_t)runs);
    }
    int alloc(int frames, int runs, int meas) {
        frames_cap = frames; runs_cap = runs; meas_cap = meas;
        int bad = up.alloc(up_bytes(frames, runs, meas), true) | out.alloc(out_bytes(frames, kIterLogCap, runs), true);
        bad |= cudaMalloc(&run_pw, sizeof(double) * 4 * (size_t)std::max(runs, 1)) != cudaSuccess;
        bad |= cudaMalloc(&trim_val, sizeof(double) * 2 * (size_t)std::max(runs, 1)) != cudaSuccess;
        bad |= cudaMalloc(&run_active, (size_t)std::max(runs, 1)) != cudaSuccess;
        bad |= cudaMalloc(&run_rej, (size_t)std::max(runs, 1)) != cudaSuccess;
        bad |= cudaMalloc(&log, sizeof(IterRecord) * kIterLogCap * (size_t)frames) != cudaSuccess;
        bad |= cudaEventCreate(&ev0) != cudaSuccess;
        bad |= cudaEventCreate(&ev1) != cudaSuccess;
        return bad;
    }
    ~MotionBufs() {
        up.release(); out.release();
        if (run_pw) cudaFree(run_pw);
        if (trim_val) cudaFree(trim_val);
        if (run_active) cudaFree(run_active);
        if (run_rej) cudaFree(run_rej);
        if (log) cudaFree(log);
        if (ev0) cudaEventDestroy(ev0);
        if (ev1) cudaEventDestroy(ev1);
    }
};

// bytes one call moved each way: what the transfer-bytes calls report for the last call
struct Transfer {
    int64_t h2d = 0, d2h = 0;
};
static const Transfer kNoTransfer{};       // a call in which nothing ran

// what solves and pose-only calls of stored windows run on: one per track (n = 1) and one per track group (one window per
// track), created by track_solver_create
struct TrackSolver {
    kba_batch* batch = nullptr;            // one capacity-shaped window per track; its raw arrays are filled by the gather kernels
    Staged<TrackDev> tdev;                 // [n] read at every solve: compaction re-points a track's arena
    Staged<TrackSel> tsel;
    Staged<int> lists;                     // the windows' solver options (BatchDev::wsp), then every selection list of a solve (keyframe
                                           // slots, landmark slots, fixation bytes): ONE copy, from the lists on when the options are
                                           // those the device holds
    std::unique_ptr<MotionBufs> motion;    // pose-only calls, allocated at the first one
    Transfer counts;                       // the last solve or pose-only call
    void release() {
        if (batch) kba_batch_destroy(batch);
        batch = nullptr;
        tdev.release(); tsel.release(); lists.release();
        motion.reset();
    }
};

// staging of a store call (select_run .. rank_run): one pinned upload, argument records of windows 1 .. W-1 | the windows' lists,
// and one download of the windows' outputs (for a selection: flow | seen | near order (all windows' candidates end to end) |
// counters [W] | cheirality | bins; for a creation: positions | flags)
struct StoreStage {
    Staged<unsigned char> up, out;
    Transfer counts;                       // the last run's
    int alloc(size_t up_bytes, size_t out_bytes) { return up.alloc(up_bytes, true) | out.alloc(out_bytes, true); }
    ~StoreStage() { up.release(); out.release(); }
};

// device allocations freed with their owner
struct DevAllocs {
    std::vector<void*> ptrs;
    template <typename T> int alloc(T** p, size_t n) {
        void* q = nullptr;
        if (cudaMalloc(&q, std::max<size_t>(n, 1) * sizeof(T)) != cudaSuccess) return 1;
        ptrs.push_back(q); *p = (T*)q; return 0;
    }
    ~DevAllocs() {
        for (void* p : ptrs) cudaFree(p);
    }
};

// scratch of a track's selections (kba_select.cu): allocated at its first selection or ranking, alone or in a group, for the
// track's capacities, then reused by every entry point (calls are serial on the handle's stream)
struct SelectBufs {
    SelectArgs a;                          // the scratch pointers; lists and outputs are set per call
    DevAllocs dev;
};

// scratch of a track's landmark creations (kba_create.cu), kept like SelectBufs: scratch and the track's cameras on the device at
// its first creation, alone or in a group
struct CreateBufs {
    CreateArgs a;                          // the scratch pointers; lists and outputs are set per call
    DevAllocs dev;
};

// scratch of a track's upkeep, flow and reclaim calls (kba_upkeep.cu, kba_keyframe.cu, kba_reclaim.cu), kept like CreateBufs: the
// stamped slot map at the first of them, alone or in a group
struct UpkeepBufs {
    unsigned long long* map = nullptr;     // [lm_cap] (stamp << 32) | payload by slot, all 0 (stamp 0: never a call's) at first
    int* blk = nullptr;                    // [ceil(lm_cap / kReclaimChunk)] free slots per chunk of a reclaimed range
    unsigned stamp = 0;                    // the last stamp a call used
    DevAllocs dev;
};

// buffers of a track's ranked selections (kba_rank.cu), kept like SelectBufs: the quantities, the scratch and the ranking at its first
// ranking, alone or in a group.  The ranking is what kba_track_solve_ranked reads.
struct RankBufs {
    unsigned char* qty = nullptr;          // the chain's quantities, as select_run lays out one window's: flow | seen | near order |
                                           // counters | cheirality | bins, for lm_cap candidates
    int* mark = nullptr;                   // [lm_cap]
    int* dcand = nullptr;                  // [m_cap]
    double* dcost = nullptr;               // [m_cap]
    int* dcnt = nullptr;                   // [kf_cap]
    int* sel_slot = nullptr;               // [lm_cap] the ranked slots
    int* gp = nullptr;                     // [lm_cap] the ranked ground candidates
    std::vector<int> kf;                   // the ranking's keyframe list
    int n_sel = 0, n_ground = 0;
    uint64_t gen = 0;                      // kba_track::gen when it was ranked
    bool valid = false;
    DevAllocs dev;
};

// a track's label scratch (k_kfs_labels), allocated at its first keyframe solve, alone or in a group
struct KfsBufs {
    int* lm_at = nullptr;                  // [lm_cap] -1 between calls
    int* last = nullptr;                   // [lm_cap]
    DevAllocs dev;
};

// the duplicate checks of a track's slot lists (check_slot_lists, flow_check, frame_check): the check that named a slot last
struct SlotStamps {
    std::vector<unsigned> kf, lm;          // [kf_cap], [lm_cap]
    unsigned cur = 0;
    void next() {  // a fresh stamp; when the stamps wrap, start over
        if (++cur == 0) { std::fill(kf.begin(), kf.end(), 0u); std::fill(lm.begin(), lm.end(), 0u); cur = 1; }
    }
};

// the store calls that stage their requests, one staging each; deactivation and depth costs share the upkeep one, a drop shares
// the push's
enum StoreCall { kSelectCall, kCreateCall, kUpkeepCall, kFlowCall, kReclaimCall, kRankCall, kPushCall, kLandmarkWriteCall, kPoseWriteCall,
                 kSnapshotCall, kKfSolveCall, kFrameStepCall, kStoreCalls };

struct EvalStage;

// what a track and a track group own alike.  A track's set is {the track}: its calls run the host code of a group's, with one
// window.
struct TrackSet {
    kba_handle* h = nullptr;
    std::vector<kba_track*> tracks;
    TrackSolver solver;                    // window i of its batch is tracks[i]'s (fused path)
    TrackSolver large;                     // some track has win_rows > kFusedMaxRows: the whole set on the large-window path, else no batch
    std::unique_ptr<StoreStage> stage[kStoreCalls];  // each at its call's first run, for every track's capacities
    const Transfer* last = &kNoTransfer;   // the transfer counts of the last call
    std::unique_ptr<EvalStage> eval;       // evaluations, at the first one
    ~TrackSet();
};

// staging of the evaluations of a track or group (kba_evaluate.cu): the output block (device + pinned), laid out per call so that
// one copy brings down exactly the call's outputs, the windows' regions in it, and the cost partials (device only).  Allocated at
// the first evaluation for the capacities of the set's tracks.
struct EvalStage {
    Staged<unsigned char> out;
    Staged<EvalWin> wins;
    double* part = nullptr;
    DevAllocs dev;
    Transfer counts;                       // the last evaluation's
    ~EvalStage() { out.release(); wins.release(); }
};
TrackSet::~TrackSet() { solver.release(); large.release(); }

// persistent, device-resident window (kba_track_*, at the end of this file)
struct kba_track {
    TrackSet set;                          // {this}
    kba_track_caps caps{};
    int n_cam = 0;
    std::unique_ptr<SelectBufs> select;    // selections and rankings, allocated at the first of them
    std::unique_ptr<CreateBufs> create;    // landmark creations, allocated at the first one
    std::unique_ptr<UpkeepBufs> upkeep;    // upkeep, flow and reclaim calls, allocated at the first of them
    std::unique_ptr<RankBufs> rank;        // rankings, allocated at the first one
    std::unique_ptr<KfsBufs> kfs;          // keyframe solves' label scratch, allocated at the first one
    SlotStamps stamps;
    uint64_t gen = 0;                      // counts the calls that changed the store: a ranking of an older generation is stale
    TrackDev td{};
    int* arena_i[2][2] = {{nullptr, nullptr}, {nullptr, nullptr}};      // [buffer][lm, cam]
    float* arena_f[2][3] = {{nullptr, nullptr, nullptr}, {nullptr, nullptr, nullptr}};  // [buffer][u, v, d]
    int arena_cur = 0, arena_used = 0;
    std::vector<int> m_off, m_cnt;         // host mirror of the arena layout
    std::vector<char> kf_live;
    DevAllocs dev;
    std::vector<double> cam_intr, cam_pose;  // host copy of the cameras: capacity windows of the track and of its groups
    int64_t h2d_push = 0;                  // rows the store writes sent: pushes and landmark values
    void point_arena() {
        td.m_lm = arena_i[arena_cur][0]; td.m_cam = arena_i[arena_cur][1];
        td.m_u = arena_f[arena_cur][0]; td.m_v = arena_f[arena_cur][1]; td.m_d = arena_f[arena_cur][2];
    }
};

// several tracks solved as one batch (kba_track_group_*, at the end of this file)
struct kba_track_group {
    TrackSet set;
};

static int validate_window(const kba_window* w, std::string& why) {
    if (!w) { why = "null window"; return KBA_ERR_BAD_ARG; }
    if (w->n_kf < 0 || w->n_lm < 0 || w->n_obs < 0 || w->n_gp < 0 || w->n_cam < 1) { why = "negative size"; return KBA_ERR_BAD_ARG; }
    if (!w->kf_pose || !w->kf_fixed || !w->cam_intr || !w->cam_pose) { why = "null keyframe/camera array"; return KBA_ERR_BAD_ARG; }
    if (w->n_lm > 0 && (!w->lm_pos || !w->lm_weight || !w->lm_obs_ptr)) { why = "null landmark array"; return KBA_ERR_BAD_ARG; }
    if (w->n_obs > 0 && (!w->obs_kf || !w->obs_u || !w->obs_v || !w->obs_d)) { why = "null observation array"; return KBA_ERR_BAD_ARG; }
    if (w->n_kf > kMaxKf) { why = "more than 128 keyframes per window"; return KBA_ERR_CAPACITY; }
    if (w->n_cam > kMaxCam) { why = "more than 8 cameras per window"; return KBA_ERR_CAPACITY; }
    if ((w->n_gp > 0 || w->plane_reg_weight > 0) && !w->kf_plane) { why = "ground-plane residuals need kf_plane"; return KBA_ERR_BAD_ARG; }
    if (w->n_gp > 0 && (!w->gp_lm || !w->gp_kf || !w->gp_weight)) { why = "null ground-plane array"; return KBA_ERR_BAD_ARG; }
    for (int g = 0; g < w->n_gp; ++g)
        if (w->gp_lm[g] < 0 || w->gp_lm[g] >= w->n_lm || w->gp_kf[g] < 0 || w->gp_kf[g] >= w->n_kf) { why = "ground-plane index out of range"; return KBA_ERR_BAD_ARG; }
    if (w->speed_weight > 0 && (w->speed_kf < 0 || w->speed_kf >= w->n_kf || !(w->speed_dt > 0))) { why = "speed prior: keyframe out of range or dt <= 0"; return KBA_ERR_BAD_ARG; }
    if (w->n_lm > 0) {
        if (w->lm_obs_ptr[0] != 0) { why = "lm_obs_ptr[0] != 0"; return KBA_ERR_BAD_ARG; }
        for (int j = 0; j < w->n_lm; ++j)
            if (w->lm_obs_ptr[j + 1] < w->lm_obs_ptr[j]) { why = "lm_obs_ptr is not non-decreasing"; return KBA_ERR_BAD_ARG; }
        if (w->lm_obs_ptr[w->n_lm] != w->n_obs) { why = "lm_obs_ptr[n_lm] != n_obs"; return KBA_ERR_BAD_ARG; }
    } else if (w->n_obs != 0) { why = "observations without landmarks"; return KBA_ERR_BAD_ARG; }
    if (w->n_gp > 0) {  // at most one ground-plane residual per landmark (one Landmark::is_ground_plane flag, cpp:519-560)
        std::vector<unsigned char> seen((size_t)w->n_lm, 0);
        for (int g = 0; g < w->n_gp; ++g) {
            if (seen[w->gp_lm[g]]) { why = "two ground-plane residuals on one landmark"; return KBA_ERR_BAD_ARG; }
            seen[w->gp_lm[g]] = 1;
        }
    }
    for (int o = 0; o < w->n_obs; ++o) {
        if (w->obs_kf[o] < 0 || w->obs_kf[o] >= w->n_kf) { why = "obs_kf out of range"; return KBA_ERR_BAD_ARG; }
        if (w->obs_cam && (w->obs_cam[o] < 0 || w->obs_cam[o] >= w->n_cam)) { why = "obs_cam out of range"; return KBA_ERR_BAD_ARG; }
    }
    if (w->scale_weight > 0 && (w->scale_kf0 < 0 || w->scale_kf0 >= w->n_kf || w->scale_kf1 < 0 || w->scale_kf1 >= w->n_kf)) {
        why = "scale regulariser keyframe out of range"; return KBA_ERR_BAD_ARG;
    }
    return KBA_OK;
}

static void fill_window(kba_batch* b, int wi, const kba_window* w) {
    const WinDesc& d = b->desc_h[wi];
    memcpy(b->pose0.h + 7 * (size_t)d.kf_off, w->kf_pose, sizeof(double) * 7 * w->n_kf);
    memcpy(b->kf_fixed.h + d.kf_off, w->kf_fixed, w->n_kf);
    for (int k = 0; k < w->n_kf; ++k) {
        double* pl = b->plane0.h + 4 * (size_t)(d.kf_off + k);
        if (w->kf_plane) memcpy(pl, w->kf_plane + 4 * k, 4 * sizeof(double));
        else { pl[0] = 0; pl[1] = 0; pl[2] = 1; pl[3] = 0; }
    }
    for (int c = 0; c < w->n_cam; ++c) {
        double* o = b->cam.h + kCamStride * (size_t)(d.cam_off + c);
        quat_to_rot<double>(w->cam_pose + 7 * c, o);
        o[9] = w->cam_pose[7 * c + 4]; o[10] = w->cam_pose[7 * c + 5]; o[11] = w->cam_pose[7 * c + 6];
        o[12] = w->cam_intr[3 * c]; o[13] = w->cam_intr[3 * c + 1]; o[14] = w->cam_intr[3 * c + 2]; o[15] = 0;
    }
    // Landmarks are stored sorted by (first keyframe, last keyframe): consecutive landmarks then touch the same rows of
    // the reduced system, which is what lets the Schur kernel skip most tiles.  lm_orig maps back to the caller's order.
    const int nl = w->n_lm;
    int* orig = b->lm_orig.h + d.lm_off;
    {
        std::vector<long long> key(nl);
        for (int j = 0; j < nl; ++j) {
            const int o0 = w->lm_obs_ptr[j], o1 = w->lm_obs_ptr[j + 1];
            const int k0 = o1 > o0 ? w->obs_kf[o0] : w->n_kf, k1 = o1 > o0 ? w->obs_kf[o1 - 1] : w->n_kf;
            key[j] = ((long long)k0 << 40) | ((long long)k1 << 20) | 0;
            orig[j] = j;
        }
        std::stable_sort(orig, orig + nl, [&](int a, int c) { return key[a] < key[c]; });
    }
    int* lp = b->lm_ptr.h + d.lm_off + wi;
    int* kp = b->kf_ptr.h + d.kf_off + wi;
    std::fill(kp, kp + w->n_kf + 1, 0);
    int pos = 0, max_rank = 0;
    lp[0] = 0;
    for (int jn = 0; jn < nl; ++jn) {
        const int jo = orig[jn];
        memcpy(b->lm0.h + 3 * (size_t)(d.lm_off + jn), w->lm_pos + 3 * (size_t)jo, 3 * sizeof(double));
        b->lm_weight.h[d.lm_off + jn] = w->lm_weight[jo];
        for (int o = w->lm_obs_ptr[jo]; o < w->lm_obs_ptr[jo + 1]; ++o, ++pos) {
            const size_t e = (size_t)d.obs_off + pos;
            b->obs_kf.h[e] = w->obs_kf[o];
            b->obs_cam.h[e] = w->obs_cam ? w->obs_cam[o] : 0;
            b->obs_lm.h[e] = jn;
            b->obs_u.h[e] = w->obs_u[o]; b->obs_v.h[e] = w->obs_v[o]; b->obs_d.h[e] = w->obs_d[o];
            b->obs_orig.h[e] = o;
            // rank among the observations of this landmark in the same keyframe (multi-camera rigs)
            const int rank = (o > w->lm_obs_ptr[jo] && w->obs_kf[o - 1] == w->obs_kf[o]) ? b->obs_rank.h[e - 1] + 1 : 0;
            b->obs_rank.h[e] = rank;
            max_rank = std::max(max_rank, rank);
            kp[w->obs_kf[o] + 1]++;
        }
        lp[jn + 1] = pos;
    }
    b->desc_h[wi].max_rank = max_rank;
    b->desc.h[wi].max_rank = max_rank;
    // keyframe-major copy (counting sort, stable -> deterministic reduction order)
    for (int k = 0; k < w->n_kf; ++k) kp[k + 1] += kp[k];
    std::vector<int> cur(kp, kp + w->n_kf);
    for (int jn = 0; jn < nl; ++jn)
        for (int o = lp[jn]; o < lp[jn + 1]; ++o) {
            const size_t src = (size_t)d.obs_off + o;
            const size_t e = (size_t)d.obs_off + cur[b->obs_kf.h[src]]++;
            b->pm_lm.h[e] = jn;
            b->pm_cam.h[e] = b->obs_cam.h[src];
            b->pm_u.h[e] = b->obs_u.h[src]; b->pm_v.h[e] = b->obs_v.h[src]; b->pm_d.h[e] = b->obs_d.h[src];
        }
    // ground-plane residuals follow their landmark into the sorted order
    std::vector<int> gp_kf_of_lm(nl, -1);
    {
        std::vector<int> inv(nl);
        for (int jn = 0; jn < nl; ++jn) { inv[orig[jn]] = jn; b->gp_of_lm.h[d.lm_off + jn] = -1; }
        for (int g = 0; g < w->n_gp; ++g) {
            const int jn = inv[w->gp_lm[g]];
            b->gp_lm.h[d.gp_off + g] = jn;
            b->gp_kf.h[d.gp_off + g] = w->gp_kf[g];
            b->gp_weight.h[d.gp_off + g] = w->gp_weight[g];
            b->gp_of_lm.h[d.lm_off + jn] = g;
            gp_kf_of_lm[jn] = w->gp_kf[g];
            int shared = 0;
            for (int o = lp[jn]; o < lp[jn + 1]; ++o) shared |= (b->obs_kf.h[(size_t)d.obs_off + o] == w->gp_kf[g]);
            b->gp_shared.h[d.gp_off + g] = shared;
        }
    }
    for (int c = 0; c < d.n_chunks; ++c) {
        const int j0 = c * 32, j1 = std::min(nl, (c + 1) * 32);
        b->chunk_lm0.h[d.chunk_off + c] = j0;
        b->chunk_lm1.h[d.chunk_off + c] = j1;
        int k0 = w->n_kf, k1 = -1;
        for (int o = lp[j0]; o < lp[j1]; ++o) {
            const int k = b->obs_kf.h[(size_t)d.obs_off + o];
            k0 = std::min(k0, k); k1 = std::max(k1, k);
        }
        for (int j = j0; j < j1; ++j)
            if (gp_kf_of_lm[j] >= 0) { k0 = std::min(k0, gp_kf_of_lm[j]); k1 = std::max(k1, gp_kf_of_lm[j]); }
        b->chunk_k0.h[d.chunk_off + c] = k0;
        b->chunk_k1.h[d.chunk_off + c] = k1;
    }
    for (int c = 0; c < d.n_groups; ++c) {  // 8-landmark groups of the fused Schur kernel
        const int j0 = c * 8, j1 = std::min(nl, (c + 1) * 8);
        int k0 = w->n_kf, k1 = -1;
        for (int o = lp[j0]; o < lp[j1]; ++o) {
            const int k = b->obs_kf.h[(size_t)d.obs_off + o];
            k0 = std::min(k0, k); k1 = std::max(k1, k);
        }
        for (int j = j0; j < j1; ++j)
            if (gp_kf_of_lm[j] >= 0) { k0 = std::min(k0, gp_kf_of_lm[j]); k1 = std::max(k1, gp_kf_of_lm[j]); }
        b->grp_k0.h[d.grp_off + c] = k0;
        b->grp_k1.h[d.grp_off + c] = k1;
    }
}

// device-pack mode: the caller's arrays are copied as they are into the pinned staging buffers (one memcpy per array)
static void fill_window_raw(kba_batch* b, int wi, const kba_window* w) {
    const WinDesc& d = b->desc_h[wi];
    memcpy(b->pose0.h + 7 * (size_t)d.kf_off, w->kf_pose, sizeof(double) * 7 * w->n_kf);
    memcpy(b->kf_fixed.h + d.kf_off, w->kf_fixed, w->n_kf);
    for (int k = 0; k < w->n_kf; ++k) {
        double* pl = b->plane0.h + 4 * (size_t)(d.kf_off + k);
        if (w->kf_plane) memcpy(pl, w->kf_plane + 4 * k, 4 * sizeof(double));
        else { pl[0] = 0; pl[1] = 0; pl[2] = 1; pl[3] = 0; }
    }
    for (int c = 0; c < w->n_cam; ++c) {
        double* o = b->cam.h + kCamStride * (size_t)(d.cam_off + c);
        quat_to_rot<double>(w->cam_pose + 7 * c, o);
        o[9] = w->cam_pose[7 * c + 4]; o[10] = w->cam_pose[7 * c + 5]; o[11] = w->cam_pose[7 * c + 6];
        o[12] = w->cam_intr[3 * c]; o[13] = w->cam_intr[3 * c + 1]; o[14] = w->cam_intr[3 * c + 2]; o[15] = 0;
    }
    const size_t nl = (size_t)w->n_lm, no = (size_t)w->n_obs;
    memcpy(b->r_lm_pos.h + 3 * (size_t)d.lm_off, w->lm_pos, 3 * nl * sizeof(double));
    memcpy(b->r_lm_weight.h + d.lm_off, w->lm_weight, nl * sizeof(double));
    int* lp = b->r_lm_ptr.h + d.lm_off + wi;
    if (nl) memcpy(lp, w->lm_obs_ptr, (nl + 1) * sizeof(int)); else lp[0] = 0;
    memcpy(b->r_obs_kf.h + d.obs_off, w->obs_kf, no * sizeof(int));
    if (w->obs_cam) memcpy(b->r_obs_cam.h + d.obs_off, w->obs_cam, no * sizeof(int));
    else memset(b->r_obs_cam.h + d.obs_off, 0, no * sizeof(int));
    memcpy(b->r_obs_u.h + d.obs_off, w->obs_u, no * sizeof(float));
    memcpy(b->r_obs_v.h + d.obs_off, w->obs_v, no * sizeof(float));
    memcpy(b->r_obs_d.h + d.obs_off, w->obs_d, no * sizeof(float));
    if (w->n_gp) {
        memcpy(b->r_gp_lm.h + d.gp_off, w->gp_lm, w->n_gp * sizeof(int));
        memcpy(b->gp_kf.h + d.gp_off, w->gp_kf, w->n_gp * sizeof(int));
        memcpy(b->gp_weight.h + d.gp_off, w->gp_weight, w->n_gp * sizeof(double));
    }
    int max_rank = 0;  // several cameras of a rig seeing the landmark in one keyframe (observations are sorted by keyframe)
    for (int j = 0; j < w->n_lm; ++j) {
        int rank = 0;
        for (int o = w->lm_obs_ptr[j] + 1; o < w->lm_obs_ptr[j + 1]; ++o) {
            rank = (w->obs_kf[o] == w->obs_kf[o - 1]) ? rank + 1 : 0;
            max_rank = std::max(max_rank, rank);
        }
    }
    b->desc_h[wi].max_rank = max_rank;
    b->desc.h[wi].max_rank = max_rank;
}

// reduced-system rows a window can have given its constant keyframes (k_solve_begin may leave out more)
static int window_rows(const kba_window& w) {
    int n_free = 0;
    for (int k = 0; k < w.n_kf; ++k) n_free += w.kf_fixed[k] ? 0 : 1;
    return reduced_rows(n_free, w.n_gp > 0 || w.plane_reg_weight > 0);
}

struct kba_shard_comm;
kba::Exchange kba_shard_exchange(kba_shard_comm* c);  // kba_shard.cu

// How the pass sequence of a solve is issued (KBA_GRAPH, read once):
//   2 (default)  one CUDA graph launch per solve: the passes are the body of a conditional WHILE node, k_loop_cond sets the
//                condition on the device -- no host polling, no pass enqueued after the last window finished, no launch gaps;
//   1            a graph of four passes + the active-window count, launched until the count read back is zero;
//   0            kernel by kernel on the stream (always used with kernel timing on -- event pairs around the linearisation
//                launches --, with KBA_LAUNCH_CHECK, or on the legacy default stream, which cannot be captured).
// A sharded solve (NCCL all-reduces between the kernels) takes mode 1 from the second solve of its batch on, see kba_batch_solve.
static int solve_graph_mode() {
    static const int m = [] {
        const char* e = getenv("KBA_GRAPH");
        const int v = e ? atoi(e) : 2;
        return (v < 0 || v > 2) ? 2 : v;
    }();
    return m;
}

// KBA_SHARD_GRAPH=0: sharded solves stay on the stream path
static bool shard_graph_enabled() {
    static const bool on = [] { const char* e = getenv("KBA_SHARD_GRAPH"); return e ? atoi(e) != 0 : true; }();
    return on;
}

template <typename T>
static void key_append(std::vector<unsigned char>& k, const T& v) {
    const unsigned char* p = reinterpret_cast<const unsigned char*>(&v);
    k.insert(k.end(), p, p + sizeof(T));
}

// (re)builds b->sg for the given kernel arguments; false = not possible here (b->sg.unusable is set, the caller takes the stream path)
static bool build_solve_graph(kba_batch* b, const LaunchCfg& lc, int mode, int max_passes, int check_every,
                              const std::vector<unsigned char>& key) {
    kba_batch::SolveGraph& g = b->sg;
    g.destroy();
    cudaStream_t s = b->h->stream;
    Counters per{};
    cudaError_t e = cudaSuccess;
    bool capturing = false;
    int rc_pass = 0;
    if (mode == 2) {
        cudaGraphConditionalHandle handle = 0;
        cudaGraphNode_t node = nullptr;
        cudaGraphNodeParams np = {};
        e = cudaGraphCreate(&g.graph, 0);
        if (e == cudaSuccess) e = cudaGraphConditionalHandleCreate(&handle, g.graph, 1, cudaGraphCondAssignDefault);
        if (e == cudaSuccess) {
            np.type = cudaGraphNodeTypeConditional;
            np.conditional.handle = handle;
            np.conditional.type = cudaGraphCondTypeWhile;
            np.conditional.size = 1;
            e = cudaGraphAddNode(&node, g.graph, nullptr, 0, &np);
        }
        if (e == cudaSuccess) e = cudaStreamBeginCaptureToGraph(s, np.conditional.phGraph_out[0], nullptr, nullptr, 0, cudaStreamCaptureModeThreadLocal);
        if (e == cudaSuccess) {
            capturing = true;
            rc_pass = launch_pass(b->bd, lc, &per, s);
            launch_loop_cond(b->bd, (unsigned long long)handle, b->loop_pass.d, max_passes, s);
            cudaGraph_t body = nullptr;
            e = cudaStreamEndCapture(s, &body);
            capturing = false;
        }
        g.passes_per_launch = 0;  // counted on the device
    } else {
        e = cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal);
        if (e == cudaSuccess) {
            capturing = true;
            for (int i = 0; i < check_every && !rc_pass; ++i) rc_pass = launch_pass(b->bd, lc, i == 0 ? &per : nullptr, s);
            launch_count_active(b->bd, s);
            b->n_active.download(s);
            e = cudaStreamEndCapture(s, &g.graph);
            capturing = false;
        }
        g.passes_per_launch = check_every;
    }
    if (capturing) { cudaGraph_t junk = nullptr; cudaStreamEndCapture(s, &junk); }
    if (e == cudaSuccess && rc_pass) e = cudaErrorUnknown;
    if (e == cudaSuccess) e = cudaGraphInstantiate(&g.exec, g.graph, 0);
    if (e != cudaSuccess) {
        if (getenv("KBA_GRAPH_VERBOSE")) fprintf(stderr, "kba: solve graph (mode %d) not available: %s -- stream launches\n", mode, cudaGetErrorString(e));
        g.destroy();
        g.unusable = true;
        cudaGetLastError();  // the stream path starts with a clean error state
        return false;
    }
    if (getenv("KBA_GRAPH_VERBOSE")) fprintf(stderr, "kba: solve graph built (mode %d, %lld launches per pass)\n", mode, per.launches_total);
    g.key = key;
    g.per_pass = per;
    g.mode = mode;
    return true;
}

static void add_pass_counters(Counters& c, const Counters& per, long long passes) {
    c.launches_total += per.launches_total * passes; c.launches_jacobian += per.launches_jacobian * passes;
    c.launches_prep += per.launches_prep * passes; c.launches_schur += per.launches_schur * passes;
    c.launches_solve += per.launches_solve * passes; c.launches_backsub += per.launches_backsub * passes;
    c.launches_cost += per.launches_cost * passes; c.launches_update += per.launches_update * passes;
    c.launches_trim += per.launches_trim * passes;
}

extern "C" {

int kba_version(void) { return KBA_VERSION_MAJOR * 100 + KBA_VERSION_MINOR; }
// helpers for the other translation units of the library (not part of the public header)
int kba_internal_stream(kba_handle* h, cudaStream_t* s, int* device) {
    if (!h) return fail(KBA_ERR_BAD_ARG, "null handle");
    *s = h->stream; *device = h->device;
    return KBA_OK;
}
int kba_internal_fail(int code, const char* msg) { return fail(code, msg ? msg : ""); }
// at least `bytes` of device memory owned by the handle, 256-byte aligned, valid until the next call that asks for more
int kba_internal_workspace(kba_handle* h, size_t bytes, void** out) {
    if (!h || !out) return fail(KBA_ERR_BAD_ARG, "null handle");
    if (bytes > h->ws_cap) {
        CU(cudaSetDevice(h->device));
        CU(cudaStreamSynchronize(h->stream));
        if (h->ws) cudaFree(h->ws);
        h->ws = nullptr; h->ws_cap = 0;
        const size_t cap = bytes + bytes / 4 + 4096;
        CU(cudaMalloc(&h->ws, cap));
        h->ws_cap = cap;
    }
    *out = h->ws;
    return KBA_OK;
}
const char* kba_last_error(void) { return g_last_error.c_str(); }

void kba_default_options(kba_options* o) {
    if (!o) return;
    memset(o, 0, sizeof *o);
    o->depth_thres = 0.16; o->reprojection_thres = 1.6;
    o->depth_quantile = 0.95; o->reprojection_quantile = 0.95; o->gp_quantile = 1.0; o->gp_huber = 0.1;
    o->num_trim_rounds = -1; o->trim_solver_iterations = 2; o->final_solver_iterations = 100;
    o->min_landmarks_for_trimming = 100; o->min_residual_groups = 30; o->num_rounds_option = 1;
    o->solver_time_sec = 20.0;
    o->function_tolerance = 1e-6; o->gradient_tolerance = 1e-10; o->parameter_tolerance = 1e-8;
    o->initial_trust_region_radius = 1e4; o->max_trust_region_radius = 1e16; o->min_trust_region_radius = 1e-32;
    o->min_relative_decrease = 1e-3; o->min_lm_diagonal = 1e-6; o->max_lm_diagonal = 1e32;
    o->max_consecutive_invalid_steps = 5; o->precision = 0;
}

int kba_create(kba_handle** out, int device) {
    if (!out) return fail(KBA_ERR_BAD_ARG, "null out pointer");
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0)
        return fail(KBA_ERR_CUDA, "no CUDA device available: the kba_b200 library has no CPU fallback");
    if (device < 0 || device >= n) return fail(KBA_ERR_BAD_ARG, "device index out of range");
    CU(cudaSetDevice(device));
    cudaDeviceProp prop;
    CU(cudaGetDeviceProperties(&prop, device));
    // the library holds sm_90a code only (TMA bulk copies, mbarrier transaction counts, setmaxnreg), which no other compute
    // capability can load
    if (prop.major != 9 || prop.minor != 0)
        return fail(KBA_ERR_CUDA, "kba_b200 kernels are built for sm_90a (H100) only, device " + std::to_string(device) +
                                      " is sm_" + std::to_string(prop.major) + std::to_string(prop.minor));
    kba_handle* h = new kba_handle();
    h->device = device;
    h->sm_count = prop.multiProcessorCount;
    { const char* e = std::getenv("KBA_BLOCKING_SYNC"); h->blocking_sync = e && std::atoi(e) != 0; }
    CU(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
    h->own_stream = true;
    CU(cudaEventCreate(&h->ev0));
    CU(cudaEventCreate(&h->ev1));
    *out = h;
    return KBA_OK;
}

void kba_destroy(kba_handle* h) {
    if (!h) return;
    if (h->own_stream && h->stream) cudaStreamDestroy(h->stream);
    if (h->ev0) cudaEventDestroy(h->ev0);
    if (h->ev1) cudaEventDestroy(h->ev1);
    if (h->ev_block) cudaEventDestroy(h->ev_block);
    if (h->ws) cudaFree(h->ws);
    for (auto& e : h->ev_pool) cudaEventDestroy(e);
    delete h;
}

int kba_set_stream(kba_handle* h, void* s) {
    if (!h) return fail(KBA_ERR_BAD_ARG, "null handle");
    if (h->own_stream && h->stream) cudaStreamDestroy(h->stream);
    h->stream = (cudaStream_t)s;
    h->own_stream = false;
    return KBA_OK;
}

int kba_get_counters(kba_handle* h, kba_counters* out, int reset) {
    if (!h || !out) return fail(KBA_ERR_BAD_ARG, "null argument");
    const Counters& c = h->counters;
    out->launches_total = c.launches_total; out->launches_jacobian = c.launches_jacobian; out->launches_prep = c.launches_prep;
    out->launches_schur = c.launches_schur; out->launches_solve = c.launches_solve; out->launches_backsub = c.launches_backsub;
    out->launches_cost = c.launches_cost; out->launches_update = c.launches_update; out->launches_trim = c.launches_trim;
    out->ms_jacobian = c.ms_jacobian; out->jacobian_obs = c.jacobian_obs;
    if (reset) h->counters = Counters();
    return KBA_OK;
}

int kba_enable_kernel_timing(kba_handle* h, int on) {
    if (!h) return fail(KBA_ERR_BAD_ARG, "null handle");
    h->kernel_timing = on != 0;
    return KBA_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
static int batch_upload(kba_batch* b, int32_t n_windows, const kba_window* w, const int* rows);

// the fields of the batch's plan that the kernels read: the one place they are written
static void apply_plan(kba_batch* b) {
    const Plan& p = b->lc.plan;
    b->bd.nr_cap_max = p.nr_cap_max; b->bd.fused = p.fused; b->bd.p_split = p.p_split;
    b->bd.solve_tiled = p.solve_tiled; b->bd.solve_split = p.solve_split; b->bd.solve_banded = p.solve_banded;
}

// rows_of[i] (optional): reduced-system rows window i is sized for, instead of reduced_rows on all its keyframes.  A track's
// capacity window uses it: it has room for all its keyframes without plane blocks, or for 18 of them with plane blocks (fused
// solver), or for win_rows rows (large-window solver).
static int batch_create(kba_handle* h, int32_t n_windows, const kba_window* w, const int* rows_of, Purpose purpose, kba_batch** out) {
    if (!h || !w || !out || n_windows <= 0) return fail(KBA_ERR_BAD_ARG, "bad argument to kba_batch_create");
    CU(cudaSetDevice(h->device));
    std::string why;
    for (int i = 0; i < n_windows; ++i) {
        const int rc = validate_window(&w[i], why);
        if (rc != KBA_OK) return fail(rc, "window " + std::to_string(i) + ": " + why);
        if (w[i].n_kf < 3 && !w[i].landmarks_fixed)  // solve() needs 3 keyframes (cpp:630); adjustPoseOnly() has one
            return fail(KBA_ERR_NOT_ENOUGH_KF, "window " + std::to_string(i) + ": fewer than 3 keyframes");
    }
    kba_batch* b = new kba_batch();
    b->h = h;
    BatchDev& bd = b->bd;
    bd.n_win = n_windows;
    b->desc_h.resize(n_windows);
    std::vector<WinShape> shapes(n_windows);
    long long kf = 0, cam = 0, lm = 0, obs = 0, chunks = 0, soff = 0, gp = 0, groups = 0;
    for (int i = 0; i < n_windows; ++i) {
        WinDesc& d = b->desc_h[i];
        memset(&d, 0, sizeof d);
        d.n_kf = w[i].n_kf; d.n_cam = w[i].n_cam; d.n_lm = w[i].n_lm; d.n_obs = w[i].n_obs; d.n_gp = w[i].n_gp;
        d.kf_off = (int)kf; d.cam_off = (int)cam; d.lm_off = (int)lm; d.obs_off = (int)obs; d.gp_off = (int)gp;
        d.chunk_off = (int)chunks; d.n_chunks = (w[i].n_lm + 31) / 32;
        d.grp_off = (int)groups; d.n_groups = (w[i].n_lm + 7) / 8;
        groups += d.n_groups;
        d.scale_kf0 = w[i].scale_kf0; d.scale_kf1 = w[i].scale_kf1;
        d.scale_weight = w[i].scale_weight; d.scale_value = w[i].scale_value;
        WinShape& ws = shapes[i];
        ws.rows = rows_of ? rows_of[i] : reduced_rows(w[i].n_kf, w[i].n_gp > 0 || w[i].plane_reg_weight > 0);
        ws.free_rows = window_rows(w[i]);
        ws.n_chunks = d.n_chunks; ws.n_groups = d.n_groups; ws.n_lm = w[i].n_lm;
        d.nr_cap = nr_cap_of(ws.rows);
        d.plane_reg_weight = w[i].plane_reg_weight; d.plane_dist_fixed = w[i].plane_dist_fixed;
        d.s_off = soff;
        soff += (long long)d.nr_cap * d.nr_cap;
        kf += w[i].n_kf; cam += w[i].n_cam; lm += w[i].n_lm; obs += w[i].n_obs; chunks += d.n_chunks; gp += w[i].n_gp;
        bd.max_obs = std::max(bd.max_obs, w[i].n_obs); bd.max_lm = std::max(bd.max_lm, w[i].n_lm);
        bd.max_kf = std::max(bd.max_kf, w[i].n_kf); bd.max_gp = std::max(bd.max_gp, w[i].n_gp);
    }
    b->lc.knobs = read_knobs();
    b->lc.plan = make_plan(shapes.data(), n_windows, h->sm_count, b->lc.knobs, purpose);
    apply_plan(b);
    const int nr_cap_max = b->lc.plan.nr_cap_max;
    if (obs > 2000000000LL) { b->release(); delete b; return fail(KBA_ERR_CAPACITY, "batch exceeds 2^31 observations"); }
    if (nr_cap_max > kMaxReducedRows) {
        b->release();
        delete b;
        return fail(KBA_ERR_CAPACITY, "reduced system larger than 1344 rows (128 keyframes with ground-plane blocks)");
    }
    bd.tot_kf = kf; bd.tot_cam = cam; bd.tot_lm = lm; bd.tot_obs = obs; bd.tot_chunks = (int)chunks; bd.tot_gp = gp;
    bd.tot_groups = (int)groups;
    b->lc.sm_count = h->sm_count;
    // cost partials: one per CTA of k_linearize (8 warp tiles each, kba_linearize.cuh: lin_tile_bound) or per 256-observation tile of k_eval_obs
    bd.cost_parts = std::max((bd.max_obs + 255) / 256, (bd.max_obs / 16 + bd.max_lm / 32 + 4 + 7) / 8);
    bd.bs_parts = (bd.max_lm + 15) / 16;
    const bool hp = !b->lc.plan.device_pack;  // pinned host mirrors of the sorted layout are only needed when the host builds it
    int bad = 0;
    bad |= b->desc.alloc(n_windows, true);
    bad |= b->pose0.alloc(7 * kf, true); bad |= b->plane0.alloc(4 * kf, true); bad |= b->kf_fixed.alloc(kf, true);
    bad |= b->cam.alloc(kCamStride * cam, true);
    bad |= b->lm0.alloc(3 * lm, hp); bad |= b->lm_weight.alloc(lm, hp); bad |= b->lm_ptr.alloc(lm + n_windows, hp);
    bad |= b->obs_kf.alloc(obs, hp); bad |= b->obs_cam.alloc(obs, hp); bad |= b->obs_lm.alloc(obs, hp);
    bad |= b->obs_u.alloc(obs, hp); bad |= b->obs_v.alloc(obs, hp); bad |= b->obs_d.alloc(obs, hp);
    bad |= b->kf_ptr.alloc(kf + n_windows, hp); bad |= b->pm_lm.alloc(obs, hp); bad |= b->pm_cam.alloc(obs, hp);
    bad |= b->pm_u.alloc(obs, hp); bad |= b->pm_v.alloc(obs, hp); bad |= b->pm_d.alloc(obs, hp);
    bad |= b->chunk_lm0.alloc(chunks, hp); bad |= b->chunk_lm1.alloc(chunks, hp);
    bad |= b->chunk_k0.alloc(chunks, hp); bad |= b->chunk_k1.alloc(chunks, hp);
    bad |= b->lm_orig.alloc(lm, hp); bad |= b->obs_rank.alloc(obs, hp);
    if (hp) bad |= b->obs_orig.alloc(obs, true);
    bad |= b->grp_k0.alloc(groups, hp); bad |= b->grp_k1.alloc(groups, hp);
    if (b->lc.plan.device_pack) {
        bad |= b->r_lm_ptr.alloc(lm + n_windows, true); bad |= b->r_obs_kf.alloc(obs, true); bad |= b->r_obs_cam.alloc(obs, true);
        bad |= b->r_obs_u.alloc(obs, true); bad |= b->r_obs_v.alloc(obs, true); bad |= b->r_obs_d.alloc(obs, true);
        bad |= b->r_lm_pos.alloc(3 * lm, true); bad |= b->r_lm_weight.alloc(lm, true); bad |= b->r_gp_lm.alloc(gp, true);
        bad |= b->lm_user.alloc(3 * lm, true); bad |= b->rej_user.alloc(lm, true);
        bad |= b->dev_alloc(&b->raw.lm_inv, lm);
    }
    bad |= b->dev_alloc(&bd.grp_t0, groups); bad |= b->dev_alloc(&bd.grp_t1, groups); bad |= b->dev_alloc(&bd.grp_rs, groups);
    bad |= b->dev_alloc(&bd.grp_tiles, groups);
    bad |= b->dev_alloc(&bd.lin_tile, (size_t)(obs / 16) + (size_t)(lm / 32) + 4 * (size_t)n_windows + 4);
#ifdef KBA_PROF
    bad |= b->dev_alloc(&bd.prof, 16);
    if (!bad) cudaMemset(bd.prof, 0, 16 * sizeof(unsigned long long));
#endif
    bad |= b->dev_alloc(&bd.rt[0], (size_t)kPoseStride * kf); bad |= b->dev_alloc(&bd.rt[1], (size_t)kPoseStride * kf);
    {   // dense V panels of the Schur kernels; sized in kba_batch_upload from the chunks' keyframe ranges
        bd.panel_cap = 0;
        bd.vpanel = nullptr;
        bad |= b->dev_alloc(&bd.chunk_poff, chunks); bad |= b->dev_alloc(&bd.chunk_rs, chunks);
    }
    bad |= b->dev_alloc(&bd.chunk_t0, chunks); bad |= b->dev_alloc(&bd.chunk_t1, chunks); bad |= b->dev_alloc(&bd.obs_row, obs);
    bad |= b->state.alloc(n_windows, true); bad |= b->log.alloc((size_t)n_windows * kIterLogCap, true); bad |= b->wsp.alloc(n_windows, true);
    for (int q = 0; q < 2; ++q) { bad |= b->pose_out[q].alloc(7 * kf, true); bad |= b->lm_out[q].alloc(3 * lm, hp); }
    bad |= b->lm_active.alloc(lm, hp); bad |= b->n_active.alloc(1, true); bad |= b->jac_obs.alloc(1, true);
    // device-only scratch
    bad |= b->plane_out[0].alloc(4 * kf, true); bad |= b->plane_out[1].alloc(4 * kf, true);
    bad |= b->gp_lm.alloc(gp, hp); bad |= b->gp_kf.alloc(gp, true); bad |= b->gp_weight.alloc(gp, true); bad |= b->gp_of_lm.alloc(lm, hp); bad |= b->gp_shared.alloc(gp, hp);
    bad |= b->dev_alloc(&bd.gp_lin, 14 * gp); bad |= b->dev_alloc(&bd.vgp, 30 * gp);
    bad |= b->dev_alloc(&bd.gp_kfb, gp ? 65 * (size_t)kf : 0);
    bad |= b->dev_alloc(&bd.gp_cost_x, n_windows); bad |= b->dev_alloc(&bd.gp_cost_c, n_windows);
    bad |= b->dev_alloc(&bd.off_pose, kf); bad |= b->dev_alloc(&bd.off_dir, kf); bad |= b->dev_alloc(&bd.off_dist, kf);
    bad |= b->dev_alloc(&bd.bkf, 27 * kf);
    bad |= b->dev_alloc(&bd.scale_f, (size_t)n_windows * nr_cap_max); bad |= b->dev_alloc(&bd.lambda_f, (size_t)n_windows * nr_cap_max);
    bad |= b->dev_alloc(&bd.grad_f, (size_t)n_windows * nr_cap_max); bad |= b->dev_alloc(&bd.delta_f, (size_t)n_windows * nr_cap_max);
    bad |= b->dev_alloc(&bd.lm_scale, 3 * lm); bad |= b->dev_alloc(&bd.lm_linv, 6 * lm); bad |= b->dev_alloc(&bd.lm_z, 3 * lm);
    bad |= b->dev_alloc(&bd.lm_g, 3 * lm); bad |= b->dev_alloc(&bd.lm_lambda, 3 * lm); bad |= b->dev_alloc(&bd.trim_val, 3 * lm);
    bad |= b->dev_alloc(&bd.trim_reject, lm);
    bad |= b->dev_alloc(&bd.res, 3 * obs); bad |= b->dev_alloc(&bd.jp, 18 * obs);
    if (!bd.fused) bad |= b->dev_alloc(&bd.jl, 9 * obs);  // fused path: J_l is re-formed from J_p by its consumers
    else { bad |= b->dev_alloc(&bd.vobs, 18 * obs); bad |= b->dev_alloc(&bd.lm_run, lm); }  // ... and V is kept per observation, unpadded
    bad |= b->dev_alloc(&bd.cost_part_x, (size_t)n_windows * bd.cost_parts); bad |= b->dev_alloc(&bd.cost_part_c, (size_t)n_windows * bd.cost_parts);
    bad |= b->dev_alloc(&bd.bs_part, (size_t)n_windows * bd.bs_parts * 4);
    bad |= b->dev_alloc(&bd.sred, (size_t)soff * bd.p_split); bad |= b->dev_alloc(&bd.amat, (size_t)soff);
    bad |= b->dev_alloc(&bd.chol_w, (size_t)n_windows * 32 * 32); bad |= b->dev_alloc(&bd.chol_invd, (size_t)n_windows * nr_cap_max);
    if (bad) {
        const std::string msg = std::string("device/pinned allocation failed: ") + cudaGetErrorString(cudaGetLastError());
        b->release(); delete b;
        return fail(KBA_ERR_CUDA, msg);
    }
    bd.desc = b->desc.d; bd.state = b->state.d; bd.log = b->log.d; bd.wsp = b->wsp.d;
    bd.pose0 = b->pose0.d; bd.plane0 = b->plane0.d; bd.pose[0] = b->pose_out[0].d; bd.pose[1] = b->pose_out[1].d;
    bd.kf_fixed = b->kf_fixed.d; bd.cam = b->cam.d;
    bd.lm0 = b->lm0.d; bd.lm[0] = b->lm_out[0].d; bd.lm[1] = b->lm_out[1].d; bd.lm_weight = b->lm_weight.d;
    bd.lm_active = b->lm_active.d; bd.lm_ptr = b->lm_ptr.d;
    bd.obs_kf = b->obs_kf.d; bd.obs_cam = b->obs_cam.d; bd.obs_lm = b->obs_lm.d;
    bd.obs_u = b->obs_u.d; bd.obs_v = b->obs_v.d; bd.obs_d = b->obs_d.d;
    bd.kf_ptr = b->kf_ptr.d; bd.pm_lm = b->pm_lm.d; bd.pm_cam = b->pm_cam.d; bd.pm_u = b->pm_u.d; bd.pm_v = b->pm_v.d; bd.pm_d = b->pm_d.d;
    bd.chunk_lm0 = b->chunk_lm0.d; bd.chunk_lm1 = b->chunk_lm1.d; bd.chunk_k0 = b->chunk_k0.d; bd.chunk_k1 = b->chunk_k1.d;
    bd.lm_orig = b->lm_orig.d;
    bd.obs_rank = b->obs_rank.d;
    bd.grp_k0 = b->grp_k0.d; bd.grp_k1 = b->grp_k1.d;
    bd.plane[0] = b->plane_out[0].d; bd.plane[1] = b->plane_out[1].d;
    bd.gp_lm = b->gp_lm.d; bd.gp_kf = b->gp_kf.d; bd.gp_weight = b->gp_weight.d; bd.gp_of_lm = b->gp_of_lm.d; bd.gp_shared = b->gp_shared.d;
    bd.n_active = b->n_active.d;
    bd.jac_obs = b->jac_obs.d;
    if (b->lc.plan.device_pack) {
        PackRaw& r = b->raw;
        r.lm_ptr = b->r_lm_ptr.d; r.obs_kf = b->r_obs_kf.d; r.obs_cam = b->r_obs_cam.d;
        r.obs_u = b->r_obs_u.d; r.obs_v = b->r_obs_v.d; r.obs_d = b->r_obs_d.d;
        r.lm_pos = b->r_lm_pos.d; r.lm_weight = b->r_lm_weight.d; r.gp_lm = b->r_gp_lm.d; r.obs_orig = nullptr;
    }
    {   // failures from here on must give the allocations back
        cudaError_t e = cudaMemset(bd.jac_obs, 0, sizeof(unsigned long long));
        if (e == cudaSuccess) e = cudaEventCreate(&b->ev_a);
        if (e == cudaSuccess) e = cudaEventCreate(&b->ev_b);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&b->ev_poll, (h->blocking_sync ? cudaEventBlockingSync : 0) | cudaEventDisableTiming);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&b->ev_poll2, (h->blocking_sync ? cudaEventBlockingSync : 0) | cudaEventDisableTiming);
        if (e == cudaSuccess && b->loop_pass.alloc(1, true)) e = cudaErrorMemoryAllocation;
        if (e == cudaSuccess) e = configure_kernels(nr_cap_max);
        if (e == cudaSuccess && purpose == Purpose::TrackLarge) e = configure_kernels(kTiledMaxRows);  // re-planned solves factor tiled
        if (e == cudaSuccess && b->lc.plan.device_pack) e = configure_pack();
        if (e != cudaSuccess) { b->release(); delete b; return fail(KBA_ERR_CUDA, cudaGetErrorString(e)); }
    }
    *out = b;
    const int rc = batch_upload(b, n_windows, w, rows_of);
    if (rc != KBA_OK) { b->release(); delete b; *out = nullptr; }
    return rc;
}

int kba_batch_create(kba_handle* h, int32_t n_windows, const kba_window* w, kba_batch** out) {
    return batch_create(h, n_windows, w, nullptr, Purpose::Batch, out);
}

int kba_batch_upload(kba_batch* b, int32_t n_windows, const kba_window* w) { return batch_upload(b, n_windows, w, nullptr); }

// rows: as for batch_create
static int batch_upload(kba_batch* b, int32_t n_windows, const kba_window* w, const int* rows_of) {
    if (!b || !w || n_windows != b->bd.n_win) return fail(KBA_ERR_BAD_ARG, "bad argument to kba_batch_upload");
    CU(cudaSetDevice(b->h->device));  // callers may drive several handles from several host threads
    for (int i = 0; i < n_windows; ++i) {
        const WinDesc& d = b->desc_h[i];
        std::string why;
        const int rc = validate_window(&w[i], why);  // indices of the new contents are checked like at create
        if (rc != KBA_OK) return fail(rc, "kba_batch_upload: window " + std::to_string(i) + ": " + why);
        if (w[i].n_kf != d.n_kf || w[i].n_lm != d.n_lm || w[i].n_obs != d.n_obs || w[i].n_cam != d.n_cam || w[i].n_gp != d.n_gp)
            return fail(KBA_ERR_BAD_ARG, "kba_batch_upload: window shapes (keyframes, cameras, landmarks, observations, ground-plane "
                                         "residuals) differ from kba_batch_create");
        // the reduced system was sized at create
        const int rows = rows_of ? rows_of[i] : reduced_rows(w[i].n_kf, w[i].n_gp > 0 || w[i].plane_reg_weight > 0);
        if (nr_cap_of(rows) > d.nr_cap)
            return fail(KBA_ERR_BAD_ARG, "kba_batch_upload: window " + std::to_string(i) + " needs plane blocks the batch was not created with");
    }
    // packing (landmark sort, observation permutation, keyframe-major copy) is independent per window: host threads
    auto pack = [&](int i) {
        b->desc_h[i].scale_weight = w[i].scale_weight; b->desc_h[i].scale_value = w[i].scale_value;
        b->desc_h[i].scale_kf0 = w[i].scale_kf0; b->desc_h[i].scale_kf1 = w[i].scale_kf1;
        b->desc_h[i].landmarks_fixed = w[i].landmarks_fixed;
        b->desc_h[i].plane_reg_weight = w[i].plane_reg_weight; b->desc_h[i].plane_dist_fixed = w[i].plane_dist_fixed;
        b->desc_h[i].speed_kf = w[i].speed_kf; b->desc_h[i].speed_weight = w[i].speed_weight; b->desc_h[i].speed_dt = w[i].speed_dt;
        memcpy(b->desc_h[i].speed_v_before, w[i].speed_v_before, sizeof(double) * 3);
        memcpy(b->desc_h[i].speed_T_origin_before, w[i].speed_T_origin_before, sizeof(double) * 7);
        b->desc.h[i] = b->desc_h[i];
        if (b->lc.plan.device_pack) fill_window_raw(b, i, &w[i]);
        else fill_window(b, i, &w[i]);
    };
    {
        const char* e = std::getenv("KBA_HOST_THREADS");
        int nt = e ? std::atoi(e) : (int)std::min(16u, std::max(1u, std::thread::hardware_concurrency()));
        nt = std::max(1, std::min(nt, n_windows));
        if (nt == 1) {
            for (int i = 0; i < n_windows; ++i) pack(i);
        } else {
            std::atomic<int> next{0};
            std::vector<std::thread> pool;
            for (int t = 0; t < nt; ++t)
                pool.emplace_back([&] { for (int i = next.fetch_add(1); i < n_windows; i = next.fetch_add(1)) pack(i); });
            for (auto& th : pool) th.join();
        }
    }
    for (int i = 0; i < n_windows; ++i) b->lc.max_rank = std::max(b->lc.max_rank, b->desc_h[i].max_rank);
    if (b->lc.plan.fused) {  // the Schur kernel instance follows the keyframes the new contents fix
        int rows = 0;
        for (int i = 0; i < n_windows; ++i) rows = std::max(rows, window_rows(w[i]));
        b->lc.plan.fused_slots = fused_slots(rows);
    }
    if (!b->bd.fused) {   // V panel capacity: per chunk 96 columns x (rows of its keyframe range + right-hand-side tile), see k_solve_begin
        long long need = 0;
        for (int i = 0; i < n_windows; ++i) {
            const WinDesc& d = b->desc_h[i];
            const int rows_per_kf = (w[i].n_gp > 0 || w[i].plane_reg_weight > 0) ? 10 : 6;
            long long tot = 0;
            for (int c = 0; c < d.n_chunks; ++c) {
                // device packing (a track's capacity window): the ranges are built on the device at every solve, so every chunk
                // is sized for all the window's keyframes
                const int nk = b->lc.plan.device_pack ? d.n_kf : b->chunk_k1.h[d.chunk_off + c] - b->chunk_k0.h[d.chunk_off + c] + 1;
                if (nk <= 0) continue;
                const int rows = 8 * ((rows_per_kf * nk + 14 + 7) / 8) + 8;
                tot += 96LL * (((rows - 4 + 15) / 16) * 16 + 4);
            }
            need = std::max(need, tot);
        }
        if (need > b->bd.panel_cap) {
            if (b->bd.vpanel) { CU(cudaStreamSynchronize(b->h->stream)); b->dev_free(b->bd.vpanel); b->bd.vpanel = nullptr; }
            b->bd.panel_cap = (need + 1) & ~1LL;
            if (b->dev_alloc(&b->bd.vpanel, (size_t)n_windows * b->bd.panel_cap)) return fail(KBA_ERR_CUDA, "out of device memory (V panels)");
        }
        for (int i = 0; i < n_windows; ++i) { b->desc_h[i].panel_off = (long long)i * b->bd.panel_cap; b->desc.h[i].panel_off = b->desc_h[i].panel_off; }
    }
    cudaStream_t s = b->h->stream;
    if (b->lc.plan.device_pack) {  // the caller's arrays as they are (~33 B per observation), then the packing kernels
        CU(b->desc.upload(s)); CU(b->pose0.upload(s)); CU(b->plane0.upload(s)); CU(b->kf_fixed.upload(s)); CU(b->cam.upload(s));
        CU(b->r_lm_pos.upload(s)); CU(b->r_lm_weight.upload(s)); CU(b->r_lm_ptr.upload(s));
        CU(b->r_obs_kf.upload(s)); CU(b->r_obs_cam.upload(s)); CU(b->r_obs_u.upload(s)); CU(b->r_obs_v.upload(s)); CU(b->r_obs_d.upload(s));
        CU(b->r_gp_lm.upload(s)); CU(b->gp_kf.upload(s)); CU(b->gp_weight.upload(s));
        launch_pack(b->bd, b->raw, s);
        CU(cudaGetLastError());
        const BatchDev& bd = b->bd;
        b->h2d_bytes = sizeof(WinDesc) * bd.n_win + (7 + 4) * 8 * bd.tot_kf + bd.tot_kf + kCamStride * 8 * bd.tot_cam +
                       (3 + 1) * 8 * bd.tot_lm + 4 * (bd.tot_lm + bd.n_win) + (2 * 4 + 3 * 4) * bd.tot_obs + (4 + 4 + 8) * bd.tot_gp;
        return KBA_OK;
    }
    CU(b->desc.upload(s)); CU(b->pose0.upload(s)); CU(b->plane0.upload(s)); CU(b->kf_fixed.upload(s)); CU(b->cam.upload(s));
    CU(b->lm0.upload(s)); CU(b->lm_weight.upload(s)); CU(b->lm_ptr.upload(s));
    CU(b->obs_kf.upload(s)); CU(b->obs_cam.upload(s)); CU(b->obs_lm.upload(s));
    CU(b->obs_u.upload(s)); CU(b->obs_v.upload(s)); CU(b->obs_d.upload(s));
    CU(b->kf_ptr.upload(s)); CU(b->pm_lm.upload(s)); CU(b->pm_cam.upload(s)); CU(b->pm_u.upload(s)); CU(b->pm_v.upload(s)); CU(b->pm_d.upload(s));
    CU(b->chunk_lm0.upload(s)); CU(b->chunk_lm1.upload(s)); CU(b->chunk_k0.upload(s)); CU(b->chunk_k1.upload(s));
    CU(b->grp_k0.upload(s)); CU(b->grp_k1.upload(s));
    CU(b->lm_orig.upload(s)); CU(b->obs_rank.upload(s));
    CU(b->gp_lm.upload(s)); CU(b->gp_kf.upload(s)); CU(b->gp_weight.upload(s)); CU(b->gp_of_lm.upload(s)); CU(b->gp_shared.upload(s));
    const BatchDev& bd = b->bd;
    b->h2d_bytes = sizeof(WinDesc) * bd.n_win + (7 + 4) * 8 * bd.tot_kf + bd.tot_kf + kCamStride * 8 * bd.tot_cam +
                   (3 + 1) * 8 * bd.tot_lm + 4 * (bd.tot_lm + bd.n_win) + (3 * 4 + 3 * 4) * bd.tot_obs +
                   4 * (bd.tot_kf + bd.n_win) + (2 * 4 + 3 * 4) * bd.tot_obs + 8 * bd.tot_chunks + 8 * bd.tot_groups;
    return KBA_OK;
}

static SolveParams make_params(const kba_options* o) {
    SolveParams sp;
    memset(&sp, 0, sizeof sp);
    sp.gp_huber = o->gp_huber; sp.gp_quantile = o->gp_quantile;
    sp.depth_thres = o->depth_thres; sp.reprojection_thres = o->reprojection_thres;
    sp.depth_quantile = o->depth_quantile; sp.reprojection_quantile = o->reprojection_quantile;
    sp.function_tolerance = o->function_tolerance; sp.gradient_tolerance = o->gradient_tolerance;
    sp.parameter_tolerance = o->parameter_tolerance; sp.initial_radius = o->initial_trust_region_radius;
    sp.max_radius = o->max_trust_region_radius; sp.min_radius = o->min_trust_region_radius;
    sp.min_relative_decrease = o->min_relative_decrease; sp.min_lm_diagonal = o->min_lm_diagonal;
    sp.max_lm_diagonal = o->max_lm_diagonal; sp.trim_solver_iterations = o->trim_solver_iterations;
    sp.final_solver_iterations = o->final_solver_iterations; sp.min_residual_groups = o->min_residual_groups;
    sp.max_consecutive_invalid_steps = o->max_consecutive_invalid_steps;
    sp.max_solver_time = o->solver_time_sec;
    sp.rounds_override = o->num_trim_rounds; sp.min_landmarks_for_trimming = o->min_landmarks_for_trimming;
    sp.num_rounds_option = o->num_rounds_option;
    return sp;
}

// what the host derives from the options of a solve's windows
struct SolveTotals {
    int precision = 0;      // batch-wide: it selects the kernel variants
    int max_passes = 0;     // pass cap of the solve, from the largest iteration counts
    double time_cap = 0;    // host safety cap (seconds per inner solve), <= 0: none -- some window has no time limit
};

// The trimming quantiles of every path (k_trim_select, k_ev_finish, k_adjust_pose): a group rejects its landmarks of rank
// >= (int)(N * quantile), so a NaN or negative quantile would reject every landmark with a residual and one above 1 none.
static int quantile_check(const kba_options* o, std::string& why) {
    const std::pair<const char*, double> q[3] = {
        {"depth_quantile", o->depth_quantile}, {"reprojection_quantile", o->reprojection_quantile}, {"gp_quantile", o->gp_quantile}};
    for (const auto& e : q)
        if (!(e.second >= 0.0 && e.second <= 1.0)) {
            why = std::string("kba_options.") + e.first + " must lie in [0, 1] (got " + std::to_string(e.second) + ")";
            return KBA_ERR_BAD_ARG;
        }
    return KBA_OK;
}

// Every check of a solve's options, before anything is uploaded.  opts[i] is unit i's (per_unit, n entries) or opts[0] every
// unit's; live(i) false: unit i sits the solve out and its entry is not read.  Errors name the unit ("window 3: ...") when the
// options are per unit.
static int solve_options_check(int n, const kba_options* opts, bool per_unit, const char* unit, const std::function<bool(int)>& live,
                               SolveTotals& tot, std::string& why) {
    int first = -1, max_trim = 0, max_final = 0;
    bool no_cap = false;
    for (int i = 0; i < (per_unit ? n : 1); ++i) {
        if (per_unit && !live(i)) continue;
        const kba_options* o = &opts[i];
        const std::string at = per_unit ? std::string(unit) + std::to_string(i) + ": " : std::string();
        if (o->precision != 0 && o->precision != 1) { why = at + "kba_options.precision must be 0 (FP64) or 1 (FP32 linearisation)"; return KBA_ERR_BAD_ARG; }
        if (first >= 0 && o->precision != opts[first].precision) {
            why = at + "kba_options.precision differs from " + unit + std::to_string(first) + "'s: the precision is the same for the whole batch";
            return KBA_ERR_BAD_ARG;
        }
        if (quantile_check(o, why) != KBA_OK) { why = at + why; return KBA_ERR_BAD_ARG; }
        if (o->num_trim_rounds > 6 || (o->num_trim_rounds < 0 && o->num_rounds_option > 6)) {
            why = at + "at most 6 trimming rounds (KBA_MAX_SOLVES = 8 inner solves incl. one retry and the final solve)";
            return KBA_ERR_CAPACITY;
        }
        if (first < 0) { first = i; tot.precision = o->precision; tot.time_cap = o->solver_time_sec; }
        max_trim = std::max(max_trim, o->trim_solver_iterations); max_final = std::max(max_final, o->final_solver_iterations);
        no_cap |= !(o->solver_time_sec > 0);
        tot.time_cap = std::max(tot.time_cap, o->solver_time_sec);
    }
    // upper bound on passes: every solve needs (iterations + 2) passes, plus one pass per trimming step
    const int rounds_max = 7;
    tot.max_passes = rounds_max * (3 * max_trim + 4) + max_final + 8;
    if (no_cap) tot.time_cap = 0;
    return KBA_OK;
}

// The device options of every window of b into sp[0 .. n_win): opts[i] (per_window) or opts[0]; a window that sits the solve out
// keeps what the device holds (its entry is not read).  True when they differ from what the device holds, which b->wsp_dev then
// records: the caller uploads them.
static bool stage_params(kba_batch* b, bool per_window, const kba_options* opts, SolveParams* sp) {
    const int n = b->bd.n_win;
    const bool known = (int)b->wsp_dev.size() == n;
    const SolveParams one = make_params(opts);
    for (int i = 0; i < n; ++i) {
        if (b->desc_h[i].idle) {
            if (known) sp[i] = b->wsp_dev[i];
            else memset(&sp[i], 0, sizeof(SolveParams));
        } else {
            sp[i] = per_window ? make_params(&opts[i]) : one;
        }
    }
    if (known && memcmp(sp, b->wsp_dev.data(), sizeof(SolveParams) * n) == 0) return false;
    b->wsp_dev.assign(sp, sp + n);
    return true;
}

static int batch_run(kba_batch* b, const SolveTotals& tot);
static int batch_solve(kba_batch* b, bool per_window, const kba_options* opts) {
    if (!b || !opts) return fail(KBA_ERR_BAD_ARG, "bad argument to kba_batch_solve");
    SolveTotals tot;
    std::string why;
    const int rc = solve_options_check(b->bd.n_win, opts, per_window, "window ", [b](int i) { return !b->desc_h[i].idle; }, tot, why);
    if (rc != KBA_OK) return fail(rc, why);
    CU(cudaSetDevice(b->h->device));
    if (stage_params(b, per_window, opts, b->wsp.h)) CU(b->wsp.upload(b->h->stream));
    return batch_run(b, tot);
}

// a rank that fails leaves the collective solve: the in-process exchange releases the ranks waiting for it with an error
static int batch_solve_collective(kba_batch* b, bool per_window, const kba_options* opts) {
    const int rc = batch_solve(b, per_window, opts);
    if (rc != KBA_OK && b && b->bd.sharded && b->lc.xchg.abort) b->lc.xchg.abort(b->lc.xchg.user);
    return rc;
}
int kba_batch_solve(kba_batch* b, const kba_options* opt) { return batch_solve_collective(b, false, opt); }
int kba_batch_solve_opts(kba_batch* b, const kba_options* opts) { return batch_solve_collective(b, true, opts); }

// the solve of batch b with its options on the device (BatchDev::wsp), checked and derived into tot
static int batch_run(kba_batch* b, const SolveTotals& tot) {
    b->bd.precision = tot.precision;
    b->bd.lin1 = (b->lc.plan.fused && b->lc.knobs.lin_fused && tot.precision == 0 && b->lc.max_rank == 0) ? 1 : 0;
    kba_handle* h = b->h;
    CU(cudaSetDevice(h->device));
    cudaStream_t s = h->stream;
    LaunchCfg lc = b->lc;
    lc.time_jacobian = h->kernel_timing;
    if (h->kernel_timing && h->ev_pool.empty()) {
        h->ev_pool.resize(1024);
        for (auto& e : h->ev_pool) CU(cudaEventCreate(&e));
    }
    h->ev_used = 0;
    lc.ev_pool = h->ev_pool.data(); lc.ev_cap = (int)h->ev_pool.size(); lc.ev_used = &h->ev_used;
    CU(cudaMemsetAsync(b->bd.jac_obs, 0, sizeof(unsigned long long), s));
    // the evaluation kernels write the cost slots of the CTAs they launch and rely on the others being zero; the slot layout
    // differs between k_linearize and k_eval_obs (a batch may be solved with either: kba_options.precision)
    CU(cudaMemsetAsync(b->bd.cost_part_x, 0, sizeof(double) * (size_t)b->bd.n_win * b->bd.cost_parts, s));
    CU(cudaMemsetAsync(b->bd.cost_part_c, 0, sizeof(double) * (size_t)b->bd.n_win * b->bd.cost_parts, s));
    CU(cudaEventRecord(b->ev_a, s));
    if (launch_shard_gather(b->bd, lc, s)) return KBA_ERR_NCCL;  // message set by the exchange
    launch_reset(b->bd, lc, s);
    const int max_passes = tot.max_passes;
    const auto t0 = std::chrono::steady_clock::now();
    int check_every = 4;
    bool timed_out = false, poll_pending = false;
    // ---- graph paths (see solve_graph_mode) ----
    int gmode = solve_graph_mode();
    if (h->kernel_timing || launch_check_enabled() || s == nullptr || b->sg.unusable) gmode = 0;
    // Sharded solve: the NCCL all-reduces are captured with the kernels (flat graph, mode 1).  The first solve of a batch runs on
    // the stream so that NCCL sets its connections up outside a capture; the active-window count is read BEFORE the next graph is
    // launched (no look-ahead): it is identical on all ranks, and every rank must launch the same number of graphs.  The in-process
    // exchange synchronises its ranks' host threads at enqueue time, which a graph cannot hold: always the stream path.
    const bool lockstep = b->bd.sharded != 0;
    if (lockstep) gmode = (gmode && lc.xchg.capturable && shard_graph_enabled() && b->solves_done > 0) ? 1 : 0;
    if (gmode) {
        std::vector<unsigned char> key;
        key.reserve(sizeof(BatchDev) + 64);
        key_append(key, b->bd); key_append(key, gmode); key_append(key, max_passes); key_append(key, s);
        // the knobs are fixed at creation; the plan changes with uploads and track solves
        key_append(key, lc.plan); key_append(key, lc.max_rank); key_append(key, lc.xchg.user);
        if (!(b->sg.exec && b->sg.key == key) && !build_solve_graph(b, lc, gmode, max_passes, check_every, key)) gmode = 0;
    }
    if (gmode == 2) {
        CU(cudaMemsetAsync(b->loop_pass.d, 0, sizeof(int), s));
        CU(cudaGraphLaunch(b->sg.exec, s));
        CU(b->loop_pass.download(s));
        CU(cudaEventRecord(b->ev_b, s));
        CU(b->jac_obs.download(s));
        CU(wait_stream(h));
        CU(cudaGetLastError());
        CU(cudaEventElapsedTime(&b->last_solve_ms, b->ev_a, b->ev_b));
        h->counters.jacobian_obs += (long long)b->jac_obs.h[0];
        add_pass_counters(h->counters, b->sg.per_pass, b->loop_pass.h[0]);
        h->counters.launches_total += b->loop_pass.h[0];  // k_loop_cond
        b->solves_done++;
        return KBA_OK;
    }
    if (gmode == 1) {
        cudaEvent_t evs[2] = {b->ev_poll, b->ev_poll2};
        const int n_launch = (max_passes + check_every - 1) / check_every;
        int launched = 0;
        for (int g = 0; g < n_launch; ++g) {
            CU(cudaGraphLaunch(b->sg.exec, s));
            ++launched;
            CU(cudaEventRecord(evs[g & 1], s));
            if (lockstep) {
                CU(wait_event(h, evs[g & 1]));
                if (b->n_active.h[0] == 0) break;
            } else if (g >= 1) {  // the count of the previous launch is read while this one runs (the device never waits for the host)
                CU(wait_event(h, evs[(g - 1) & 1]));
                if (b->n_active.h[0] == 0) break;
                if (tot.time_cap > 0) {
                    const double el = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
                    if (el > KBA_MAX_SOLVES * tot.time_cap + 2.0) { timed_out = true; break; }
                }
            }
        }
        if (timed_out) g_last_error = "kba_batch_solve: host safety cap reached, unfinished windows carry KBA_ERR_TIMEOUT in kba_result.status";
        CU(cudaEventRecord(b->ev_b, s));
        CU(b->jac_obs.download(s));
        CU(wait_stream(h));
        CU(cudaGetLastError());
        CU(cudaEventElapsedTime(&b->last_solve_ms, b->ev_a, b->ev_b));
        h->counters.jacobian_obs += (long long)b->jac_obs.h[0];
        add_pass_counters(h->counters, b->sg.per_pass, (long long)launched * check_every);
        h->counters.launches_total += launched;  // k_count_active
        b->solves_done++;
        return KBA_OK;
    }
    for (int pass = 0; pass < max_passes; ++pass) {
        if (launch_pass(b->bd, lc, &h->counters, s)) {  // message set by the exchange
            cudaEventRecord(b->ev_b, s);
            return KBA_ERR_NCCL;
        }
        if (pass < 2) {  // a launch that fails fails in the first pass: do not let the windows spin to the safety cap
            const cudaError_t le = cudaGetLastError();
            if (le != cudaSuccess) { cudaEventRecord(b->ev_b, s); cudaStreamSynchronize(s); return fail(KBA_ERR_CUDA, std::string("kernel launch failed in kba_batch_solve: ") + cudaGetErrorString(le)); }
        }
        // Completion check without draining the queue: every `check_every` passes the active-window count is copied out behind an
        // event, the next passes are enqueued at once, and the count is READ one check later.  The device never waits for the
        // host (a synchronous poll would empty the queue a dozen times per solve); the price is
        // up to `check_every` passes enqueued after the last window finished, in which every kernel exits at once.  In a sharded
        // solve the state -- hence the count -- is identical on all ranks, so they still issue the same passes.
        if ((pass + 1) % check_every == 0 || pass + 1 == max_passes) {
            if (poll_pending) {
                CU(wait_event(h, b->ev_poll));
                poll_pending = false;
                if (b->n_active.h[0] == 0) break;
                if (tot.time_cap > 0 && !b->bd.sharded) {  // host safety cap, see below
                    const double el = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
                    if (el > KBA_MAX_SOLVES * tot.time_cap + 2.0) { timed_out = true; break; }
                }
            }
            launch_count_active(b->bd, s);
            CU(b->n_active.download(s));
            CU(cudaEventRecord(b->ev_poll, s));
            poll_pending = true;
            // max_solver_time_in_seconds is applied PER INNER SOLVE on the device (k_lm_update, like ceres), which always
            // lets the final solve start; the host only guards against a stuck device with the budget of every possible
            // inner solve.  A sharded solve is collective: its ranks must issue the same passes, so no rank may leave on
            // its own clock (the iteration caps bound it).
        }
    }
    if (timed_out) g_last_error = "kba_batch_solve: host safety cap reached, unfinished windows carry KBA_ERR_TIMEOUT in kba_result.status";
    CU(cudaEventRecord(b->ev_b, s));
    CU(b->jac_obs.download(s));
    CU(wait_stream(h));
    CU(cudaGetLastError());
    CU(cudaEventElapsedTime(&b->last_solve_ms, b->ev_a, b->ev_b));
    h->counters.jacobian_obs += (long long)b->jac_obs.h[0];
    for (int i = 0; i + 1 < h->ev_used; i += 2) {
        float ms = 0.f;
        CU(cudaEventElapsedTime(&ms, h->ev_pool[i], h->ev_pool[i + 1]));
        h->counters.ms_jacobian += ms;
    }
    b->solves_done++;
    return KBA_OK;
}

static int batch_set_shard(kba_batch* b, const kba::Exchange& xchg, int32_t lm_begin, int32_t lm_total) {
    BatchDev& bd = b->bd;
    if (bd.n_win != 1) return fail(KBA_ERR_BAD_ARG, "a sharded batch holds exactly one window (this rank's shard)");
    if (lm_begin < 0 || lm_total < lm_begin + (int)bd.tot_lm) return fail(KBA_ERR_BAD_ARG, "landmark block outside the window");
    if (bd.sharded) return fail(KBA_ERR_BAD_ARG, "kba_batch_set_shard called twice");
    const WinDesc& d = b->desc_h[0];
    CU(cudaSetDevice(b->h->device));
    cudaStream_t s = b->h->stream;
    int bad = 0;
    bad |= b->dev_alloc(&bd.xs, 16 + (size_t)xchg.world);
    if (bad) return fail(KBA_ERR_CUDA, "out of device memory (shard buffers)");
    // what the ranks must agree on (max over the ranks): the size of the reduced system, whether any rank holds ground points, and
    // the cost partial slots of the exchange (their count follows the rank's observations)
    {
        double v[4] = {(double)d.nr_cap, -(double)d.nr_cap, bd.tot_gp > 0 ? 1.0 : 0.0, (double)bd.cost_parts};
        CU(cudaMemcpyAsync(bd.xs, v, sizeof v, cudaMemcpyHostToDevice, s));
        if (xchg.allreduce(xchg.user, bd.xs, bd.xs, 4, 1, s)) return KBA_ERR_NCCL;
        CU(cudaMemcpyAsync(v, bd.xs, sizeof v, cudaMemcpyDeviceToHost, s));
        CU(cudaStreamSynchronize(s));
        if (v[0] != -v[1])
            return fail(KBA_ERR_BAD_ARG, "the shards size different reduced systems: with plane_reg_weight = 0, plane blocks exist on "
                                         "the ranks holding ground-plane residuals only; give every shard the window's plane_reg_weight");
        bd.shard_gp = v[2] > 0.0 ? 1 : 0;
        bd.shard_cost_parts = (int)v[3];
    }
    const long long n_g = bd.shard_gp ? 65LL * d.n_kf + 1 : 0;  // kba_kernels.cu: shard_gp_doubles
    const size_t n_x = (size_t)d.nr_cap * d.nr_cap + (size_t)d.n_kf * 27 + (size_t)n_g + (size_t)bd.shard_cost_parts + 2;
    bad |= b->dev_alloc(&bd.trim_send, 3 * (size_t)lm_total); bad |= b->dev_alloc(&bd.trim_glob, 3 * (size_t)lm_total);
    bad |= b->dev_alloc(&bd.reject_glob, (size_t)lm_total);
    bad |= b->dev_alloc(&bd.x_send, n_x); bad |= b->dev_alloc(&bd.x_recv, n_x);
    if (bd.shard_gp) {
        bad |= b->dev_alloc(&bd.gp_send, (size_t)lm_total); bad |= b->dev_alloc(&bd.gp_kf_glob, (size_t)lm_total);
        bad |= b->dev_alloc(&bd.act_glob, (size_t)lm_total); bad |= b->dev_alloc(&bd.kf_gp_glob, (size_t)d.n_kf);
    }
    if (bad) return fail(KBA_ERR_CUDA, "out of device memory (shard buffers)");
    CU(cudaMemsetAsync(bd.xs, 0, (16 + (size_t)xchg.world) * sizeof(double), s));
    CU(cudaMemsetAsync(bd.trim_send, 0, 3 * (size_t)lm_total * sizeof(double), s));
    CU(cudaMemsetAsync(bd.x_send, 0, n_x * sizeof(double), s));
    CU(cudaMemsetAsync(bd.x_recv, 0, n_x * sizeof(double), s));
    bd.shard_rank = xchg.rank; bd.shard_world = xchg.world;
    bd.sharded = 1; bd.lm_begin = lm_begin; bd.lm_total = lm_total;
    b->lc.xchg = xchg;
    b->lc.shard_win.nr_cap = d.nr_cap; b->lc.shard_win.n_kf = d.n_kf;
    return KBA_OK;
}

int kba_batch_set_shard(kba_batch* b, kba_shard_comm* comm, int32_t lm_begin, int32_t lm_total) {
    if (!b || !comm) return fail(KBA_ERR_BAD_ARG, "bad argument to kba_batch_set_shard");
    const kba::Exchange xchg = kba_shard_exchange(comm);
    const int rc = batch_set_shard(b, xchg, lm_begin, lm_total);
    if (rc != KBA_OK && xchg.abort) xchg.abort(xchg.user);  // see kba_batch_solve
    return rc;
}

int kba_batch_download(kba_batch* b, kba_result* res) {
    if (!b || !res) return fail(KBA_ERR_BAD_ARG, "bad argument to kba_batch_download");
    CU(cudaSetDevice(b->h->device));
    cudaStream_t s = b->h->stream;
    CU(b->state.download(s)); CU(b->log.download(s));
    CU(b->pose_out[0].download(s)); CU(b->pose_out[1].download(s));
    const BatchDev& bd = b->bd;
    if (b->lc.plan.device_pack) {  // landmarks come back in the caller's order: one kernel, one copy per array
        launch_unpack_landmarks(bd, b->lm_user.d, b->rej_user.d, s);
        CU(b->lm_user.download(s)); CU(b->rej_user.download(s));
    } else {
        CU(b->lm_out[0].download(s)); CU(b->lm_out[1].download(s)); CU(b->lm_active.download(s));
    }
    CU(b->plane_out[0].download(s)); CU(b->plane_out[1].download(s));
    CU(wait_stream(b->h));
    b->d2h_bytes = sizeof(WinState) * bd.n_win + 2 * (7 + 4) * 8 * bd.tot_kf + (b->lc.plan.device_pack ? 1 : 2) * 3 * 8 * bd.tot_lm + bd.tot_lm;
    for (int i = 0; i < bd.n_win; ++i) {
        const WinDesc& d = b->desc_h[i];
        const WinState& st = b->state.h[i];
        kba_result& r = res[i];
        const int cur = st.cur;
        if (r.kf_pose) memcpy(r.kf_pose, b->pose_out[cur].h + 7 * (size_t)d.kf_off, sizeof(double) * 7 * d.n_kf);
        if (r.kf_plane) memcpy(r.kf_plane, b->plane_out[cur].h + 4 * (size_t)d.kf_off, sizeof(double) * 4 * d.n_kf);
        if (b->lc.plan.device_pack) {
            if (r.lm_pos) memcpy(r.lm_pos, b->lm_user.h + 3 * (size_t)d.lm_off, 3 * sizeof(double) * d.n_lm);
            if (r.lm_rejected) memcpy(r.lm_rejected, b->rej_user.h + d.lm_off, d.n_lm);
        } else {
            const int* orig = b->lm_orig.h + d.lm_off;
            if (r.lm_pos)
                for (int j = 0; j < d.n_lm; ++j) memcpy(r.lm_pos + 3 * (size_t)orig[j], b->lm_out[cur].h + 3 * (size_t)(d.lm_off + j), 3 * sizeof(double));
            if (r.lm_rejected) for (int j = 0; j < d.n_lm; ++j) r.lm_rejected[orig[j]] = !b->lm_active.h[d.lm_off + j];
        }
        r.num_solves = st.n_solves;
        for (int q = 0; q < st.n_solves && q < KBA_MAX_SOLVES; ++q) {
            const SolveSummary& ss = st.solves[q];
            kba_solve_summary& o = r.solves[q];
            o.initial_cost = ss.initial_cost; o.final_cost = ss.final_cost; o.num_iterations = ss.num_iterations;
            o.num_successful_steps = ss.num_successful_steps; o.termination = ss.termination;
            o.num_landmarks = ss.num_landmarks; o.num_residual_blocks = ss.num_residual_blocks; o.reserved_ = 0;
        }
        r.initial_cost = st.n_solves > 0 ? st.solves[0].initial_cost : 0.0;
        r.final_cost = st.n_solves > 0 ? st.solves[st.n_solves - 1].final_cost : 0.0;
        r.status = (st.phase == PH_DONE) ? KBA_OK : KBA_ERR_TIMEOUT;  // host safety cap hit (see kba_batch_solve)
        r.time_sec = 1e-3 * b->last_solve_ms;
        int n = 0;
        if (r.iterations) {
            for (; n < st.log_n && n < r.iterations_capacity; ++n) {
                const IterRecord& e = b->log.h[(size_t)i * kIterLogCap + n];
                kba_iteration& o = r.iterations[n];
                o.cost = e.cost; o.cost_change = e.cost_change; o.gradient_max_norm = e.gradient_max_norm;
                o.step_norm = e.step_norm; o.relative_decrease = e.relative_decrease; o.trust_region_radius = e.radius;
                o.iteration = e.iteration; o.solve_index = e.solve_index; o.step_is_valid = e.valid; o.step_is_successful = e.successful;
            }
        }
        r.num_iteration_records = n;
    }
    return KBA_OK;
}

int kba_batch_transfer_bytes(kba_batch* b, int64_t* h2d, int64_t* d2h) {
    if (!b) return fail(KBA_ERR_BAD_ARG, "null batch");
    if (h2d) *h2d = (int64_t)b->h2d_bytes;
    if (d2h) *d2h = (int64_t)b->d2h_bytes;
    return KBA_OK;
}

void kba_batch_destroy(kba_batch* b) {
    if (!b) return;
    cudaStreamSynchronize(b->h->stream);
#ifdef KBA_PROF
    if (b->bd.prof) {
        unsigned long long c[16];
        cudaMemcpy(c, b->bd.prof, sizeof c, cudaMemcpyDeviceToHost);
        fprintf(stderr, "[kba prof] fused Schur kernel, cycles summed over warps: consumers wait %llu multiply %llu | producers "
                "wait-empty %llu set-up %llu copies %llu\n", c[0], c[1], c[4], c[5], c[6]);
    }
#endif
    b->release();
    delete b;
}

int kba_batch_jacobian_pass(kba_batch* b, const kba_options* opt, int32_t repeats, float* ms_out) {
    if (!b || !opt || repeats < 1) return fail(KBA_ERR_BAD_ARG, "bad argument to kba_batch_jacobian_pass");
    kba_handle* h = b->h;
    cudaStream_t s = h->stream;
    if (opt->precision != 0 && opt->precision != 1) return fail(KBA_ERR_BAD_ARG, "kba_options.precision must be 0 or 1");
    b->bd.precision = opt->precision;
    if (stage_params(b, false, opt, b->wsp.h)) CU(b->wsp.upload(s));
    launch_reset(b->bd, b->lc, s);
    launch_force_linearize(b->bd, s);
    CU(cudaEventRecord(b->ev_a, s));
    for (int i = 0; i < repeats; ++i) launch_jacobian_only(b->bd, s);
    CU(cudaEventRecord(b->ev_b, s));
    CU(cudaStreamSynchronize(s));
    CU(cudaGetLastError());
    float ms = 0.f;
    CU(cudaEventElapsedTime(&ms, b->ev_a, b->ev_b));
    if (ms_out) *ms_out = ms;
    h->counters.launches_total += repeats; h->counters.launches_jacobian += repeats;
    h->counters.ms_jacobian += ms; h->counters.jacobian_obs += (long long)repeats * b->bd.tot_obs;
    CU(cudaMemsetAsync(b->bd.jac_obs, 0, sizeof(unsigned long long), s));
    return KBA_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
static int solve_batch(kba_handle* h, int32_t n_windows, const kba_window* w, bool per_window, const kba_options* opts, kba_result* res) {
    if (!h || !w || !opts || !res) return fail(KBA_ERR_BAD_ARG, "null argument to kba_solve_batch");
    SolveTotals tot;
    std::string why;
    int rc = solve_options_check(n_windows, opts, per_window, "window ", [](int) { return true; }, tot, why);
    if (rc != KBA_OK) return fail(rc, why);
    kba_batch* b = nullptr;
    rc = kba_batch_create(h, n_windows, w, &b);
    if (rc != KBA_OK) return rc;
    rc = batch_solve(b, per_window, opts);
    if (rc == KBA_OK) rc = kba_batch_download(b, res);
    kba_batch_destroy(b);
    return rc;
}

int kba_solve_batch(kba_handle* h, int32_t n_windows, const kba_window* w, const kba_options* opt, kba_result* res) {
    return solve_batch(h, n_windows, w, false, opt, res);
}
int kba_solve_batch_opts(kba_handle* h, int32_t n_windows, const kba_window* w, const kba_options* opts, kba_result* res) {
    return solve_batch(h, n_windows, w, true, opts, res);
}

int kba_solve_window(kba_handle* h, const kba_window* w, const kba_options* opt, kba_result* res) {
    return kba_solve_batch(h, 1, w, opt, res);
}

int kba_eval(kba_handle* h, const kba_window* w, const kba_options* opt, kba_eval_out* out) {
    if (!h || !w || !opt || !out) return fail(KBA_ERR_BAD_ARG, "null argument to kba_eval");
    kba_batch* b = nullptr;
    int rc = batch_create(h, 1, w, nullptr, Purpose::HostPack, &b);
    if (rc != KBA_OK) return rc;
    float ms;
    rc = kba_batch_jacobian_pass(b, opt, 1, &ms);
    if (rc != KBA_OK) { kba_batch_destroy(b); return rc; }
    const BatchDev& bd = b->bd;
    const size_t n = (size_t)w->n_obs;
    std::vector<double> res_h(3 * n + 1), jp_h(18 * n + 1), jl_h(9 * n + 1), cost_h(bd.cost_parts);
    std::vector<int> offp(w->n_kf);
    WinState st;
    cudaStream_t s = h->stream;
    cudaError_t ce = cudaSuccess;
    auto cp = [&](void* dst, const void* src, size_t bytes) {
        if (ce == cudaSuccess) ce = cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, s);
    };
    cp(res_h.data(), bd.res, 3 * n * sizeof(double));
    cp(jp_h.data(), bd.jp, 18 * n * sizeof(double));
    double* jl_dev = bd.jl;
    if (bd.fused) {  // J_l is not materialised on the fused path: expand it on the device the way its consumers do
        if (b->dev_alloc(&jl_dev, 9 * n)) { kba_batch_destroy(b); return fail(KBA_ERR_CUDA, "out of device memory (kba_eval)"); }
        launch_expand_jl(bd, jl_dev, s);
    }
    cp(jl_h.data(), jl_dev, 9 * n * sizeof(double));
    cp(cost_h.data(), bd.cost_part_x, bd.cost_parts * sizeof(double));
    cp(offp.data(), bd.off_pose, w->n_kf * sizeof(int));
    cp(&st, bd.state, sizeof(WinState));
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(s);
    if (ce != cudaSuccess) { kba_batch_destroy(b); return fail(KBA_ERR_CUDA, cudaGetErrorString(ce)); }
    for (size_t e = 0; e < n; ++e) {  // e: internal (sorted) observation slot, o: the caller's observation index
        const size_t o = (size_t)b->obs_orig.h[e];
        const bool fixed = offp[w->obs_kf[o]] < 0;
        // precision 1: the streams hold floats (same component-major layout); J_l expanded on the fused path is FP64 either way
        auto at = [&](const std::vector<double>& v, size_t idx, bool f32) {
            return f32 ? (double)reinterpret_cast<const float*>(v.data())[idx] : v[idx];
        };
        const bool f32 = opt->precision != 0;
        if (out->residual) for (int q = 0; q < 3; ++q) out->residual[3 * o + q] = at(res_h, q * n + e, f32);
        if (out->jac_pose) for (int q = 0; q < 18; ++q) out->jac_pose[18 * o + q] = fixed ? 0.0 : at(jp_h, q * n + e, f32);
        if (out->jac_lm) for (int q = 0; q < 9; ++q) out->jac_lm[9 * o + q] = at(jl_h, q * n + e, f32 && !bd.fused);
    }
    if (out->cost) { double c = 0; for (int q = 0; q < bd.cost_parts; ++q) c += cost_h[q]; out->cost[0] = c; }
    if (out->failed) out->failed[0] = st.eval_failed;
    kba_batch_destroy(b);
    return KBA_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// persistent, device-resident window (include/kba_b200.h, kba_track_*)
// ---------------------------------------------------------------------------------------------------------------------
void kba_track_destroy(kba_track* t) {
    if (!t) return;
    cudaStreamSynchronize(t->set.h->stream);
    delete t;
}

// A dummy window of a track's largest shape: the batch created from it has the capacity every later solve of the track fits in.
// The observations are spread evenly over the landmarks and, within a landmark, over the keyframes in ascending order: the packing
// kernels run once on this window (create = upload), and their per-landmark loops (insertion sort of a track, k_track_sort /
// k_pack_obs) are written for tracks of a few dozen observations -- one landmark carrying all 2^18 of them kept a single GPU
// thread busy for minutes.
// Its reduced system is sized for the larger of its windows without plane blocks (6 rows per keyframe) and with them (10 rows per
// keyframe, for at most kTrackPlaneKf keyframes): 192 rows at 30 keyframes, the fused path.  The capacity window of the fused
// solver of a track with win_rows > kFusedMaxRows is clipped to kTrackFusedKf keyframes; that of its large-window solver has all
// win_keyframes and at least win_rows rows.
constexpr int kTrackPlaneKf = (kFusedMaxRows - 1) / 10;    // 18 keyframes with plane blocks
constexpr int kTrackFusedKf = (kFusedMaxRows - 1) / 6;     // 30 keyframes without
static bool has_large(const kba_track_caps& c) { return c.win_rows > kFusedMaxRows; }
struct CapacityWindow {
    std::vector<double> pose, plane, lmp, lmw, gw;
    std::vector<uint8_t> fixed;
    std::vector<int32_t> ptr, okf, gl, gk;
    std::vector<float> u, v, d;
    kba_window w{};
    int rows = 0;
    CapacityWindow(const kba_track_caps& c, bool large, int n_cam, const double* cam_intr, const double* cam_pose) {
        const int K = large ? c.win_keyframes : std::min(c.win_keyframes, kTrackFusedKf);
        const int L = c.win_landmarks, O = c.win_observations, G = c.win_ground;
        rows = std::max(reduced_rows(K, false), G > 0 ? reduced_rows(std::min(K, kTrackPlaneKf), true) : 0);
        if (large) rows = std::max(rows, c.win_rows);
        pose.assign(7 * (size_t)K, 0.0); plane.assign(4 * (size_t)K, 0.0); lmp.assign(3 * (size_t)L, 0.0); lmw.assign(L, 1.0);
        gw.assign(std::max(G, 1), 1.0);
        fixed.assign(K, 0);
        ptr.assign(L + 1, O); okf.assign(O, 1); gl.assign(std::max(G, 1), 0); gk.assign(std::max(G, 1), 1);
        u.assign(O, 0.f); v.assign(O, 0.f); d.assign(O, -1.f);
        for (int k = 0; k < K; ++k) { pose[7 * k] = 1.0; plane[4 * k + 2] = 1.0; }
        for (int j = 0; j < L; ++j) lmp[3 * j + 2] = 10.0;
        for (int g = 0; g < G; ++g) gl[g] = g;
        fixed[0] = 1;
        for (int j = 0; j <= L; ++j) ptr[j] = (int32_t)(((long long)O * j) / L);
        for (int j = 0; j < L; ++j) {
            const int n = ptr[j + 1] - ptr[j];
            for (int i = 0; i < n; ++i) okf[ptr[j] + i] = (n <= K) ? i : (int32_t)(((long long)i * K) / n);  // non-decreasing
        }
        w.n_kf = K; w.n_cam = n_cam; w.n_lm = L; w.n_obs = O; w.n_gp = G;
        w.kf_pose = pose.data(); w.kf_fixed = fixed.data(); w.kf_plane = plane.data(); w.cam_intr = cam_intr; w.cam_pose = cam_pose;
        w.lm_pos = lmp.data(); w.lm_weight = lmw.data(); w.lm_obs_ptr = ptr.data(); w.obs_kf = okf.data(); w.obs_u = u.data();
        w.obs_v = v.data(); w.obs_d = d.data(); w.gp_lm = gl.data(); w.gp_kf = gk.data(); w.gp_weight = gw.data();
        w.plane_reg_weight = G > 0 ? 10.0 : 0.0;
    }
};

// what one solve of the stored window asks for (the arguments of kba_track_solve, one kba_track_request of a group)
struct TrackRequest {
    int32_t n_kf = 0;
    const int32_t* kf_slot = nullptr;
    const uint8_t* kf_fixed = nullptr;
    int32_t n_lm = 0;
    const int32_t* lm_slot = nullptr;
    const kba_window* sel = nullptr;       // nullptr: the track sits a group solve out
    int max_meas = 0, n_free = 0;          // filled by track_check: largest keyframe measurement count, free keyframes
    int n_meas = 0;                        // filled by track_check: measurements of the listed keyframes, a bound on the observations
    bool device_gp = false;                // filled by track_check: sel->gp_lm lists candidates, attached by k_track_ground
    int rows = 0;                          // filled by track_check: reduced rows kba_batch_create sizes the window for (reduced_rows,
                                           // plane blocks counted whenever candidates are given)
    bool ranked = false;                   // the landmarks are the track's ranking (kba_track_solve_ranked): lm_slot is not read
    bool rank_gp = false;                  // ... and so are the ground-plane candidates (sel->n_gp of them)
    kba_window ranked_sel{};               // a ranked request's window (ranked_check): sel points here
};

// ground points attached on the device: candidates in gp_lm, no keyframes or weights
static bool device_attached(const kba_window* sel) { return sel->n_gp > 0 && sel->gp_lm && !sel->gp_kf && !sel->gp_weight; }

// plane_reg_weight < 0: the reference's rule (cpp:717-719), 10 iff a ground-plane residual is in the window.  Host lists resolve
// it here; with candidates k_track_ground resolves it from the residuals it keeps.
static double plane_reg_weight(const kba_window* sel) {
    return sel->plane_reg_weight < 0 ? (sel->n_gp > 0 ? 10.0 : 0.0) : sel->plane_reg_weight;
}

// every argument check of a track solve, before anything is uploaded or launched
static int track_check(const kba_track* t, TrackRequest& q, std::string& why) {
    if (!q.kf_slot || !q.kf_fixed || (!q.lm_slot && !q.ranked) || !q.sel) { why = "null argument"; return KBA_ERR_BAD_ARG; }
    const kba_track_caps& c = t->caps;
    const kba_window* sel = q.sel;
    if (q.n_kf < 3) { why = "fewer than 3 keyframes"; return KBA_ERR_NOT_ENOUGH_KF; }
    if (q.n_kf > c.win_keyframes || q.n_lm > c.win_landmarks || q.n_lm < 0 || sel->n_gp < 0 || sel->n_gp > c.win_ground) {
        why = "window larger than the capacities given to kba_track_create"; return KBA_ERR_CAPACITY;
    }
    long long n_meas = 0;
    q.max_meas = 0; q.n_free = 0;
    for (int k = 0; k < q.n_kf; ++k) {
        const int slot = q.kf_slot[k];
        if (slot < 0 || slot >= t->td.kf_cap || !t->kf_live[slot]) { why = "keyframe slot not pushed"; return KBA_ERR_BAD_ARG; }
        n_meas += t->m_cnt[slot]; q.max_meas = std::max(q.max_meas, t->m_cnt[slot]);
        q.n_free += q.kf_fixed[k] ? 0 : 1;
    }
    if (n_meas > c.win_observations) { why = "more observations than win_observations"; return KBA_ERR_CAPACITY; }
    q.n_meas = (int)n_meas;
    for (int j = 0; j < q.n_lm && !q.ranked; ++j)
        if (q.lm_slot[j] < 0 || q.lm_slot[j] >= t->td.lm_cap) { why = "landmark slot out of range"; return KBA_ERR_BAD_ARG; }
    q.device_gp = q.rank_gp || device_attached(sel);
    if (q.rank_gp) {
        // the ranking's ground candidates: ascending indices into its selection by construction
    } else if (q.device_gp) {
        for (int g = 0; g < sel->n_gp; ++g)
            if (sel->gp_lm[g] < 0 || sel->gp_lm[g] >= q.n_lm || (g > 0 && sel->gp_lm[g] <= sel->gp_lm[g - 1])) {
                why = "ground-plane candidates must be strictly ascending indices into lm_slot"; return KBA_ERR_BAD_ARG;
            }
    } else {
        for (int g = 0; g < sel->n_gp; ++g)
            if (!sel->gp_lm || !sel->gp_kf || !sel->gp_weight || sel->gp_lm[g] < 0 || sel->gp_lm[g] >= q.n_lm || sel->gp_kf[g] < 0 ||
                sel->gp_kf[g] >= q.n_kf) {
                why = "ground-plane index out of range (or only one of gp_kf / gp_weight given)"; return KBA_ERR_BAD_ARG;
            }
    }
    const bool planes = sel->n_gp > 0 || sel->plane_reg_weight > 0;
    if (planes && c.win_ground == 0) { why = "the track was created without ground-plane capacity"; return KBA_ERR_CAPACITY; }
    q.rows = reduced_rows(q.n_kf, planes);
    if (c.win_rows == 0) {
        // a request that can carry plane blocks stays on the fused path with all its keyframes (kba_batch_create's small_syrk rule)
        if ((sel->n_gp > 0 || sel->plane_reg_weight != 0) && reduced_rows(q.n_kf, true) > kFusedMaxRows) {
            why = "more than 18 keyframes with ground-plane blocks (184 reduced rows) -- such windows go through kba_solve_window";
            return KBA_ERR_CAPACITY;
        }
    } else if (q.rows > c.win_rows) {
        why = "a window of " + std::to_string(q.rows) + " reduced rows (6 per keyframe, 10 with ground-plane blocks, plus one) is larger "
              "than win_rows = " + std::to_string(c.win_rows);
        return KBA_ERR_CAPACITY;
    }
    if (sel->scale_weight != 0 && (sel->scale_kf0 < 0 || sel->scale_kf0 >= q.n_kf || sel->scale_kf1 < 0 || sel->scale_kf1 >= q.n_kf)) {
        why = "scale regulariser keyframe out of range"; return KBA_ERR_BAD_ARG;
    }
    return KBA_OK;
}

// the window descriptor of a checked request (n_obs is written by the gather kernels); offsets and capacities stay as created
static void track_desc(WinDesc& d, const kba_track* t, const TrackRequest& q) {
    const kba_window* sel = q.sel;
    d.n_kf = q.n_kf; d.n_lm = q.n_lm; d.n_obs = 0;
    d.n_gp = q.device_gp ? 0 : sel->n_gp;  // candidates: k_track_ground writes the count it keeps
    d.n_chunks = (q.n_lm + 31) / 32; d.n_groups = (q.n_lm + 7) / 8;
    d.scale_kf0 = sel->scale_kf0; d.scale_kf1 = sel->scale_kf1; d.scale_weight = sel->scale_weight; d.scale_value = sel->scale_value;
    d.plane_reg_weight = q.device_gp ? sel->plane_reg_weight : plane_reg_weight(sel);
    d.plane_dist_fixed = sel->plane_dist_fixed; d.landmarks_fixed = 0;
    d.speed_kf = 0; d.speed_weight = 0; d.speed_dt = 1;
    d.max_rank = t->n_cam > 1 ? t->n_cam - 1 : 0;  // a rig may see a landmark from several cameras of one keyframe
    d.idle = 0;
}

// reduced rows of the free keyframes of a checked request, which select the fused Schur kernel instance.  The launch
// configuration is fixed before the gather, so a request with candidates counts plane rows even if none of them is attached: an
// 18-free-keyframe window with nothing attached runs the seven-slot kernel where kba_solve_window runs the six-slot one (and
// rounds differently).
static int track_free_rows(const TrackRequest& q) {
    return reduced_rows(q.n_free, q.device_gp || q.sel->n_gp > 0 || plane_reg_weight(q.sel) > 0);
}

// a track sitting a group solve out: nothing to gather, k_reset_state puts the window straight into PH_DONE
static void idle_desc(WinDesc& d) {
    d.n_kf = 0; d.n_lm = 0; d.n_obs = 0; d.n_gp = 0; d.n_chunks = 0; d.n_groups = 0;
    d.scale_weight = 0; d.plane_reg_weight = 0; d.plane_dist_fixed = 0; d.landmarks_fixed = 0; d.speed_weight = 0; d.max_rank = 0;
    d.idle = 1;
}

static void idle_result(kba_result& r) {
    r.num_iteration_records = 0; r.num_solves = 0; r.status = KBA_OK;
    r.initial_cost = 0.0; r.final_cost = 0.0; r.time_sec = 0.0;
}

static TrackSel track_sel(const TrackRequest& q, const int* kf_slot_d, const uint8_t* kf_fixed_d, const int* lm_slot_d, const int* cand_d) {
    TrackSel ts;
    ts.kf_slot = kf_slot_d; ts.kf_fixed = kf_fixed_d; ts.lm_slot = lm_slot_d; ts.n_kf = q.n_kf; ts.n_lm = q.n_lm; ts.max_meas = q.max_meas;
    ts.auto_scale = q.sel->scale_weight < 0 ? 1 : 0;
    if (q.device_gp) { ts.gp_cand = cand_d; ts.n_cand = q.sel->n_gp; }
    return ts;
}

// ints at the front of TrackSolver::lists that hold the options of n windows
static size_t params_ints(int n) {
    static_assert(sizeof(SolveParams) % 8 == 0, "the lists after the options stay 8-byte aligned");
    return (size_t)n * sizeof(SolveParams) / sizeof(int);
}

// the solver of tracks ts[0..n): one capacity window per track, so its batch has room for every window a track's caps allow on
// the fused path (large = false) or on the large-window path.  On failure everything it allocated is freed again.
static int track_solver_create(kba_handle* h, int n, kba_track* const* ts, bool large, TrackSolver& sv, const std::string& who) {
    std::vector<std::unique_ptr<CapacityWindow>> cws;
    std::vector<kba_window> ws;
    std::vector<int> rows;
    size_t list_ints = params_ints(n);
    for (int i = 0; i < n; ++i) {
        const kba_track* t = ts[i];
        cws.emplace_back(new CapacityWindow(t->caps, large, t->n_cam, t->cam_intr.data(), t->cam_pose.data()));
        ws.push_back(cws.back()->w);
        rows.push_back(cws.back()->rows);
        list_ints += (size_t)t->caps.win_keyframes + t->caps.win_landmarks + (t->caps.win_keyframes + 3) / 4 + t->caps.win_ground;
    }
    const int rc = batch_create(h, n, ws.data(), rows.data(), large ? Purpose::TrackLarge : Purpose::TrackFused, &sv.batch);
    if (rc != KBA_OK) return rc;
    if (!sv.batch->lc.plan.device_pack) { sv.release(); return fail(KBA_ERR_CAPACITY, who + ": device packing is disabled (KBA_FUSED / KBA_DEVICE_PACK)"); }
    int bad = 0;
    bad |= sv.tdev.alloc(n, true); bad |= sv.tsel.alloc(n, true); bad |= sv.lists.alloc(list_ints, true);
    if (bad) { sv.release(); return fail(KBA_ERR_CUDA, who + ": out of memory"); }
    sv.batch->bd.wsp = reinterpret_cast<const SolveParams*>(sv.lists.d);  // the options travel with the lists
    return KBA_OK;
}

int kba_track_create(kba_handle* h, const kba_track_caps* c, int32_t n_cam, const double* cam_intr, const double* cam_pose, kba_track** out) {
    if (!h || !c || !out || !cam_intr || !cam_pose || n_cam < 1) return fail(KBA_ERR_BAD_ARG, "bad argument to kba_track_create");
    if (c->max_keyframes < 3 || c->max_landmarks < 1 || c->max_measurements < 1 || c->win_keyframes < 3 || c->win_landmarks < 1 ||
        c->win_observations < 1 || c->win_ground < 0 || c->win_ground > c->win_landmarks)
        return fail(KBA_ERR_BAD_ARG, "kba_track_create: capacities");
    if (c->win_rows < 0 || (c->win_rows > 0 && c->win_rows < reduced_rows(c->win_keyframes, false)))
        return fail(KBA_ERR_BAD_ARG, "kba_track_create: win_rows must be 0 or at least 6 * win_keyframes + 1");
    if (c->win_rows > kTrackMaxRows)
        return fail(KBA_ERR_CAPACITY, "kba_track_create: win_rows larger than 640 (the largest window a track's solver is sized for)");
    if (c->win_rows == 0 && reduced_rows(c->win_keyframes, false) > kFusedMaxRows)
        return fail(KBA_ERR_CAPACITY, "kba_track_create: the stored window must fit the fused path (<= 184 reduced rows: 30 keyframes; "
                                      "<= 32768 landmarks) -- give win_rows for larger windows");
    if (c->win_landmarks > kPackMaxLandmarks)
        return fail(KBA_ERR_CAPACITY, "kba_track_create: more than 32768 landmarks per window (the device sort)");
    CU(cudaSetDevice(h->device));
    kba_track* t = new kba_track();
    t->set.h = h; t->set.tracks = {t}; t->caps = *c; t->n_cam = n_cam;
    t->cam_intr.assign(cam_intr, cam_intr + 3 * (size_t)n_cam);
    t->cam_pose.assign(cam_pose, cam_pose + 7 * (size_t)n_cam);
    int rc = track_solver_create(h, 1, &t, false, t->set.solver, "kba_track_create");
    if (rc == KBA_OK && has_large(*c)) rc = track_solver_create(h, 1, &t, true, t->set.large, "kba_track_create");
    if (rc != KBA_OK) { delete t; return rc; }
    int bad = 0;
    TrackDev& td = t->td;
    DevAllocs& dev = t->dev;
    td.kf_cap = c->max_keyframes; td.lm_cap = c->max_landmarks; td.m_cap = c->max_measurements;
    bad |= dev.alloc(&td.kf_pose, 7 * (size_t)td.kf_cap); bad |= dev.alloc(&td.kf_plane, 4 * (size_t)td.kf_cap);
    bad |= dev.alloc(&td.m_off, td.kf_cap); bad |= dev.alloc(&td.m_cnt, td.kf_cap);
    for (int b2 = 0; b2 < 2; ++b2) {
        for (int q = 0; q < 2; ++q) bad |= dev.alloc(&t->arena_i[b2][q], td.m_cap);
        for (int q = 0; q < 3; ++q) bad |= dev.alloc(&t->arena_f[b2][q], td.m_cap);
    }
    bad |= dev.alloc(&td.lm_pos, 3 * (size_t)td.lm_cap); bad |= dev.alloc(&td.lm_weight, td.lm_cap); bad |= dev.alloc(&td.sel_index, td.lm_cap);
    bad |= dev.alloc(&td.cursor, c->win_landmarks); bad |= dev.alloc(&td.key, c->win_observations); bad |= dev.alloc(&td.n_depth, 1);
    if (bad) { kba_track_destroy(t); return fail(KBA_ERR_CUDA, "kba_track_create: out of memory"); }
    t->point_arena();
    t->m_off.assign(td.kf_cap, 0); t->m_cnt.assign(td.kf_cap, 0); t->kf_live.assign(td.kf_cap, 0);
    t->stamps.kf.assign(td.kf_cap, 0u); t->stamps.lm.assign(td.lm_cap, 0u);
    cudaStream_t s = h->stream;
    CU(cudaMemsetAsync(td.sel_index, 0xff, sizeof(int) * (size_t)td.lm_cap, s));
    CU(cudaMemsetAsync(td.m_cnt, 0, sizeof(int) * (size_t)td.kf_cap, s));
    CU(cudaMemsetAsync(td.lm_pos, 0, sizeof(double) * 3 * (size_t)td.lm_cap, s));  // a slot never written saves as 0
    CU(cudaMemsetAsync(td.lm_weight, 0, sizeof(double) * (size_t)td.lm_cap, s));
    CU(cudaStreamSynchronize(s));
    *out = t;
    return KBA_OK;
}

// the host side of the gather of tracks ts[0..n) into sv's batch, window i = ts[i]'s: what staging the requests leaves for the launch
struct StagedLists {
    TrackGrid grid;
    size_t used = 0;                       // ints of sv.lists in use (the options' included)
    int64_t h2d = 0;                       // bytes the upload moves, the options' excluded
    int max_rank = 0, max_free = 0;        // of the windows that do not sit out: rig rank, free reduced rows (track_free_rows)
    std::vector<WinShape> solved;          // rows and chunks of those windows (large-window path)
    bool any_gp = false;                   // some window has host ground-plane lists
};

// descriptors, selection lists (one pinned buffer) and track stores as they are now of requests qs[0..n), each checked by
// track_check or sitting out (sel == nullptr), into sv's staging
static void stage_requests(TrackSolver& sv, int n, kba_track* const* ts, const TrackRequest* qs, StagedLists& sl) {
    kba_batch* b = sv.batch;
    sl.solved.assign(n, WinShape{});
    sl.used = params_ints(n);
    sl.h2d = (int64_t)n * (int64_t)(sizeof(WinDesc) + sizeof(TrackDev) + sizeof(TrackSel));
    for (int i = 0; i < n; ++i) {
        const kba_track* t = ts[i];
        const TrackRequest& q = qs[i];
        WinDesc& d = b->desc_h[i];
        sv.tdev.h[i] = t->td;  // compaction re-points a track's arena: read at every solve
        if (!q.sel) {
            idle_desc(d);
            sv.tsel.h[i] = TrackSel{};
        } else {
            track_desc(d, t, q);
            sl.max_rank = std::max(sl.max_rank, d.max_rank);
            sl.max_free = std::max(sl.max_free, track_free_rows(q));
            sl.solved[i].rows = q.rows; sl.solved[i].n_chunks = d.n_chunks;
            // lists: keyframe slots | landmark slots | fixation bytes | ground-plane candidates
            // (a ranked request's landmarks and ground candidates are the track's ranking, already on the device)
            const kba_window* sel = q.sel;
            const int n_cand = q.device_gp ? sel->n_gp : 0, fixed_ints = (q.n_kf + 3) / 4;
            int* l = sv.lists.h + sl.used;
            const int* ld = sv.lists.d + sl.used;
            size_t at = (size_t)q.n_kf;
            memcpy(l, q.kf_slot, q.n_kf * sizeof(int));
            const int* lm_d = q.ranked ? ts[i]->rank->sel_slot : ld + at;
            if (!q.ranked) { memcpy(l + at, q.lm_slot, q.n_lm * sizeof(int)); at += (size_t)q.n_lm; }
            memcpy(l + at, q.kf_fixed, q.n_kf);
            const uint8_t* fx_d = reinterpret_cast<const uint8_t*>(ld + at);
            at += (size_t)fixed_ints;
            const int* cand_d = q.rank_gp ? ts[i]->rank->gp : ld + at;
            if (n_cand && !q.rank_gp) { memcpy(l + at, sel->gp_lm, n_cand * sizeof(int)); at += (size_t)n_cand; }
            sv.tsel.h[i] = track_sel(q, ld, fx_d, lm_d, cand_d);
            sl.used += at;
            if (sel->n_gp && !q.device_gp) {
                memcpy(b->r_gp_lm.h + d.gp_off, sel->gp_lm, sel->n_gp * sizeof(int)); memcpy(b->gp_kf.h + d.gp_off, sel->gp_kf, sel->n_gp * sizeof(int));
                memcpy(b->gp_weight.h + d.gp_off, sel->gp_weight, sel->n_gp * sizeof(double));
                sl.any_gp = true;
            }
            sl.grid.max_kf = std::max(sl.grid.max_kf, q.n_kf); sl.grid.max_lm = std::max(sl.grid.max_lm, q.n_lm);
            sl.grid.max_meas = std::max(sl.grid.max_meas, q.max_meas);
            sl.grid.any_cand |= n_cand > 0;
            sl.h2d += (int64_t)q.n_kf * 5 + (q.ranked ? 0 : (int64_t)q.n_lm * 4) +
                      (q.device_gp ? (q.rank_gp ? 0 : (int64_t)n_cand * 4) : (int64_t)sel->n_gp * 16);
        }
        b->desc.h[i] = d;
    }
}

// the staged requests up, then the gather of every window from its store.  The options go up in the lists' copy when they differ
// from what the device holds (a re-solve with the same ones: none).
static int upload_and_gather(kba_handle* h, TrackSolver& sv, bool per_track, const kba_options* opts, StagedLists& sl) {
    kba_batch* b = sv.batch;
    cudaStream_t s = h->stream;
    const size_t p_ints = params_ints(b->bd.n_win);
    const size_t from = stage_params(b, per_track, opts, reinterpret_cast<SolveParams*>(sv.lists.h)) ? 0 : p_ints;
    sl.h2d += (int64_t)((p_ints - from) * sizeof(int));
    CU(b->desc.upload(s));
    CU(cudaMemcpyAsync(sv.lists.d + from, sv.lists.h + from, (sl.used - from) * sizeof(int), cudaMemcpyHostToDevice, s));
    CU(sv.tdev.upload(s)); CU(sv.tsel.upload(s));
    if (sl.any_gp) { CU(b->r_gp_lm.upload(s)); CU(b->gp_kf.upload(s)); CU(b->gp_weight.upload(s)); }
    launch_track_gather(b->bd, b->raw, sv.tdev.d, sv.tsel.d, sl.grid, s);
    return KBA_OK;
}

// one solve of the stored windows of tracks ts[0..n) as one batch, window i = ts[i]'s; qs[i] is checked by track_check or sits
// the solve out (sel == nullptr).  kba_track_solve (n = 1) and kba_track_group_solve.
static int track_solve(kba_handle* h, TrackSolver& sv, int n, kba_track* const* ts, const TrackRequest* qs, bool per_track,
                       const kba_options* opts, const SolveTotals& tot, kba_result* res) {
    kba_batch* b = sv.batch;
    CU(cudaSetDevice(h->device));
    cudaStream_t s = h->stream;
    StagedLists sl;
    stage_requests(sv, n, ts, qs, sl);
    for (int i = 0; i < n; ++i)
        if (qs[i].sel) ts[i]->gen++;  // the solve writes the store back
    // one launch configuration for the whole batch, as kba_batch_solve has for any batch
    b->lc.max_rank = sl.max_rank;
    b->lc.plan.fused_slots = fused_slots(sl.max_free);
    if (!b->lc.plan.fused) {  // the buffers are sized for the largest values (batch_create, Purpose::TrackLarge)
        replan_large(b->lc.plan, sl.solved.data(), n, h->sm_count, b->lc.knobs);
        for (int i = 0; i < n; ++i) b->desc.h[i].nr_cap = b->desc_h[i].nr_cap = nr_cap_of(sl.solved[i].rows);
        apply_plan(b);
    }
    int rc = upload_and_gather(h, sv, per_track, opts, sl);
    if (rc != KBA_OK) return rc;
    sv.counts.h2d = sl.h2d;
    // ---- pack, solve, write back
    launch_pack(b->bd, b->raw, s);
    CU(cudaGetLastError());
    rc = batch_run(b, tot);
    if (rc != KBA_OK) return rc;
    launch_track_writeback(b->bd, sv.tdev.d, sv.tsel.d, sl.grid, s);
    rc = kba_batch_download(b, res);
    sv.counts.d2h = (int64_t)b->d2h_bytes;
    return rc;
}

// the checks of a solve of track t's ranking: q holds the caller's keyframe lists and window; it is pointed at the ranking and at
// q.ranked_sel, the caller's window with the ranking's ground-candidate count
static int ranked_check(kba_track* t, TrackRequest& q, std::string& why) {
    if (!q.kf_slot || !q.kf_fixed || !q.sel) { why = "null argument"; return KBA_ERR_BAD_ARG; }
    const RankBufs* rb = t->rank.get();
    if (!rb || !rb->valid) { why = "the track has no ranking to solve (kba_track_rank_landmarks)"; return KBA_ERR_BAD_ARG; }
    if (rb->gen != t->gen) { why = "the ranking is stale: the store changed after it was ranked"; return KBA_ERR_BAD_ARG; }
    if (q.n_kf != (int)rb->kf.size() || !std::equal(rb->kf.begin(), rb->kf.end(), q.kf_slot)) {
        why = "the keyframes differ from the ranking's"; return KBA_ERR_BAD_ARG;
    }
    const kba_window* sel = q.sel;
    q.ranked_sel = *sel;
    const bool from_ranking = sel->n_gp > 0 && !sel->gp_lm && !sel->gp_kf && !sel->gp_weight;
    if (from_ranking) q.ranked_sel.n_gp = rb->n_ground;
    q.n_lm = rb->n_sel; q.lm_slot = nullptr; q.sel = &q.ranked_sel;
    q.rank_gp = from_ranking && rb->n_ground > 0;
    return track_check(t, q, why);
}

static std::string track_prefix(bool group, int i) { return group ? "track " + std::to_string(i) + ": " : std::string(); }

// one solve of the windows of a track (group = false) or of a group, qs[i] track i's request.  Every request is checked in track
// order before anything is uploaded or launched; in a group, one with n_kf == 0 sits the solve out.  The solver is the one
// kba_batch_create would choose for the whole batch: the large-window path as soon as one window needs more than kFusedMaxRows
// reduced rows.
static int set_solve(TrackSet& s, bool group, const std::string& who, TrackRequest* qs, bool per_track, const kba_options* opts,
                     kba_result* res) {
    const int n = (int)s.tracks.size();
    bool any = false, large = false;
    SolveTotals tot;
    std::string owhy;
    const int orc = solve_options_check(n, opts, per_track, "track ", [&](int i) { return !(group && qs[i].n_kf == 0); }, tot, owhy);
    if (orc != KBA_OK) return fail(orc, who + owhy);
    for (int i = 0; i < n; ++i) {
        TrackRequest& q = qs[i];
        if (group && q.n_kf == 0) { q.sel = nullptr; continue; }  // sits this solve out
        std::string why;
        const int rc = q.ranked ? ranked_check(s.tracks[i], q, why) : track_check(s.tracks[i], q, why);
        if (rc != KBA_OK) return fail(rc, who + track_prefix(group, i) + why);
        any = true;
        large |= q.rows > kFusedMaxRows;
    }
    if (!any) {  // nothing to solve: no upload, no launch, every result idle
        for (int i = 0; i < n; ++i) idle_result(res[i]);
        s.last = &kNoTransfer;
        return KBA_OK;
    }
    TrackSolver& sv = large ? s.large : s.solver;
    s.last = &sv.counts;
    return track_solve(s.h, sv, n, s.tracks.data(), qs, per_track, opts, tot, res);
}

static TrackRequest track_request(int32_t n_kf, const int32_t* kf_slot, const uint8_t* kf_fixed, int32_t n_lm, const int32_t* lm_slot,
                                  const kba_window* sel, bool ranked) {
    TrackRequest q;
    q.n_kf = n_kf; q.kf_slot = kf_slot; q.kf_fixed = kf_fixed; q.n_lm = n_lm; q.lm_slot = lm_slot; q.sel = sel; q.ranked = ranked;
    return q;
}

int kba_track_solve(kba_track* t, int32_t n_kf, const int32_t* kf_slot, const uint8_t* kf_fixed, int32_t n_lm, const int32_t* lm_slot,
                    const kba_window* sel, const kba_options* opt, kba_result* res) {
    if (!t || !opt || !res) return fail(KBA_ERR_BAD_ARG, "null argument to kba_track_solve");
    TrackRequest q = track_request(n_kf, kf_slot, kf_fixed, n_lm, lm_slot, sel, false);
    return set_solve(t->set, false, "kba_track_solve: ", &q, false, opt, res);
}

int kba_track_transfer_bytes(kba_track* t, int64_t* h2d, int64_t* d2h, int64_t* push) {
    if (!t) return fail(KBA_ERR_BAD_ARG, "null track");
    if (h2d) *h2d = t->set.last->h2d;
    if (d2h) *d2h = t->set.last->d2h;
    if (push) *push = t->h2d_push;
    return KBA_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// several persistent windows solved in one batch (include/kba_b200.h, kba_track_group_*)
// ---------------------------------------------------------------------------------------------------------------------
void kba_track_group_destroy(kba_track_group* g) {
    if (!g) return;
    cudaStreamSynchronize(g->set.h->stream);
    delete g;
}

int kba_track_group_create(kba_handle* h, int32_t n_tracks, kba_track* const* tracks, kba_track_group** out) {
    if (!h || !tracks || !out || n_tracks < 1) return fail(KBA_ERR_BAD_ARG, "kba_track_group_create: empty group or null argument");
    for (int i = 0; i < n_tracks; ++i) {
        if (!tracks[i]) return fail(KBA_ERR_BAD_ARG, "kba_track_group_create: track " + std::to_string(i) + " is null");
        if (tracks[i]->set.h != h) return fail(KBA_ERR_BAD_ARG, "kba_track_group_create: track " + std::to_string(i) + " belongs to another handle");
        for (int j = 0; j < i; ++j)
            if (tracks[j] == tracks[i])
                return fail(KBA_ERR_BAD_ARG, "kba_track_group_create: track " + std::to_string(i) + " is also track " + std::to_string(j));
    }
    CU(cudaSetDevice(h->device));
    kba_track_group* g = new kba_track_group();
    g->set.h = h;
    g->set.tracks.assign(tracks, tracks + n_tracks);
    int rc = track_solver_create(h, n_tracks, tracks, false, g->set.solver, "kba_track_group_create");
    bool large = false;
    for (int i = 0; i < n_tracks; ++i) large |= has_large(tracks[i]->caps);
    if (rc == KBA_OK && large) rc = track_solver_create(h, n_tracks, tracks, true, g->set.large, "kba_track_group_create");
    if (rc != KBA_OK) { delete g; return rc; }
    *out = g;
    return KBA_OK;
}

static int group_solve(kba_track_group* g, const kba_track_request* req, bool per_track, const kba_options* opts, kba_result* res,
                       const std::string& who) {
    if (!g || !req || !opts || !res) return fail(KBA_ERR_BAD_ARG, "null argument to " + who.substr(0, who.size() - 2));
    std::vector<TrackRequest> qs;
    for (size_t i = 0; i < g->set.tracks.size(); ++i)
        qs.push_back(track_request(req[i].n_kf, req[i].kf_slot, req[i].kf_fixed, req[i].n_lm, req[i].lm_slot, req[i].sel, false));
    return set_solve(g->set, true, who, qs.data(), per_track, opts, res);
}
int kba_track_group_solve(kba_track_group* g, const kba_track_request* req, const kba_options* opt, kba_result* res) {
    return group_solve(g, req, false, opt, res, "kba_track_group_solve: ");
}
int kba_track_group_solve_opts(kba_track_group* g, const kba_track_request* req, const kba_options* opts, kba_result* res) {
    return group_solve(g, req, true, opts, res, "kba_track_group_solve_opts: ");
}

int kba_track_group_transfer_bytes(kba_track_group* g, int64_t* h2d, int64_t* d2h) {
    if (!g) return fail(KBA_ERR_BAD_ARG, "null track group");
    if (h2d) *h2d = g->set.last->h2d;
    if (d2h) *d2h = g->set.last->d2h;
    return KBA_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// evaluation of the stored windows at the store's state (include/kba_b200.h, kba_track_evaluate / kba_track_group_evaluate)
// ---------------------------------------------------------------------------------------------------------------------
static size_t al8(size_t b) { return (b + 7) & ~(size_t)7; }

// one call's output block: the windows' records, then each array for the call's totals (observation bounds TO, landmarks TL,
// ground-plane lists TG), back to back, 8-byte aligned
extern "C++" {  // templates have C++ linkage
struct EvalLayout {
    size_t head = 0, res = 0, rho = 0, trim = 0, gp_w = 0, gp_r = 0, obs_lm = 0, obs_kf = 0, obs_cam = 0, gp_lm = 0, gp_kf = 0, rej = 0, bytes = 0;
    EvalLayout(size_t W, size_t TO, size_t TL, size_t TG) {
        size_t at = 0;
        auto put = [&at](size_t& off, size_t b) { off = at; at += al8(b); };
        put(head, sizeof(EvalHead) * W);
        put(res, 24 * TO); put(rho, 16 * TO); put(trim, 16 * TL); put(gp_w, 8 * TG); put(gp_r, 8 * TG);
        put(obs_lm, 4 * TO); put(obs_kf, 4 * TO); put(obs_cam, 4 * TO); put(gp_lm, 4 * TG); put(gp_kf, 4 * TG); put(rej, 2 * TL);
        bytes = at;
    }
    template <typename T> T* at(unsigned char* base, size_t off) const { return reinterpret_cast<T*>(base + off); }
    EvalOut view(unsigned char* b, double* part) const {
        EvalOut o;
        o.head = at<EvalHead>(b, head); o.res = at<double>(b, res); o.rho = at<double>(b, rho); o.trim = at<double>(b, trim);
        o.gp_w = at<double>(b, gp_w); o.gp_r = at<double>(b, gp_r); o.obs_lm = at<int>(b, obs_lm); o.obs_kf = at<int>(b, obs_kf);
        o.obs_cam = at<int>(b, obs_cam); o.gp_lm = at<int>(b, gp_lm); o.gp_kf = at<int>(b, gp_kf); o.rej = at<unsigned char>(b, rej);
        o.part = part;
        return o;
    }
};
}  // extern "C++"

static int eval_stage(TrackSet& s, const std::string& who) {
    if (s.eval) return KBA_OK;
    size_t TO = 0, TL = 0, TG = 0, parts = 0;
    for (const kba_track* t : s.tracks) {
        TO += (size_t)t->caps.win_observations; TL += (size_t)t->caps.win_landmarks; TG += (size_t)t->caps.win_ground;
        parts += (size_t)(t->caps.win_landmarks + 63) / 64;
    }
    std::unique_ptr<EvalStage> e(new EvalStage());
    const size_t n = s.tracks.size();
    int bad = e->out.alloc(EvalLayout(n, TO, TL, TG).bytes, true) | e->wins.alloc(n, true);
    bad |= e->dev.alloc(&e->part, 3 * std::max<size_t>(parts, 1));
    if (bad) return fail(KBA_ERR_CUDA, who + "out of memory (evaluation staging)");
    s.eval = std::move(e);
    return KBA_OK;
}

static bool obs_arrays(const kba_evaluate_out& o) { return o.obs_lm || o.obs_kf || o.obs_cam || o.residual || o.rho; }

// one evaluation of the windows of a track (group = false) or of a group, qs[i] track i's request; the checks are a solve's (and
// FP64 only), in track order before anything is uploaded; in a group a request with n_kf == 0 sits the call out
static int set_evaluate(TrackSet& s, bool group, const std::string& who, TrackRequest* qs, bool per_track, const kba_options* opts,
                        kba_evaluate_out* out) {
    const int n = (int)s.tracks.size();
    auto live = [&](int i) { return !(group && qs[i].n_kf == 0); };
    SolveTotals tot;
    std::string owhy;
    const int orc = solve_options_check(n, opts, per_track, "track ", live, tot, owhy);
    if (orc != KBA_OK) return fail(orc, who + owhy);
    // FP64 only: per track, the entries of the tracks that are evaluated; one set, whenever some track is evaluated
    for (int i = 0; i < n; ++i) {
        if (!live(i)) continue;
        const int o = per_track ? i : 0;
        if (opts[o].precision != 0)
            return fail(KBA_ERR_BAD_ARG, who + (per_track ? track_prefix(true, i) : std::string()) + "kba_options.precision must be 0: evaluation is FP64 only");
        if (!per_track) break;
    }
    bool any = false, large = false;
    for (int i = 0; i < n; ++i) {
        TrackRequest& q = qs[i];
        if (!live(i)) { q.sel = nullptr; continue; }
        std::string why;
        int rc = track_check(s.tracks[i], q, why);
        if (rc == KBA_OK && obs_arrays(out[i]) && out[i].obs_capacity < 0) { why = "negative obs_capacity"; rc = KBA_ERR_BAD_ARG; }
        if (rc != KBA_OK) return fail(rc, who + track_prefix(group, i) + why);
        any = true;
        large |= q.rows > kFusedMaxRows;
    }
    if (!any) { s.last = &kNoTransfer; return KBA_OK; }
    kba_handle* h = s.h;
    CU(cudaSetDevice(h->device));
    int rc = eval_stage(s, who);
    if (rc != KBA_OK) return rc;
    EvalStage& e = *s.eval;
    TrackSolver& sv = large ? s.large : s.solver;
    cudaStream_t st = h->stream;
    // the windows' regions: observations bounded by the listed keyframes' measurements, the ground-plane lists by their request
    size_t TO = 0, TL = 0, TG = 0, parts = 0;
    int max_lm = 0;
    for (int i = 0; i < n; ++i) {
        const TrackRequest& q = qs[i];
        EvalWin& ew = e.wins.h[i];
        ew = EvalWin{};
        ew.obs0 = (int)TO; ew.lm0 = (int)TL; ew.gp0 = (int)TG; ew.part0 = (int)parts;
        if (!q.sel) continue;
        ew.n_part = (q.n_lm + 63) / 64;
        TO += (size_t)q.n_meas; TL += (size_t)q.n_lm; TG += (size_t)q.sel->n_gp; parts += (size_t)ew.n_part;
        max_lm = std::max(max_lm, q.n_lm);
    }
    for (int i = 0; i < n; ++i) e.wins.h[i].n_lm_total = (int)TL;
    const EvalLayout lay(n, TO, TL, TG);
    StagedLists sl;
    stage_requests(sv, n, s.tracks.data(), qs, sl);
    rc = upload_and_gather(h, sv, per_track, opts, sl);
    if (rc != KBA_OK) return rc;
    CU(e.wins.upload(st));
    launch_evaluate(sv.batch->bd, sv.batch->raw, e.wins.d, lay.view(e.out.d, e.part), max_lm, st);
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(e.out.h, e.out.d, lay.bytes, cudaMemcpyDeviceToHost, st));
    CU(wait_stream(h));
    e.counts.h2d = sl.h2d + (int64_t)(sizeof(EvalWin) * n);
    e.counts.d2h = (int64_t)lay.bytes;
    s.last = &e.counts;
    // the results: a short observation capacity fails the call after every n_obs is written
    const EvalOut o = lay.view(e.out.h, nullptr);
    int short_at = -1;
    for (int i = 0; i < n; ++i) {
        if (!qs[i].sel) continue;
        out[i].n_obs = o.head[i].n_obs;
        if (short_at < 0 && obs_arrays(out[i]) && o.head[i].n_obs > out[i].obs_capacity) short_at = i;
    }
    if (short_at >= 0)
        return fail(KBA_ERR_CAPACITY, who + track_prefix(group, short_at) + "the window has " + std::to_string(o.head[short_at].n_obs) +
                                          " observations, more than obs_capacity = " + std::to_string(out[short_at].obs_capacity));
    for (int i = 0; i < n; ++i) {
        if (!qs[i].sel) continue;
        const EvalWin& ew = e.wins.h[i];
        const EvalHead& hd = o.head[i];
        kba_evaluate_out& r = out[i];
        const size_t no = (size_t)hd.n_obs, nl = (size_t)qs[i].n_lm, ng = (size_t)hd.n_gp;
        r.n_gp = hd.n_gp; r.failed = hd.failed;
        memcpy(r.cost, hd.cost, sizeof r.cost);
        if (r.obs_lm) memcpy(r.obs_lm, o.obs_lm + ew.obs0, 4 * no);
        if (r.obs_kf) memcpy(r.obs_kf, o.obs_kf + ew.obs0, 4 * no);
        if (r.obs_cam) memcpy(r.obs_cam, o.obs_cam + ew.obs0, 4 * no);
        if (r.residual) memcpy(r.residual, o.res + 3 * (size_t)ew.obs0, 24 * no);
        if (r.rho) memcpy(r.rho, o.rho + 2 * (size_t)ew.obs0, 16 * no);
        if (r.trim_repr) memcpy(r.trim_repr, o.trim + ew.lm0, 8 * nl);
        if (r.trim_depth) memcpy(r.trim_depth, o.trim + TL + ew.lm0, 8 * nl);
        if (r.rejected_repr) memcpy(r.rejected_repr, o.rej + ew.lm0, nl);
        if (r.rejected_depth) memcpy(r.rejected_depth, o.rej + TL + ew.lm0, nl);
        if (r.gp_lm) memcpy(r.gp_lm, o.gp_lm + ew.gp0, 4 * ng);
        if (r.gp_kf) memcpy(r.gp_kf, o.gp_kf + ew.gp0, 4 * ng);
        if (r.gp_weight) memcpy(r.gp_weight, o.gp_w + ew.gp0, 8 * ng);
        if (r.gp_residual) memcpy(r.gp_residual, o.gp_r + ew.gp0, 8 * ng);
    }
    return KBA_OK;
}

int kba_track_evaluate(kba_track* t, const kba_track_request* req, const kba_options* opt, kba_evaluate_out* out) {
    if (!t || !req || !opt || !out) return fail(KBA_ERR_BAD_ARG, "null argument to kba_track_evaluate");
    TrackRequest q = track_request(req->n_kf, req->kf_slot, req->kf_fixed, req->n_lm, req->lm_slot, req->sel, false);
    return set_evaluate(t->set, false, "kba_track_evaluate: ", &q, false, opt, out);
}

static int group_evaluate(kba_track_group* g, const kba_track_request* req, bool per_track, const kba_options* opts, kba_evaluate_out* out,
                          const std::string& who) {
    if (!g || !req || !opts || !out) return fail(KBA_ERR_BAD_ARG, "null argument to " + who.substr(0, who.size() - 2));
    std::vector<TrackRequest> qs;
    for (size_t i = 0; i < g->set.tracks.size(); ++i)
        qs.push_back(track_request(req[i].n_kf, req[i].kf_slot, req[i].kf_fixed, req[i].n_lm, req[i].lm_slot, req[i].sel, false));
    return set_evaluate(g->set, true, who, qs.data(), per_track, opts, out);
}
int kba_track_group_evaluate(kba_track_group* g, const kba_track_request* req, const kba_options* opt, kba_evaluate_out* out) {
    return group_evaluate(g, req, false, opt, out, "kba_track_group_evaluate: ");
}
int kba_track_group_evaluate_opts(kba_track_group* g, const kba_track_request* req, const kba_options* opts, kba_evaluate_out* out) {
    return group_evaluate(g, req, true, opts, out, "kba_track_group_evaluate_opts: ");
}

// ---------------------------------------------------------------------------------------------------------------------
// store calls of a track and of a group (landmark selection, creation, upkeep, frame flow, reclaim, ranking): one driver, which a
// single call runs with the track's one-track set
// ---------------------------------------------------------------------------------------------------------------------
// the slot lists of one request of track t, checked with a fresh stamp of its duplicate checks: keyframes pushed, landmarks in
// range, no slot listed twice.  max_meas: arena entries of the largest listed keyframe.
static int check_slot_lists(kba_track* t, int n_kf, const int32_t* kf_slot, int n_lm, const int32_t* lm_slot, int& max_meas,
                            std::string& why) {
    SlotStamps& st = t->stamps;
    st.next();
    max_meas = 0;
    for (int k = 0; k < n_kf; ++k) {
        const int s = kf_slot[k];
        if (s < 0 || s >= t->td.kf_cap || !t->kf_live[s]) { why = "keyframe slot not pushed"; return KBA_ERR_BAD_ARG; }
        if (st.kf[s] == st.cur) { why = "keyframe slot listed twice"; return KBA_ERR_BAD_ARG; }
        st.kf[s] = st.cur;
        max_meas = std::max(max_meas, t->m_cnt[s]);
    }
    for (int j = 0; j < n_lm; ++j) {
        const int s = lm_slot[j];
        if (s < 0 || s >= t->td.lm_cap) { why = "landmark slot out of range"; return KBA_ERR_BAD_ARG; }
        if (st.lm[s] == st.cur) { why = "landmark slot listed twice"; return KBA_ERR_BAD_ARG; }
        st.lm[s] = st.cur;
    }
    return KBA_OK;
}

// One store call of the tracks of s (group = false: a single call), req[i] / out[i] track i's.  C describes the call:
//   Request, Out         its public request and output types; Req the checked request of one window
//   slot, staging        its staging in s.stage and the staging's name in errors
//   sits_out(q)          a group's request that sits the call out: not checked, except what sit_out_check reads; a single
//                        request is checked, and then does not run (a reclaim of an empty range: the other checks refuse it)
//   sat_out(o, group)    what a request that sat out writes once the call succeeded
//                        (the store writes have no outputs: out is null, and neither is called)
//   make, check          the request of one window, and every check of it before anything is uploaded
//   capacity(n, ts, ..)  the staging's upload and download bytes for tracks ts[0..n) at their capacities (n = 1: a single call's)
//   run                  the requests that do not sit out as the windows of one launch sequence; a failure of request w it
//                        reports as (bad = w, why)
// Requests are checked in track order, and the first failure, named after its track in a group, returns before anything is
// uploaded or written.  A call in which nothing runs reports no transfers.
extern "C++" {  // templates have C++ linkage
template <class C>
static int store_call(TrackSet& s, bool group, const std::string& who, const typename C::Request* req, typename C::Out* out) {
    const int n = (int)s.tracks.size();
    std::vector<typename C::Req> rs;
    std::vector<int> track_of;             // rs[w] is the request of track track_of[w]
    for (int i = 0; i < n; ++i) {
        const bool sits_out = C::sits_out(req[i]);
        std::string why;
        int rc;
        typename C::Req r;
        if (group && sits_out) {
            rc = out ? C::sit_out_check(out[i], why) : KBA_OK;
        } else {
            r = C::make(s.tracks[i], req[i], out ? out + i : nullptr);
            rc = C::check(r, why);
        }
        if (rc != KBA_OK) return fail(rc, who + track_prefix(group, i) + why);
        if (!sits_out) { rs.push_back(r); track_of.push_back(i); }
    }
    if (rs.empty()) {  // no upload, no launch
        s.last = &kNoTransfer;
    } else {
        std::unique_ptr<StoreStage>& st = s.stage[C::slot];
        if (!st) {
            size_t up = 0, down = 0;
            C::capacity(n, s.tracks.data(), up, down);
            std::unique_ptr<StoreStage> fresh(new StoreStage());
            if (fresh->alloc(up, down)) return fail(KBA_ERR_CUDA, who + "out of memory for the " + C::staging + " staging");
            st = std::move(fresh);
        }
        int bad = -1;
        std::string why;
        const int rc = C::run(s.h, *st, (int)rs.size(), rs.data(), bad, why);
        if (rc != KBA_OK) return bad < 0 ? rc : fail(rc, who + track_prefix(group, track_of[bad]) + why);
        s.last = &st->counts;
    }
    for (int i = 0; i < n && out; ++i)
        if (C::sits_out(req[i])) C::sat_out(out + i, group);
    return KBA_OK;
}
}  // extern "C++"

// ---------------------------------------------------------------------------------------------------------------------
// landmark selection on the stored window (include/kba_b200.h, kba_track_select_landmarks / kba_track_group_select_landmarks;
// kernels in kba_select.cu): a single call is a one-window call of select_run, as a group's requests are
// ---------------------------------------------------------------------------------------------------------------------
// download of a call: 18 bytes per candidate (flow, seen, near order, cheirality, bin) and 16 per window (its counters)
static size_t select_out_bytes(size_t cands, size_t windows) { return 18 * cands + 16 * windows; }

static int select_alloc(kba_track* t, std::string& why) {
    std::unique_ptr<SelectBufs> sb(new SelectBufs());
    const TrackDev& td = t->td;
    const size_t L = (size_t)td.lm_cap, K = (size_t)td.kf_cap;
    SelectArgs& a = sb->a;
    double* cams = nullptr;
    int bad = 0;
    DevAllocs& dev = sb->dev;
    bad |= dev.alloc(&a.cand_of, L); bad |= dev.alloc(&a.kf_T, 12 * K); bad |= dev.alloc(&a.cam_T, 12 * (size_t)kMaxCam);
    bad |= dev.alloc(&a.path, 3 * K); bad |= dev.alloc(&a.pt, 3 * L); bad |= dev.alloc(&a.cnt, L); bad |= dev.alloc(&a.cursor, L);
    bad |= dev.alloc(&a.obs_off, L); bad |= dev.alloc(&a.in_list, L); bad |= dev.alloc(&a.vkey, L); bad |= dev.alloc(&a.sorted, L);
    bad |= dev.alloc(&a.near_flag, L); bad |= dev.alloc(&a.okey, (size_t)td.m_cap); bad |= dev.alloc(&a.bounds, 6);
    bad |= dev.alloc(&cams, 7 * (size_t)t->n_cam);
    if (bad) { why = "out of memory for the selection buffers"; return KBA_ERR_CUDA; }
    cudaStream_t s = t->set.h->stream;
    cudaError_t e = cudaMemsetAsync(a.cand_of, 0xff, sizeof(int) * L, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(cams, t->cam_pose.data(), sizeof(double) * 7 * (size_t)t->n_cam, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) { why = std::string("selection buffers: ") + cudaGetErrorString(e); return KBA_ERR_CUDA; }
    a.cam_pose7 = cams; a.n_cam = t->n_cam;
    t->select = std::move(sb);
    return KBA_OK;
}

// one selection request of track t (one window of select_run)
struct SelectReq {
    kba_track* t = nullptr;
    int n_kf = 0, n_cand = 0;
    const int* kf_slot = nullptr;
    const int* lm_slot = nullptr;
    const kba_select_params* p = nullptr;
    const kba_select_out* o = nullptr;
    int max_meas = 0;                      // set by select_check: arena entries of the largest listed keyframe
    bool quantities_only = false;          // a ranking's selection: the quantities stay on the device, `o` is not used
};

// every check of one request, before anything is uploaded; allocates the track's selection buffers at its first selection
static int select_check(SelectReq& r, std::string& why) {
    kba_track* t = r.t;
    const kba_select_out* o = r.o;
    if (!r.kf_slot || !r.p || (r.n_cand > 0 && !r.lm_slot) ||
        (!r.quantities_only && (!o || !o->cheiral || !o->bin || !o->near_order || !o->n_near || !o->flow || !o->seen))) {
        why = "null argument"; return KBA_ERR_BAD_ARG;
    }
    if (r.n_kf < 1 || r.n_cand < 0) { why = "no keyframes or a negative size"; return KBA_ERR_BAD_ARG; }
    if (r.n_kf > t->td.kf_cap || r.n_cand > t->td.lm_cap) { why = "more keyframes or candidates than the track's slots"; return KBA_ERR_CAPACITY; }
    for (int q = 0; q < 3; ++q)
        if (!(r.p->voxel_size[q] > 0.0) || !std::isfinite(r.p->voxel_size[q])) { why = "voxel sizes must be finite and positive"; return KBA_ERR_BAD_ARG; }
    const cudaError_t e = cudaSetDevice(t->set.h->device);
    if (e != cudaSuccess) { why = std::string("cudaSetDevice: ") + cudaGetErrorString(e); return KBA_ERR_CUDA; }
    if (!t->select) { const int rc = select_alloc(t, why); if (rc != KBA_OK) return rc; }
    return check_slot_lists(t, r.n_kf, r.kf_slot, r.n_cand, r.lm_slot, r.max_meas, why);
}

// W checked requests of distinct tracks as the W windows of one launch sequence: one upload (the argument records of windows
// 1 .. W-1, then every window's lists), one download (the outputs of all windows), one synchronisation, then the scatter into the
// callers' arrays.  Window 0's record travels in the launch parameters (kba_select.cu).
static int select_run(kba_handle* h, StoreStage& st, int W, const SelectReq* r) {
    CU(cudaSetDevice(h->device));
    cudaStream_t s = h->stream;
    SelectGrid g;
    size_t n_list = 0, N = 0;
    for (int w = 0; w < W; ++w) {
        const SelectReq& q = r[w];
        n_list += (size_t)q.n_kf + q.n_cand; N += (size_t)q.n_cand;
        g.max_kf = std::max(g.max_kf, q.n_kf); g.max_cand = std::max(g.max_cand, q.n_cand);
        g.max_init = std::max(g.max_init, std::max(std::max(q.n_kf, q.n_cand), q.t->n_cam));
        g.max_meas = std::max(g.max_meas, q.max_meas);
    }
    // ---- staging: records | lists up; flow | seen | near order (by candidate of all windows) | counters (by window) | cheirality | bins down
    const size_t o_lists = sizeof(SelectArgs) * (size_t)(W - 1), up_bytes = o_lists + 4 * n_list;
    const size_t o_seen = 8 * N, o_near = o_seen + 4 * N, o_cnt = o_near + 4 * N, o_ch = o_cnt + 16 * (size_t)W, o_bin = o_ch + N;
    const size_t out_bytes = o_bin + N;
    int* lists_h = reinterpret_cast<int*>(st.up.h + o_lists);
    const int* lists_d = reinterpret_cast<const int*>(st.up.d + o_lists);
    unsigned char* d = st.out.d;
    SelectLaunch l;
    l.rest = reinterpret_cast<const SelectArgs*>(st.up.d);
    l.n_win = W;
    size_t li = 0, c0 = 0;
    for (int w = 0; w < W; ++w) {
        const SelectReq& q = r[w];
        memcpy(lists_h + li, q.kf_slot, 4 * (size_t)q.n_kf);
        if (q.n_cand) memcpy(lists_h + li + q.n_kf, q.lm_slot, 4 * (size_t)q.n_cand);
        SelectArgs a = q.t->select->a;
        a.td = q.t->td;
        a.kf_slot = lists_d + li; a.lm_slot = lists_d + li + q.n_kf; a.n_kf = q.n_kf; a.n_cand = q.n_cand;
        for (int k = 0; k < 3; ++k) a.leaf[k] = q.p->voxel_size[k];
        a.roi_far = q.p->roi_far; a.roi_middle = q.p->roi_middle;
        a.flow = reinterpret_cast<double*>(d + 8 * c0); a.seen = reinterpret_cast<int*>(d + o_seen + 4 * c0);
        a.near_order = reinterpret_cast<int*>(d + o_near + 4 * c0);
        a.counters = reinterpret_cast<int*>(d + o_cnt + 16 * (size_t)w); a.n_near = a.counters + 1;
        a.cheiral = d + o_ch + c0; a.bin = reinterpret_cast<signed char*>(d + o_bin + c0);
        if (w == 0) l.w0 = a;
        else memcpy(st.up.h + sizeof(SelectArgs) * (size_t)(w - 1), &a, sizeof(SelectArgs));
        li += (size_t)q.n_kf + q.n_cand; c0 += (size_t)q.n_cand;
    }
    // ---- one upload, one launch sequence, one download, one synchronisation
    CU(cudaMemcpyAsync(st.up.d, st.up.h, up_bytes, cudaMemcpyHostToDevice, s));
    launch_select(l, g, s);
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(st.out.h, st.out.d, out_bytes, cudaMemcpyDeviceToHost, s));
    CU(wait_stream(h));
    // ---- scatter
    const unsigned char* hb = st.out.h;
    c0 = 0;
    for (int w = 0; w < W; ++w) {
        const kba_select_out* o = r[w].o;
        const size_t n = (size_t)r[w].n_cand;
        memcpy(o->flow, hb + 8 * c0, 8 * n); memcpy(o->seen, hb + o_seen + 4 * c0, 4 * n); memcpy(o->near_order, hb + o_near + 4 * c0, 4 * n);
        memcpy(o->n_near, hb + o_cnt + 16 * (size_t)w + 4, 4);
        memcpy(o->cheiral, hb + o_ch + c0, n); memcpy(o->bin, hb + o_bin + c0, n);
        c0 += n;
    }
    st.counts.h2d = (int64_t)up_bytes;
    st.counts.d2h = (int64_t)out_bytes;
    return KBA_OK;
}

struct Select {
    using Request = kba_select_request;
    using Out = kba_select_out;
    using Req = SelectReq;
    static constexpr StoreCall slot = kSelectCall;
    static constexpr const char* staging = "selection";
    static bool sits_out(const Request& q) { return q.n_kf == 0; }
    static int sit_out_check(const Out& o, std::string& why) {  // the request's n_near is written
        if (o.n_near) return KBA_OK;
        why = "null argument"; return KBA_ERR_BAD_ARG;
    }
    static void sat_out(Out* o, bool) { *o->n_near = 0; }
    static Req make(kba_track* t, const Request& q, Out* o) {
        Req r;
        r.t = t; r.n_kf = q.n_kf; r.n_cand = q.n_cand; r.kf_slot = q.kf_slot; r.lm_slot = q.lm_slot; r.p = q.params; r.o = o;
        return r;
    }
    static int check(Req& r, std::string& why) { return select_check(r, why); }
    static void capacity(int n, kba_track* const* ts, size_t& up, size_t& down) {
        size_t lists = 0, cands = 0;
        for (int i = 0; i < n; ++i) { lists += (size_t)ts[i]->td.kf_cap + ts[i]->td.lm_cap; cands += (size_t)ts[i]->td.lm_cap; }
        up = sizeof(SelectArgs) * (size_t)(n - 1) + 4 * lists;
        down = select_out_bytes(cands, (size_t)n);
    }
    static int run(kba_handle* h, StoreStage& st, int W, Req* r, int&, std::string&) { return select_run(h, st, W, r); }
};

int kba_track_select_landmarks(kba_track* t, int32_t n_kf, const int32_t* kf_slot, int32_t n_cand, const int32_t* lm_slot,
                               const kba_select_params* p, kba_select_out* o) {
    static const std::string who = "kba_track_select_landmarks: ";
    if (!t) return fail(KBA_ERR_BAD_ARG, who + "null argument");
    const kba_select_request q = {n_kf, n_cand, kf_slot, lm_slot, p};
    return store_call<Select>(t->set, false, who, &q, o);
}

int kba_track_group_select_landmarks(kba_track_group* g, const kba_select_request* req, kba_select_out* out) {
    static const std::string who = "kba_track_group_select_landmarks: ";
    if (!g || !req || !out) return fail(KBA_ERR_BAD_ARG, who + "null argument");
    return store_call<Select>(g->set, true, who, req, out);
}

// ---------------------------------------------------------------------------------------------------------------------
// landmark creation of push() on the stored window (include/kba_b200.h, kba_track_create_landmarks /
// kba_track_group_create_landmarks; kernels in kba_create.cu): a single call is a one-window call of create_run
// ---------------------------------------------------------------------------------------------------------------------
static int create_alloc(kba_track* t, std::string& why) {
    std::unique_ptr<CreateBufs> cb(new CreateBufs());
    const TrackDev& td = t->td;
    const size_t L = (size_t)td.lm_cap, K = (size_t)td.kf_cap, NC = (size_t)t->n_cam;
    CreateArgs& a = cb->a;
    double* intr = nullptr, *pose = nullptr;
    int bad = 0;
    DevAllocs& dev = cb->dev;
    bad |= dev.alloc(&a.req_of, L); bad |= dev.alloc(&a.ray_T, 12 * K * NC); bad |= dev.alloc(&a.intr_inv, 9 * NC);
    bad |= dev.alloc(&a.cnt, L); bad |= dev.alloc(&a.cursor, L); bad |= dev.alloc(&a.off, L); bad |= dev.alloc(&a.key, (size_t)td.m_cap);
    bad |= dev.alloc(&a.total, 1); bad |= dev.alloc(&intr, 3 * NC); bad |= dev.alloc(&pose, 7 * NC);
    if (bad) { why = "out of memory for the creation buffers"; return KBA_ERR_CUDA; }
    cudaStream_t s = t->set.h->stream;
    cudaError_t e = cudaMemsetAsync(a.req_of, 0xff, sizeof(int) * L, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(intr, t->cam_intr.data(), sizeof(double) * 3 * NC, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(pose, t->cam_pose.data(), sizeof(double) * 7 * NC, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) { why = std::string("creation buffers: ") + cudaGetErrorString(e); return KBA_ERR_CUDA; }
    a.cam_intr = intr; a.cam_pose7 = pose; a.n_cam = t->n_cam;
    t->create = std::move(cb);
    return KBA_OK;
}

// one creation request of track t (one window of create_run)
struct CreateReq {
    kba_track* t = nullptr;
    const kba_create_request* q = nullptr;
    kba_create_out* o = nullptr;
    int max_meas = 0;                      // set by create_check: arena entries of the largest listed keyframe
};

// every check of one request, before anything is uploaded; allocates the track's creation buffers at its first creation
static int create_check(CreateReq& r, std::string& why) {
    kba_track* t = r.t;
    const kba_create_request& q = *r.q;
    if (!q.kf_slot || (q.n_new > 0 && (!q.lm_slot || !r.o->pos || !r.o->flags))) { why = "null argument"; return KBA_ERR_BAD_ARG; }
    if (q.n_kf < 1 || q.n_new < 0) { why = "no keyframes or a negative size"; return KBA_ERR_BAD_ARG; }
    if (q.n_kf > t->td.kf_cap || q.n_new > t->td.lm_cap) { why = "more keyframes or landmarks than the track's slots"; return KBA_ERR_CAPACITY; }
    if (q.kf_new < 0 || q.kf_new >= q.n_kf) { why = "kf_new outside [0, n_kf)"; return KBA_ERR_BAD_ARG; }
    const cudaError_t e = cudaSetDevice(t->set.h->device);
    if (e != cudaSuccess) { why = std::string("cudaSetDevice: ") + cudaGetErrorString(e); return KBA_ERR_CUDA; }
    if (!t->create) { const int rc = create_alloc(t, why); if (rc != KBA_OK) return rc; }
    return check_slot_lists(t, q.n_kf, q.kf_slot, q.n_new, q.lm_slot, r.max_meas, why);
}

// W checked requests of distinct tracks as the W windows of one launch sequence: one upload (the argument records of windows
// 1 .. W-1, then every window's lists), one download (positions of all windows | their flags), one synchronisation, then the
// scatter into the callers' arrays.  Window 0's record travels in the launch parameters (kba_create.cu).
static int create_run(kba_handle* h, StoreStage& st, int W, const CreateReq* r) {
    CU(cudaSetDevice(h->device));
    for (int w = 0; w < W; ++w) r[w].t->gen++;
    cudaStream_t s = h->stream;
    CreateGrid g;
    size_t n_list = 0, N = 0;
    for (int w = 0; w < W; ++w) {
        const kba_create_request& q = *r[w].q;
        n_list += (size_t)q.n_kf + q.n_new; N += (size_t)q.n_new;
        g.max_kf = std::max(g.max_kf, q.n_kf); g.max_new = std::max(g.max_new, q.n_new);
        g.max_init = std::max(g.max_init, std::max(q.n_new, q.n_kf * r[w].t->n_cam));
        g.max_meas = std::max(g.max_meas, r[w].max_meas);
    }
    const size_t o_lists = sizeof(CreateArgs) * (size_t)(W - 1), up_bytes = o_lists + 4 * n_list;
    const size_t o_flags = 24 * N, out_bytes = o_flags + N;
    int* lists_h = reinterpret_cast<int*>(st.up.h + o_lists);
    const int* lists_d = reinterpret_cast<const int*>(st.up.d + o_lists);
    unsigned char* d = st.out.d;
    CreateLaunch l;
    l.rest = reinterpret_cast<const CreateArgs*>(st.up.d);
    l.n_win = W;
    size_t li = 0, c0 = 0;
    for (int w = 0; w < W; ++w) {
        const kba_create_request& q = *r[w].q;
        memcpy(lists_h + li, q.kf_slot, 4 * (size_t)q.n_kf);
        if (q.n_new) memcpy(lists_h + li + q.n_kf, q.lm_slot, 4 * (size_t)q.n_new);
        CreateArgs a = r[w].t->create->a;
        a.td = r[w].t->td;
        a.kf_slot = lists_d + li; a.lm_slot = lists_d + li + q.n_kf;
        a.n_kf = q.n_kf; a.kf_new = q.kf_new; a.n_new = q.n_new;
        a.pos = reinterpret_cast<double*>(d + 24 * c0); a.flags = d + o_flags + c0;
        if (w == 0) l.w0 = a;
        else memcpy(st.up.h + sizeof(CreateArgs) * (size_t)(w - 1), &a, sizeof(CreateArgs));
        li += (size_t)q.n_kf + q.n_new; c0 += (size_t)q.n_new;
    }
    CU(cudaMemcpyAsync(st.up.d, st.up.h, up_bytes, cudaMemcpyHostToDevice, s));
    launch_create(l, g, s);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpyAsync(st.out.h, st.out.d, out_bytes, cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = wait_stream(h);
    if (e != cudaSuccess) {
        // k_cr_init fills each window's slot -> request map and only k_cr_land clears it: after a failed launch sequence the maps
        // are cleared here, so that no later call reads this call's request indices (a sticky error leaves the context unusable
        // anyway, and these calls then fail as well)
        for (int w = 0; w < W; ++w) cudaMemsetAsync(r[w].t->create->a.req_of, 0xff, sizeof(int) * (size_t)r[w].t->td.lm_cap, s);
        cudaStreamSynchronize(s);
        return fail(KBA_ERR_CUDA, std::string("landmark creation: ") + cudaGetErrorString(e));
    }
    const unsigned char* hb = st.out.h;
    c0 = 0;
    for (int w = 0; w < W; ++w) {
        const size_t n = (size_t)r[w].q->n_new;
        if (n) { memcpy(r[w].o->pos, hb + 24 * c0, 24 * n); memcpy(r[w].o->flags, hb + o_flags + c0, n); }
        c0 += n;
    }
    st.counts.h2d = (int64_t)up_bytes;
    st.counts.d2h = (int64_t)out_bytes;
    return KBA_OK;
}

struct Create {
    using Request = kba_create_request;
    using Out = kba_create_out;
    using Req = CreateReq;
    static constexpr StoreCall slot = kCreateCall;
    static constexpr const char* staging = "creation";
    static bool sits_out(const Request& q) { return q.n_kf == 0; }
    static int sit_out_check(const Out&, std::string&) { return KBA_OK; }
    static void sat_out(Out*, bool) {}
    static Req make(kba_track* t, const Request& q, Out* o) {
        Req r;
        r.t = t; r.q = &q; r.o = o;
        return r;
    }
    static int check(Req& r, std::string& why) { return create_check(r, why); }
    static void capacity(int n, kba_track* const* ts, size_t& up, size_t& down) {
        size_t lists = 0, lms = 0;
        for (int i = 0; i < n; ++i) { lists += (size_t)ts[i]->td.kf_cap + ts[i]->td.lm_cap; lms += (size_t)ts[i]->td.lm_cap; }
        up = sizeof(CreateArgs) * (size_t)(n - 1) + 4 * lists;
        down = 25 * lms;
    }
    static int run(kba_handle* h, StoreStage& st, int W, Req* r, int&, std::string&) { return create_run(h, st, W, r); }
};

int kba_track_create_landmarks(kba_track* t, const kba_create_request* req, kba_create_out* out) {
    static const std::string who = "kba_track_create_landmarks: ";
    if (!t || !req || !out) return fail(KBA_ERR_BAD_ARG, who + "null argument");
    return store_call<Create>(t->set, false, who, req, out);
}

int kba_track_group_create_landmarks(kba_track_group* g, const kba_create_request* req, kba_create_out* out) {
    static const std::string who = "kba_track_group_create_landmarks: ";
    if (!g || !req || !out) return fail(KBA_ERR_BAD_ARG, who + "null argument");
    return store_call<Create>(g->set, true, who, req, out);
}

// ---------------------------------------------------------------------------------------------------------------------
// window upkeep on the stored window (include/kba_b200.h, kba_track_deactivate_keyframes / kba_track_depth_costs and their group
// forms; kernels in kba_upkeep.cu): a single call is a one-window call of upkeep_run
// ---------------------------------------------------------------------------------------------------------------------
// the largest download of one window of track t: deactivation 5 * n_kf + n_lm, depth costs 4 * n_kf + 12 * B with B <= m_cap
static size_t upkeep_out_cap(const kba_track* t) {
    const size_t K = (size_t)t->td.kf_cap, L = (size_t)t->td.lm_cap, M = (size_t)t->td.m_cap;
    return std::max(5 * K + L, 4 * K + 12 * M);
}

// one upkeep request of track t (one window of upkeep_run), either kind
struct UpkeepReq {
    kba_track* t = nullptr;
    int n_kf = 0, n_lm = 0;
    const int32_t* kf_slot = nullptr, *lm_slot = nullptr;
    const kba_deactivate_request* dq = nullptr;  // deactivation
    kba_deactivate_out* dout = nullptr;
    kba_depth_out* cout = nullptr;                // depth costs
    int cap = 0;
    int bound = 0, max_meas = 0;                  // set by upkeep_check: the depth costs' B, arena entries of the largest keyframe
};

// the track's upkeep scratch (the slot map), allocated at its first upkeep, flow or reclaim call
static int upkeep_bufs(kba_track* t, std::string& why) {
    const cudaError_t e = cudaSetDevice(t->set.h->device);
    if (e != cudaSuccess) { why = std::string("cudaSetDevice: ") + cudaGetErrorString(e); return KBA_ERR_CUDA; }
    if (!t->upkeep) {
        std::unique_ptr<UpkeepBufs> ub(new UpkeepBufs());
        const size_t L = (size_t)t->td.lm_cap, C = (L + kReclaimChunk - 1) / kReclaimChunk;
        if (ub->dev.alloc(&ub->map, L) | ub->dev.alloc(&ub->blk, C)) { why = "out of memory for the upkeep buffers"; return KBA_ERR_CUDA; }
        cudaError_t me = cudaMemsetAsync(ub->map, 0, sizeof(unsigned long long) * L, t->set.h->stream);
        if (me == cudaSuccess) me = cudaStreamSynchronize(t->set.h->stream);
        if (me != cudaSuccess) { why = std::string("upkeep buffers: ") + cudaGetErrorString(me); return KBA_ERR_CUDA; }
        t->upkeep = std::move(ub);
    }
    return KBA_OK;
}

// every check of one request, before anything is uploaded; allocates the track's slot map at its first upkeep call
static int upkeep_check(UpkeepReq& r, std::string& why) {
    kba_track* t = r.t;
    const bool depth = r.cout != nullptr;
    if (!r.kf_slot || (r.n_lm > 0 && !r.lm_slot)) { why = "null argument"; return KBA_ERR_BAD_ARG; }
    if (depth ? (!r.cout->off || (r.cap > 0 && (!r.cout->cand || !r.cout->cost)))
              : (!r.dout->kf_active || !r.dout->kf_common || (r.n_lm > 0 && !r.dout->lm_active))) {
        why = "null argument"; return KBA_ERR_BAD_ARG;
    }
    if (r.n_kf < 1 || r.n_lm < 0 || r.cap < 0) { why = "no keyframes or a negative size"; return KBA_ERR_BAD_ARG; }
    if (r.n_kf > t->td.kf_cap || r.n_lm > t->td.lm_cap) { why = "more keyframes or landmarks than the track's slots"; return KBA_ERR_CAPACITY; }
    int rc = upkeep_bufs(t, why);
    if (rc == KBA_OK) rc = check_slot_lists(t, r.n_kf, r.kf_slot, r.n_lm, r.lm_slot, r.max_meas, why);
    if (rc != KBA_OK) return rc;
    int64_t bound = 0;
    for (int k = 0; k < r.n_kf; ++k) bound += std::min(r.n_lm, t->m_cnt[r.kf_slot[k]]);
    r.bound = (int)bound;  // <= the arena entries of distinct keyframes <= m_cap
    if (depth && r.cap < r.bound) { why = "cap below the sum over keyframes of min(n_elig, arena entries)"; return KBA_ERR_CAPACITY; }
    return KBA_OK;
}

// W checked requests of distinct tracks, all of one kind, as the W windows of one launch sequence: one upload (the argument
// records of windows 1 .. W-1, then every window's lists), one download, one synchronisation, then the scatter into the callers'
// arrays.  Downloads: deactivation kf_common of all windows | kf_active | lm_active; depth costs cost | cnt | cand, each window's
// pairs at its keyframes' bounds.  Window 0's record travels in the launch parameters (kba_upkeep.cu).
static int upkeep_run(kba_handle* h, StoreStage& st, int W, const UpkeepReq* r, bool depth) {
    CU(cudaSetDevice(h->device));
    cudaStream_t s = h->stream;
    UpkeepGrid g;
    size_t n_list = 0, SK = 0, SL = 0, SB = 0;
    for (int w = 0; w < W; ++w) {
        n_list += (size_t)r[w].n_kf + r[w].n_lm; SK += (size_t)r[w].n_kf; SL += (size_t)r[w].n_lm; SB += (size_t)r[w].bound;
        g.max_kf = std::max(g.max_kf, r[w].n_kf); g.max_lm = std::max(g.max_lm, r[w].n_lm);
        g.max_meas = std::max(g.max_meas, r[w].max_meas);
    }
    const size_t o_lists = sizeof(UpkeepArgs) * (size_t)(W - 1), up_bytes = o_lists + 4 * n_list;
    // deactivation: common | active | lm_active; depth: cost | cnt | cand
    const size_t o2 = depth ? 8 * SB : 4 * SK, o3 = depth ? o2 + 4 * SK : o2 + SK;
    const size_t out_bytes = depth ? o3 + 4 * SB : o3 + SL;
    int* lists_h = reinterpret_cast<int*>(st.up.h + o_lists);
    const int* lists_d = reinterpret_cast<const int*>(st.up.d + o_lists);
    unsigned char* d = st.out.d;
    UpkeepLaunch l;
    l.rest = reinterpret_cast<const UpkeepArgs*>(st.up.d);
    l.n_win = W;
    size_t li = 0, cK = 0, cL = 0, cB = 0;
    for (int w = 0; w < W; ++w) {
        const UpkeepReq& q = r[w];
        UpkeepBufs& ub = *q.t->upkeep;
        if (ub.stamp >= 0xfffffff0u) {  // the stamps wrap: the map starts over from all 0
            CU(cudaMemsetAsync(ub.map, 0, sizeof(unsigned long long) * (size_t)q.t->td.lm_cap, s));
            ub.stamp = 0;
        }
        memcpy(lists_h + li, q.kf_slot, 4 * (size_t)q.n_kf);
        if (q.n_lm) memcpy(lists_h + li + q.n_kf, q.lm_slot, 4 * (size_t)q.n_lm);
        UpkeepArgs a;
        a.td = q.t->td;
        a.kf_slot = lists_d + li; a.lm_slot = lists_d + li + q.n_kf;
        a.n_kf = q.n_kf; a.n_lm = q.n_lm;
        a.stamp = ub.stamp + 1; ub.stamp += 2;
        a.map = ub.map;
        if (depth) {
            a.cost = reinterpret_cast<double*>(d + 8 * cB); a.cnt = reinterpret_cast<int*>(d + o2 + 4 * cK);
            a.cand = reinterpret_cast<int*>(d + o3 + 4 * cB);
        } else {
            a.min_connecting = q.dq->min_connecting; a.min_window = q.dq->min_window; a.max_window = q.dq->max_window;
            a.kf_common = reinterpret_cast<int*>(d + 4 * cK); a.kf_active = d + o2 + cK; a.lm_active = d + o3 + cL;
        }
        if (w == 0) l.w0 = a;
        else memcpy(st.up.h + sizeof(UpkeepArgs) * (size_t)(w - 1), &a, sizeof(UpkeepArgs));
        li += (size_t)q.n_kf + q.n_lm; cK += (size_t)q.n_kf; cL += (size_t)q.n_lm; cB += (size_t)q.bound;
    }
    CU(cudaMemcpyAsync(st.up.d, st.up.h, up_bytes, cudaMemcpyHostToDevice, s));
    if (depth) launch_depth_costs(l, g, s);
    else launch_deactivate(l, g, s);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpyAsync(st.out.h, st.out.d, out_bytes, cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = wait_stream(h);
    if (e != cudaSuccess) {
        // a failed sequence may have left any of this call's stamps in the maps: they go back to all 0 here, so that the map's
        // state does not depend on how far the sequence got (a sticky error leaves the context unusable anyway, and these calls
        // then fail as well)
        for (int w = 0; w < W; ++w) cudaMemsetAsync(r[w].t->upkeep->map, 0, sizeof(unsigned long long) * (size_t)r[w].t->td.lm_cap, s);
        cudaStreamSynchronize(s);
        return fail(KBA_ERR_CUDA, std::string(depth ? "depth costs: " : "keyframe deactivation: ") + cudaGetErrorString(e));
    }
    const unsigned char* hb = st.out.h;
    cK = cL = cB = 0;
    for (int w = 0; w < W; ++w) {
        const UpkeepReq& q = r[w];
        const size_t K = (size_t)q.n_kf, L = (size_t)q.n_lm;
        if (depth) {
            const int* cnt = reinterpret_cast<const int*>(hb + o2 + 4 * cK);
            int32_t* off = q.cout->off;
            size_t base = cB;  // keyframe k's pairs in the download start at the sum of the earlier keyframes' bounds
            off[0] = 0;
            for (size_t k = 0; k < K; ++k) {
                const int n = cnt[k];
                if (n) {
                    memcpy(q.cout->cand + off[k], hb + o3 + 4 * base, 4 * (size_t)n);
                    memcpy(q.cout->cost + off[k], hb + 8 * base, 8 * (size_t)n);
                }
                off[k + 1] = off[k] + n;
                base += (size_t)std::min(q.n_lm, q.t->m_cnt[q.kf_slot[k]]);
            }
        } else {
            memcpy(q.dout->kf_common, hb + 4 * cK, 4 * K);
            memcpy(q.dout->kf_active, hb + o2 + cK, K);
            if (L) memcpy(q.dout->lm_active, hb + o3 + cL, L);
        }
        cK += K; cL += L; cB += (size_t)q.bound;
    }
    st.counts.h2d = (int64_t)up_bytes;
    st.counts.d2h = (int64_t)out_bytes;
    return KBA_OK;
}

extern "C++" {  // overloads and templates have C++ linkage
static UpkeepReq upkeep_req(kba_track* t, const kba_deactivate_request& q, kba_deactivate_out* o) {
    UpkeepReq r;
    r.t = t; r.n_kf = q.n_kf; r.n_lm = q.n_lm; r.kf_slot = q.kf_slot; r.lm_slot = q.lm_slot; r.dq = &q; r.dout = o;
    return r;
}

static UpkeepReq upkeep_req(kba_track* t, const kba_depth_request& q, kba_depth_out* o) {
    UpkeepReq r;
    r.t = t; r.n_kf = q.n_kf; r.n_lm = q.n_elig; r.kf_slot = q.kf_slot; r.lm_slot = q.lm_slot; r.cout = o; r.cap = q.cap;
    return r;
}

// deactivation (Depth = false) and depth costs (Depth = true): one staging, one check, one run
template <class Q, class O, bool Depth>
struct Upkeep {
    using Request = Q;
    using Out = O;
    using Req = UpkeepReq;
    static constexpr StoreCall slot = kUpkeepCall;
    static constexpr const char* staging = "upkeep";
    static bool sits_out(const Request& q) { return q.n_kf == 0; }
    static int sit_out_check(const Out&, std::string&) { return KBA_OK; }
    static void sat_out(Out*, bool) {}
    static Req make(kba_track* t, const Request& q, Out* o) { return upkeep_req(t, q, o); }
    static int check(Req& r, std::string& why) { return upkeep_check(r, why); }
    static void capacity(int n, kba_track* const* ts, size_t& up, size_t& down) {
        size_t lists = 0;
        down = 0;
        for (int i = 0; i < n; ++i) { lists += (size_t)ts[i]->td.kf_cap + ts[i]->td.lm_cap; down += upkeep_out_cap(ts[i]); }
        up = sizeof(UpkeepArgs) * (size_t)(n - 1) + 4 * lists;
    }
    static int run(kba_handle* h, StoreStage& st, int W, Req* r, int&, std::string&) { return upkeep_run(h, st, W, r, Depth); }
};
}  // extern "C++"
using Deactivate = Upkeep<kba_deactivate_request, kba_deactivate_out, false>;
using DepthCosts = Upkeep<kba_depth_request, kba_depth_out, true>;

int kba_track_deactivate_keyframes(kba_track* t, const kba_deactivate_request* req, kba_deactivate_out* out) {
    static const std::string who = "kba_track_deactivate_keyframes: ";
    if (!t || !req || !out) return fail(KBA_ERR_BAD_ARG, who + "null argument");
    return store_call<Deactivate>(t->set, false, who, req, out);
}

int kba_track_depth_costs(kba_track* t, const kba_depth_request* req, kba_depth_out* out) {
    static const std::string who = "kba_track_depth_costs: ";
    if (!t || !req || !out) return fail(KBA_ERR_BAD_ARG, who + "null argument");
    return store_call<DepthCosts>(t->set, false, who, req, out);
}

int kba_track_group_deactivate_keyframes(kba_track_group* g, const kba_deactivate_request* req, kba_deactivate_out* out) {
    static const std::string who = "kba_track_group_deactivate_keyframes: ";
    if (!g || !req || !out) return fail(KBA_ERR_BAD_ARG, who + "null argument");
    return store_call<Deactivate>(g->set, true, who, req, out);
}

int kba_track_group_depth_costs(kba_track_group* g, const kba_depth_request* req, kba_depth_out* out) {
    static const std::string who = "kba_track_group_depth_costs: ";
    if (!g || !req || !out) return fail(KBA_ERR_BAD_ARG, who + "null argument");
    return store_call<DepthCosts>(g->set, true, who, req, out);
}

// ---------------------------------------------------------------------------------------------------------------------
// the flow scheme of keyframe selection on the stored window (include/kba_b200.h, kba_track_frame_flow /
// kba_track_group_frame_flow; kernels in kba_keyframe.cu): a single call is a one-window call of flow_run
// ---------------------------------------------------------------------------------------------------------------------
// one frame-flow request of track t (one window of flow_run)
struct FlowReq {
    kba_track* t = nullptr;
    const kba_flow_request* q = nullptr;
    kba_flow_out* o = nullptr;
};

// every check of one request, before anything is uploaded; allocates the track's upkeep scratch at its first upkeep or flow call
static int flow_check(kba_track* t, const kba_flow_request* q, std::string& why) {
    const int n = q->n_meas;
    if (n < 0) { why = "negative size"; return KBA_ERR_BAD_ARG; }
    if (n > 0 && (!q->lm_slot || !q->u || !q->v)) { why = "null argument"; return KBA_ERR_BAD_ARG; }
    if (q->kf_last < 0 || q->kf_last >= t->td.kf_cap || !t->kf_live[q->kf_last]) { why = "kf_last not pushed"; return KBA_ERR_BAD_ARG; }
    if (n > t->caps.win_observations) { why = "more measurements than win_observations"; return KBA_ERR_CAPACITY; }
    const int rb = upkeep_bufs(t, why);
    if (rb != KBA_OK) return rb;
    SlotStamps& st = t->stamps;
    st.next();
    for (int i = 0; i < n; ++i) {
        const int s = q->lm_slot[i], c = q->cam ? q->cam[i] : 0;
        if (s < 0 || s >= t->td.lm_cap) { why = "landmark slot out of range"; return KBA_ERR_BAD_ARG; }
        if (c < 0 || c >= t->n_cam) { why = "camera out of range"; return KBA_ERR_BAD_ARG; }
        if (i > 0 && s == q->lm_slot[i - 1]) {
            if (c <= (q->cam ? q->cam[i - 1] : 0)) { why = "camera not ascending inside a run"; return KBA_ERR_BAD_ARG; }
            continue;
        }
        if (st.lm[s] == st.cur) { why = "landmark slot reappears after its run"; return KBA_ERR_BAD_ARG; }
        st.lm[s] = st.cur;
    }
    return KBA_OK;
}

// a flow record's mean_flow_sq.  Without a match it is 0 / 0: the NaN's bits are the host CPU's default NaN in the facade (x86-64:
// sign bit set), which the device's canonical NaN is not, so the library forms this one quotient with the host's own arithmetic.
static double mean_flow_sq(const FlowRes& r) {
    if (r.n_matched != 0) return r.mean_flow_sq;
    volatile double zero = 0.;
    const double q0 = r.flow_sum / zero;
    return q0 * q0;
}

// W checked requests of distinct tracks as the W windows of one launch sequence: one upload (the argument records of windows
// 1 .. W-1, then every window's lm | cam | u | v), one download (the FlowRes records of all windows, then their match indices),
// one synchronisation, then the scatter into the callers' outputs.  Window 0's record travels in the launch parameters.
static int flow_run(kba_handle* h, StoreStage& st, int W, const FlowReq* r) {
    CU(cudaSetDevice(h->device));
    cudaStream_t s = h->stream;
    FlowGrid g;
    size_t SN = 0;
    for (int w = 0; w < W; ++w) {
        SN += (size_t)r[w].q->n_meas;
        g.max_last = std::max(g.max_last, r[w].t->m_cnt[r[w].q->kf_last]);
    }
    const size_t o_lists = sizeof(FlowArgs) * (size_t)(W - 1), up_bytes = o_lists + 16 * SN;
    const size_t o_match = sizeof(FlowRes) * (size_t)W, out_bytes = o_match + 4 * SN;
    unsigned char* up_h = st.up.h + o_lists;
    const unsigned char* up_d = st.up.d + o_lists;
    FlowLaunch l;
    l.rest = reinterpret_cast<const FlowArgs*>(st.up.d);
    l.n_win = W;
    size_t li = 0, mi = 0;
    for (int w = 0; w < W; ++w) {
        const kba_flow_request& q = *r[w].q;
        const size_t n = (size_t)q.n_meas;
        UpkeepBufs& ub = *r[w].t->upkeep;
        if (ub.stamp >= 0xfffffff0u) {  // the stamps wrap: the map starts over from all 0
            CU(cudaMemsetAsync(ub.map, 0, sizeof(unsigned long long) * (size_t)r[w].t->td.lm_cap, s));
            ub.stamp = 0;
        }
        int32_t* lm = reinterpret_cast<int32_t*>(up_h + li);
        int32_t* cam = lm + n;
        if (n) {
            memcpy(lm, q.lm_slot, 4 * n);
            if (q.cam) memcpy(cam, q.cam, 4 * n);
            else memset(cam, 0, 4 * n);
            memcpy(cam + n, q.u, 4 * n);
            memcpy(cam + 2 * n, q.v, 4 * n);
        }
        FlowArgs a;
        a.td = r[w].t->td;
        a.kf_last = q.kf_last; a.n_meas = q.n_meas;
        a.lm_slot = reinterpret_cast<const int*>(up_d + li); a.cam = a.lm_slot + n;
        a.u = reinterpret_cast<const float*>(a.cam + n); a.v = a.u + n;
        a.min_median_flow = q.min_median_flow;
        a.stamp = ++ub.stamp;
        a.map = ub.map;
        a.res = reinterpret_cast<FlowRes*>(st.out.d) + w;
        a.match = reinterpret_cast<int*>(st.out.d + o_match) + mi;
        if (w == 0) l.w0 = a;
        else memcpy(st.up.h + sizeof(FlowArgs) * (size_t)(w - 1), &a, sizeof(FlowArgs));
        li += 16 * n; mi += n;
    }
    CU(cudaMemcpyAsync(st.up.d, st.up.h, up_bytes, cudaMemcpyHostToDevice, s));
    launch_frame_flow(l, g, s);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpyAsync(st.out.h, st.out.d, out_bytes, cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = wait_stream(h);
    if (e != cudaSuccess) {
        // as upkeep_run: the maps go back to all 0, whatever stamps the failed sequence left in them
        for (int w = 0; w < W; ++w) cudaMemsetAsync(r[w].t->upkeep->map, 0, sizeof(unsigned long long) * (size_t)r[w].t->td.lm_cap, s);
        cudaStreamSynchronize(s);
        return fail(KBA_ERR_CUDA, std::string("frame flow: ") + cudaGetErrorString(e));
    }
    const FlowRes* res = reinterpret_cast<const FlowRes*>(st.out.h);
    const int32_t* match = reinterpret_cast<const int32_t*>(st.out.h + o_match);
    mi = 0;
    for (int w = 0; w < W; ++w) {
        kba_flow_out& o = *r[w].o;
        const size_t n = (size_t)r[w].q->n_meas;
        o.n_matched = res[w].n_matched;
        o.usable = (uint8_t)res[w].usable;
        o.flow_sum = res[w].flow_sum;
        o.mean_flow_sq = mean_flow_sq(res[w]);
        if (o.match && n) memcpy(o.match, match + mi, 4 * n);
        mi += n;
    }
    st.counts.h2d = (int64_t)up_bytes;
    st.counts.d2h = (int64_t)out_bytes;
    return KBA_OK;
}

struct Flow {
    using Request = kba_flow_request;
    using Out = kba_flow_out;
    using Req = FlowReq;
    static constexpr StoreCall slot = kFlowCall;
    static constexpr const char* staging = "flow";
    static bool sits_out(const Request& q) { return q.kf_last < 0; }
    static int sit_out_check(const Out&, std::string&) { return KBA_OK; }
    static void sat_out(Out*, bool) {}
    static Req make(kba_track* t, const Request& q, Out* o) {
        Req r;
        r.t = t; r.q = &q; r.o = o;
        return r;
    }
    static int check(Req& r, std::string& why) { return flow_check(r.t, r.q, why); }
    static void capacity(int n, kba_track* const* ts, size_t& up, size_t& down) {  // win_observations measurements per track
        size_t obs = 0;
        for (int i = 0; i < n; ++i) obs += (size_t)ts[i]->caps.win_observations;
        up = sizeof(FlowArgs) * (size_t)(n - 1) + 16 * obs;
        down = sizeof(FlowRes) * (size_t)n + 4 * obs;
    }
    static int run(kba_handle* h, StoreStage& st, int W, Req* r, int&, std::string&) { return flow_run(h, st, W, r); }
};

int kba_track_frame_flow(kba_track* t, const kba_flow_request* req, kba_flow_out* out) {
    static const std::string who = "kba_track_frame_flow: ";
    if (!t || !req || !out) return fail(KBA_ERR_BAD_ARG, who + "null argument");
    return store_call<Flow>(t->set, false, who, req, out);
}

int kba_track_group_frame_flow(kba_track_group* g, const kba_flow_request* req, kba_flow_out* out) {
    static const std::string who = "kba_track_group_frame_flow: ";
    if (!g || !req || !out) return fail(KBA_ERR_BAD_ARG, who + "null argument");
    return store_call<Flow>(g->set, true, who, req, out);
}

// ---------------------------------------------------------------------------------------------------------------------
// free landmark slots of the stored window (include/kba_b200.h, kba_track_reclaim_landmarks / kba_track_group_reclaim_landmarks;
// kernels in kba_reclaim.cu): a single call is a one-window call of reclaim_run
// ---------------------------------------------------------------------------------------------------------------------
// the largest download of one window of track t: positions, weights and slots of a range of lm_cap slots, and n_free
static size_t reclaim_out_cap(const kba_track* t) { return 36 * (size_t)t->td.lm_cap + 4; }

// one reclaim request of track t (one window of reclaim_run)
struct ReclaimReq {
    kba_track* t = nullptr;
    const kba_reclaim_request* q = nullptr;
    kba_reclaim_out* o = nullptr;
};

// every check of one request, before anything is uploaded; allocates the track's upkeep scratch at its first upkeep, flow or
// reclaim call
static int reclaim_check(kba_track* t, const kba_reclaim_request* q, const kba_reclaim_out* o, std::string& why) {
    if (q->lo < 0 || q->hi < q->lo || q->hi > t->td.lm_cap) { why = "slot range not within [0, max_landmarks]"; return KBA_ERR_BAD_ARG; }
    if (q->hi > q->lo && !o->free_slot) { why = "null argument"; return KBA_ERR_BAD_ARG; }
    return upkeep_bufs(t, why);
}

// W checked requests of distinct tracks, none of them an empty range, as the W windows of one launch sequence: one upload (the
// argument records of windows 1 .. W-1, then every window's live keyframe slots), one download (the positions of the windows that
// ask for them | their weights | every window's slots | n_free of every window, each window's part sized for its whole range),
// one synchronisation, then the scatter into the callers' outputs.  Window 0's record travels in the launch parameters.
static int reclaim_run(kba_handle* h, StoreStage& st, int W, const ReclaimReq* r) {
    CU(cudaSetDevice(h->device));
    for (int w = 0; w < W; ++w) r[w].t->gen++;
    cudaStream_t s = h->stream;
    ReclaimGrid g;
    size_t SP = 0, SW = 0, SN = 0;
    for (int w = 0; w < W; ++w) {
        const size_t n = (size_t)(r[w].q->hi - r[w].q->lo);
        SN += n; SP += r[w].o->pos ? n : 0; SW += r[w].o->weight ? n : 0;
        g.max_range = std::max(g.max_range, r[w].q->hi - r[w].q->lo);
    }
    const size_t o_lists = sizeof(ReclaimArgs) * (size_t)(W - 1);
    const size_t o_w = 24 * SP, o_s = o_w + 8 * SW, o_n = o_s + 4 * SN, out_bytes = o_n + 4 * (size_t)W;
    int* lists_h = reinterpret_cast<int*>(st.up.h + o_lists);
    const int* lists_d = reinterpret_cast<const int*>(st.up.d + o_lists);
    unsigned char* d = st.out.d;
    ReclaimLaunch l;
    l.rest = reinterpret_cast<const ReclaimArgs*>(st.up.d);
    l.n_win = W;
    size_t li = 0, cP = 0, cW = 0, cN = 0;
    for (int w = 0; w < W; ++w) {
        kba_track* t = r[w].t;
        UpkeepBufs& ub = *t->upkeep;
        if (ub.stamp >= 0xfffffff0u) {  // the stamps wrap: the map starts over from all 0
            CU(cudaMemsetAsync(ub.map, 0, sizeof(unsigned long long) * (size_t)t->td.lm_cap, s));
            ub.stamp = 0;
        }
        ReclaimArgs a;
        a.td = t->td;
        a.kf_live = lists_d + li;
        for (int k = 0; k < t->td.kf_cap; ++k) {
            if (!t->kf_live[k]) continue;
            lists_h[li + (size_t)a.n_live++] = k;
            g.max_meas = std::max(g.max_meas, t->m_cnt[k]);
        }
        g.max_live = std::max(g.max_live, a.n_live);
        const size_t n = (size_t)(r[w].q->hi - r[w].q->lo);
        a.lo = r[w].q->lo; a.hi = r[w].q->hi;
        a.stamp = ++ub.stamp;
        a.map = ub.map; a.blk = ub.blk;
        a.n_free = reinterpret_cast<int*>(d + o_n) + w;
        a.free_slot = reinterpret_cast<int*>(d + o_s) + cN;
        if (r[w].o->pos) { a.pos = reinterpret_cast<double*>(d) + 3 * cP; cP += n; }
        if (r[w].o->weight) { a.weight = reinterpret_cast<double*>(d + o_w) + cW; cW += n; }
        if (w == 0) l.w0 = a;
        else memcpy(st.up.h + sizeof(ReclaimArgs) * (size_t)(w - 1), &a, sizeof(ReclaimArgs));
        li += (size_t)a.n_live; cN += n;
    }
    const size_t up_bytes = o_lists + 4 * li;
    CU(cudaMemcpyAsync(st.up.d, st.up.h, up_bytes, cudaMemcpyHostToDevice, s));
    launch_reclaim(l, g, s);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaMemcpyAsync(st.out.h, st.out.d, out_bytes, cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = wait_stream(h);
    if (e != cudaSuccess) {
        // as upkeep_run: the maps go back to all 0, whatever stamps the failed sequence left in them
        for (int w = 0; w < W; ++w) cudaMemsetAsync(r[w].t->upkeep->map, 0, sizeof(unsigned long long) * (size_t)r[w].t->td.lm_cap, s);
        cudaStreamSynchronize(s);
        return fail(KBA_ERR_CUDA, std::string("landmark reclaim: ") + cudaGetErrorString(e));
    }
    const unsigned char* hb = st.out.h;
    const int32_t* n_free = reinterpret_cast<const int32_t*>(hb + o_n);
    cP = cW = cN = 0;
    for (int w = 0; w < W; ++w) {
        kba_reclaim_out& o = *r[w].o;
        const size_t n = (size_t)(r[w].q->hi - r[w].q->lo), nf = (size_t)n_free[w];
        o.n_free = n_free[w];
        if (nf) memcpy(o.free_slot, hb + o_s + 4 * cN, 4 * nf);
        if (o.pos) { if (nf) memcpy(o.pos, hb + 24 * cP, 24 * nf); cP += n; }
        if (o.weight) { if (nf) memcpy(o.weight, hb + o_w + 8 * cW, 8 * nf); cW += n; }
        cN += n;
    }
    st.counts.h2d = (int64_t)up_bytes;
    st.counts.d2h = (int64_t)out_bytes;
    return KBA_OK;
}

struct Reclaim {
    using Request = kba_reclaim_request;
    using Out = kba_reclaim_out;
    using Req = ReclaimReq;
    static constexpr StoreCall slot = kReclaimCall;
    static constexpr const char* staging = "reclaim";
    static bool sits_out(const Request& q) { return q.hi == q.lo; }
    static int sit_out_check(const Out&, std::string&) { return KBA_OK; }
    static void sat_out(Out* o, bool group) {  // a single call's empty range has no free slot; a group's leaves out[i] as it is
        if (!group) o->n_free = 0;
    }
    static Req make(kba_track* t, const Request& q, Out* o) {
        Req r;
        r.t = t; r.q = &q; r.o = o;
        return r;
    }
    static int check(Req& r, std::string& why) { return reclaim_check(r.t, r.q, r.o, why); }
    static void capacity(int n, kba_track* const* ts, size_t& up, size_t& down) {  // every keyframe slot, a range of max_landmarks
        size_t kfs = 0;
        down = 0;
        for (int i = 0; i < n; ++i) { kfs += (size_t)ts[i]->td.kf_cap; down += reclaim_out_cap(ts[i]); }
        up = sizeof(ReclaimArgs) * (size_t)(n - 1) + 4 * kfs;
    }
    static int run(kba_handle* h, StoreStage& st, int W, Req* r, int&, std::string&) { return reclaim_run(h, st, W, r); }
};

int kba_track_reclaim_landmarks(kba_track* t, const kba_reclaim_request* req, kba_reclaim_out* out) {
    static const std::string who = "kba_track_reclaim_landmarks: ";
    if (!t || !req || !out) return fail(KBA_ERR_BAD_ARG, who + "null argument");
    return store_call<Reclaim>(t->set, false, who, req, out);
}

int kba_track_group_reclaim_landmarks(kba_track_group* g, const kba_reclaim_request* req, kba_reclaim_out* out) {
    static const std::string who = "kba_track_group_reclaim_landmarks: ";
    if (!g || !req || !out) return fail(KBA_ERR_BAD_ARG, who + "null argument");
    return store_call<Reclaim>(g->set, true, who, req, out);
}

// ---------------------------------------------------------------------------------------------------------------------
// motion-only frames against the persistent store (include/kba_b200.h, kba_track_adjust_pose / kba_track_group_adjust_pose)
// ---------------------------------------------------------------------------------------------------------------------
// every check of one frame, before anything is uploaded; n_runs = landmarks of the frame, rounds = trimming rounds it runs
static int frame_check(kba_track* t, const kba_track_frame* f, const kba_options* opt, int& n_runs, int& rounds, std::string& why) {
    n_runs = 0;
    if (f->n_meas < 0) { why = "negative n_meas"; return KBA_ERR_BAD_ARG; }
    if (!f->pose7 || !f->lm_slot || !f->u || !f->v || !f->d) { why = "null pose or measurement array"; return KBA_ERR_BAD_ARG; }
    if (f->speed_weight > 0 && !(f->speed_dt > 0)) { why = "speed prior: dt <= 0"; return KBA_ERR_BAD_ARG; }
    if (f->n_meas > t->caps.win_observations) { why = "more measurements than win_observations"; return KBA_ERR_CAPACITY; }
    SlotStamps& st = t->stamps;
    st.next();
    for (int i = 0; i < f->n_meas; ++i) {
        const int slot = f->lm_slot[i];
        if (slot < 0 || slot >= t->td.lm_cap) { why = "landmark slot out of range"; return KBA_ERR_BAD_ARG; }
        if (f->cam && (f->cam[i] < 0 || f->cam[i] >= t->n_cam)) { why = "camera index out of range"; return KBA_ERR_BAD_ARG; }
        if (i > 0 && slot == f->lm_slot[i - 1]) continue;
        if (st.lm[slot] == st.cur) { why = "landmark slot " + std::to_string(slot) + " reappears after its run"; return KBA_ERR_BAD_ARG; }
        st.lm[slot] = st.cur;
        ++n_runs;
    }
    if (n_runs > t->caps.win_landmarks) { why = "more landmarks than win_landmarks"; return KBA_ERR_CAPACITY; }
    rounds = opt->num_trim_rounds;  // k_reset_state's rule on the frame's landmark count
    if (rounds < 0) rounds = (n_runs > opt->min_landmarks_for_trimming) ? opt->num_rounds_option : 0;
    if (rounds > 6) rounds = 6;
    return KBA_OK;
}

static int options_check(const kba_options* opt, std::string& why) {
    if (opt->precision != 0) { why = "a frame is solved in FP64 only (kba_options.precision must be 0)"; return KBA_ERR_BAD_ARG; }
    if (quantile_check(opt, why) != KBA_OK) return KBA_ERR_BAD_ARG;
    if (opt->num_trim_rounds > 6 || (opt->num_trim_rounds < 0 && opt->num_rounds_option > 6)) {
        why = "at most 6 trimming rounds (KBA_MAX_SOLVES = 8 inner solves incl. one retry and the final solve)"; return KBA_ERR_CAPACITY;
    }
    return KBA_OK;
}

// one frame's results of k_adjust_pose (its FrameRes, log_cap iteration records, `runs` rejection flags) into r; ms the kernel's time
static void frame_result(const FrameRes& R, const IterRecord* lg, int log_cap, const unsigned char* rej, int runs, float ms, kba_result& r) {
    if (r.kf_pose) memcpy(r.kf_pose, R.pose, sizeof(R.pose));
    if (r.lm_rejected) memcpy(r.lm_rejected, rej, (size_t)runs);
    r.num_solves = R.n_solves;
    for (int k = 0; k < R.n_solves && k < KBA_MAX_SOLVES; ++k) {
        const SolveSummary& ss = R.solves[k];
        kba_solve_summary& o = r.solves[k];
        o.initial_cost = ss.initial_cost; o.final_cost = ss.final_cost; o.num_iterations = ss.num_iterations;
        o.num_successful_steps = ss.num_successful_steps; o.termination = ss.termination;
        o.num_landmarks = ss.num_landmarks; o.num_residual_blocks = ss.num_residual_blocks; o.reserved_ = 0;
    }
    r.initial_cost = R.n_solves > 0 ? R.solves[0].initial_cost : 0.0;
    r.final_cost = R.n_solves > 0 ? R.solves[R.n_solves - 1].final_cost : 0.0;
    r.status = R.done ? KBA_OK : KBA_ERR_TIMEOUT;
    r.time_sec = 1e-3 * ms;
    int k = 0;
    if (r.iterations) {
        for (; k < R.log_n && k < r.iterations_capacity && k < log_cap; ++k) {
            const IterRecord& e = lg[k];
            kba_iteration& o = r.iterations[k];
            o.cost = e.cost; o.cost_change = e.cost_change; o.gradient_max_norm = e.gradient_max_norm;
            o.step_norm = e.step_norm; o.relative_decrease = e.relative_decrease; o.trust_region_radius = e.radius;
            o.iteration = e.iteration; o.solve_index = e.solve_index; o.step_is_valid = e.valid; o.step_is_successful = e.successful;
        }
    }
    r.num_iteration_records = k;
}

// frames f[i] of tracks ts[i] (already checked; runs[i] landmarks, rounds[i] trimming rounds; n_meas == 0: idle) as one launch;
// opts[i] (per_frame) or opts[0] are their options
static int adjust_pose_run(kba_handle* h, MotionBufs& mb, int n, kba_track* const* ts, const kba_track_frame* f, const int* runs,
                           const int* rounds, bool per_frame, const kba_options* opts, kba_result* res, Transfer& tr) {
    std::vector<int> live;
    int M = 0, Rn = 0, log_cap = 0;
    bool any_cam = false;
    for (int i = 0; i < n; ++i) {
        if (f[i].n_meas == 0) { idle_result(res[i]); continue; }
        live.push_back(i);
        M += f[i].n_meas; Rn += runs[i];
        any_cam |= f[i].cam != nullptr;
        if (res[i].iterations) log_cap = std::max(log_cap, std::min(res[i].iterations_capacity, kIterLogCap));
    }
    tr = Transfer{};
    const int nf = (int)live.size();
    if (nf == 0) return KBA_OK;
    CU(cudaSetDevice(h->device));
    cudaStream_t s = h->stream;
    // ---- staged upload: descriptors | options | run starts | slots | cameras | u | v | d
    unsigned char* base = mb.up.h;
    FrameDesc* fd = reinterpret_cast<FrameDesc*>(base);
    size_t off = MotionBufs::al(sizeof(FrameDesc) * (size_t)nf);
    SolveParams* sp = reinterpret_cast<SolveParams*>(base + off); const size_t o_sp = off; off += MotionBufs::al(sizeof(SolveParams) * (size_t)nf);
    int* rs = reinterpret_cast<int*>(base + off); const size_t o_rs = off; off += MotionBufs::al(4 * ((size_t)Rn + nf));
    const size_t o_lm = off; off += MotionBufs::al(4 * (size_t)M);
    const size_t o_cam = off; if (any_cam) off += MotionBufs::al(4 * (size_t)M);
    const size_t o_u = off; off += MotionBufs::al(4 * (size_t)M);
    const size_t o_v = off; off += MotionBufs::al(4 * (size_t)M);
    const size_t o_d = off; off += MotionBufs::al(4 * (size_t)M);
    int mo = 0, ro = 0, rso = 0;
    for (int q = 0; q < nf; ++q) {
        const int i = live[q];
        const kba_track_frame& F = f[i];
        const kba_track* t = ts[i];
        FrameDesc& d = fd[q];
        d.n_meas = F.n_meas; d.n_runs = runs[i]; d.meas_off = mo; d.run_off = ro; d.rs_off = rso; d.rounds_total = rounds[i];
        sp[q] = make_params(&opts[per_frame ? i : 0]);
        d.lm_pos = t->td.lm_pos; d.lm_weight = t->td.lm_weight;
        d.cam16 = t->set.solver.batch->bd.cam + (size_t)t->set.solver.batch->desc_h[0].cam_off * kCamStride; d.n_cam = t->n_cam; d.pad = 0;
        memcpy(d.pose7, F.pose7, sizeof(d.pose7));
        d.speed_weight = F.speed_weight; d.speed_dt = F.speed_dt;
        memcpy(d.speed_v_before, F.speed_v_before, sizeof(d.speed_v_before));
        memcpy(d.speed_T_origin_before, F.speed_T_origin_before, sizeof(d.speed_T_origin_before));
        int r = 0;
        for (int k = 0; k < F.n_meas; ++k)
            if (k == 0 || F.lm_slot[k] != F.lm_slot[k - 1]) rs[rso + r++] = k;
        rs[rso + r] = F.n_meas;
        memcpy(base + o_lm + 4 * (size_t)mo, F.lm_slot, 4 * (size_t)F.n_meas);
        if (any_cam) {
            if (F.cam) memcpy(base + o_cam + 4 * (size_t)mo, F.cam, 4 * (size_t)F.n_meas);
            else memset(base + o_cam + 4 * (size_t)mo, 0, 4 * (size_t)F.n_meas);
        }
        memcpy(base + o_u + 4 * (size_t)mo, F.u, 4 * (size_t)F.n_meas);
        memcpy(base + o_v + 4 * (size_t)mo, F.v, 4 * (size_t)F.n_meas);
        memcpy(base + o_d + 4 * (size_t)mo, F.d, 4 * (size_t)F.n_meas);
        mo += F.n_meas; ro += runs[i]; rso += runs[i] + 1;
    }
    unsigned char* dev = mb.up.d;
    MotionArgs a;
    a.fd = reinterpret_cast<const FrameDesc*>(dev);
    a.sp = reinterpret_cast<const SolveParams*>(dev + o_sp);
    a.run_start = reinterpret_cast<const int*>(dev + o_rs);
    a.lm_slot = reinterpret_cast<const int*>(dev + o_lm);
    a.cam = any_cam ? reinterpret_cast<const int*>(dev + o_cam) : nullptr;
    a.u = reinterpret_cast<const float*>(dev + o_u);
    a.v = reinterpret_cast<const float*>(dev + o_v);
    a.d = reinterpret_cast<const float*>(dev + o_d);
    a.run_pw = mb.run_pw; a.run_active = mb.run_active; a.run_rej = mb.run_rej; a.trim_val = mb.trim_val; a.log = mb.log;
    a.total_runs = Rn; a.log_cap = log_cap;
    const size_t o_log = MotionBufs::al(sizeof(FrameRes) * (size_t)nf);
    const size_t o_rej = o_log + MotionBufs::al(sizeof(IterRecord) * (size_t)nf * log_cap);
    const size_t n_out = o_rej + MotionBufs::al((size_t)Rn);
    a.res = reinterpret_cast<FrameRes*>(mb.out.d);
    a.res_log = reinterpret_cast<IterRecord*>(mb.out.d + o_log);
    a.res_rej = mb.out.d + o_rej;
    // ---- one upload, one launch, one download, one synchronisation
    CU(cudaMemcpyAsync(mb.up.d, mb.up.h, off, cudaMemcpyHostToDevice, s));
    CU(cudaEventRecord(mb.ev0, s));
    launch_adjust_pose(a, nf, s);
    CU(cudaEventRecord(mb.ev1, s));
    CU(cudaMemcpyAsync(mb.out.h, mb.out.d, n_out, cudaMemcpyDeviceToHost, s));
    CU(wait_stream(h));
    CU(cudaGetLastError());
    float ms = 0.f;
    CU(cudaEventElapsedTime(&ms, mb.ev0, mb.ev1));
    h->counters.launches_total += 1;
    tr.h2d = (int64_t)off; tr.d2h = (int64_t)n_out;
    // ---- results
    const FrameRes* fr = reinterpret_cast<const FrameRes*>(mb.out.h);
    const IterRecord* lg = reinterpret_cast<const IterRecord*>(mb.out.h + o_log);
    const unsigned char* rj = mb.out.h + o_rej;
    for (int q = 0; q < nf; ++q)
        frame_result(fr[q], lg + (size_t)q * log_cap, log_cap, rj + fd[q].run_off, runs[live[q]], ms, res[live[q]]);
    return KBA_OK;
}

static int motion_alloc(std::unique_ptr<MotionBufs>& mb, int n, kba_track* const* ts) {
    if (mb) return KBA_OK;
    int runs = 0, meas = 0;
    for (int i = 0; i < n; ++i) { runs += ts[i]->caps.win_landmarks; meas += ts[i]->caps.win_observations; }
    std::unique_ptr<MotionBufs> m(new MotionBufs());
    if (m->alloc(n, runs, meas)) return fail(KBA_ERR_CUDA, "adjust_pose: out of memory");
    mb = std::move(m);
    return KBA_OK;
}

// a pose-only call of a track (group = false) or of a group: the options and every frame are checked before anything is uploaded
// or launched.  Errors start with `who`; a group's name the failing track.
static int track_adjust_pose(TrackSet& s, bool group, const std::string& who, const kba_track_frame* f, bool per_frame,
                             const kba_options* opts, kba_result* res) {
    TrackSolver& sv = s.solver;
    s.last = &sv.counts;
    std::string why;
    const int n = (int)s.tracks.size();
    int rc = KBA_OK;
    for (int i = 0; i < (per_frame ? n : 1); ++i) {
        if (per_frame && f[i].n_meas == 0) continue;  // a frame that sits the call out: its entry is not read
        rc = options_check(&opts[i], why);
        if (rc != KBA_OK) return fail(rc, who + (per_frame ? track_prefix(true, i) : std::string()) + why);
    }
    CU(cudaSetDevice(s.h->device));
    rc = motion_alloc(sv.motion, n, s.tracks.data());
    if (rc != KBA_OK) return rc;
    std::vector<int> runs(n, 0), rounds(n, 0);
    for (int i = 0; i < n; ++i) {
        if (f[i].n_meas == 0) continue;
        rc = frame_check(s.tracks[i], &f[i], &opts[per_frame ? i : 0], runs[i], rounds[i], why);
        if (rc != KBA_OK) return fail(rc, who + track_prefix(group, i) + why);
    }
    return adjust_pose_run(s.h, *sv.motion, n, s.tracks.data(), f, runs.data(), rounds.data(), per_frame, opts, res, sv.counts);
}

int kba_track_adjust_pose(kba_track* t, const kba_track_frame* f, const kba_options* opt, kba_result* res) {
    if (!t || !f || !opt || !res) return fail(KBA_ERR_BAD_ARG, "null argument to kba_track_adjust_pose");
    return track_adjust_pose(t->set, false, "kba_track_adjust_pose: ", f, false, opt, res);
}

int kba_track_group_adjust_pose(kba_track_group* g, const kba_track_frame* f, const kba_options* opt, kba_result* res) {
    if (!g || !f || !opt || !res) return fail(KBA_ERR_BAD_ARG, "null argument to kba_track_group_adjust_pose");
    return track_adjust_pose(g->set, true, "kba_track_group_adjust_pose: ", f, false, opt, res);
}

int kba_track_group_adjust_pose_opts(kba_track_group* g, const kba_track_frame* f, const kba_options* opts, kba_result* res) {
    if (!g || !f || !opts || !res) return fail(KBA_ERR_BAD_ARG, "null argument to kba_track_group_adjust_pose_opts");
    return track_adjust_pose(g->set, true, "kba_track_group_adjust_pose_opts: ", f, true, opts, res);
}

// ---------------------------------------------------------------------------------------------------------------------
// ranked landmark selection on the stored window, and solves of the ranking (include/kba_b200.h, kba_track_rank_landmarks /
// kba_track_solve_ranked and their group forms; kernels in kba_select.cu and kba_rank.cu)
// ---------------------------------------------------------------------------------------------------------------------
static int rank_alloc(kba_track* t, std::string& why) {
    std::unique_ptr<RankBufs> rb(new RankBufs());
    const size_t L = (size_t)t->td.lm_cap, K = (size_t)t->td.kf_cap, M = (size_t)t->td.m_cap;
    int bad = 0;
    DevAllocs& dev = rb->dev;
    bad |= dev.alloc(&rb->qty, select_out_bytes(L, 1)); bad |= dev.alloc(&rb->mark, L); bad |= dev.alloc(&rb->dcand, M);
    bad |= dev.alloc(&rb->dcost, M); bad |= dev.alloc(&rb->dcnt, K); bad |= dev.alloc(&rb->sel_slot, L); bad |= dev.alloc(&rb->gp, L);
    if (bad) { why = "out of memory for the ranking buffers"; return KBA_ERR_CUDA; }
    t->rank = std::move(rb);
    return KBA_OK;
}

struct RankReq {
    kba_track* t = nullptr;
    const kba_rank_request* q = nullptr;
    kba_rank_out* o = nullptr;
    SelectReq s;                           // the selection chain of the same lists
};

// the checks of a ranking's caps, candidate count and AddDepth entries
static int rank_entries_check(int n_cand, int max_near, int max_middle, int max_far, int n_depth, const kba_depth_entry* depth,
                              std::string& why) {
    if (n_depth > 0 && !depth) { why = "null argument"; return KBA_ERR_BAD_ARG; }
    if (max_near < 0 || max_middle < 0 || max_far < 0 || n_depth < 0) { why = "a negative cap or size"; return KBA_ERR_BAD_ARG; }
    for (int e = 0; e < n_depth; ++e)
        if (depth[e].ind < 0 || depth[e].wanted < 0) { why = "an AddDepth entry with a negative index or count"; return KBA_ERR_BAD_ARG; }
    if (n_cand > kRankMaxCand) { why = "more than 57344 candidates"; return KBA_ERR_CAPACITY; }
    if (n_depth > kRankMaxDepth) { why = "more than 1024 AddDepth entries"; return KBA_ERR_CAPACITY; }
    return KBA_OK;
}

// every check of one request, before anything is uploaded; allocates the track's selection and ranking buffers at its first call
static int rank_check(RankReq& r, std::string& why) {
    const kba_rank_request* q = r.q;
    if (!r.o || (q->n_cand > 0 && (!r.o->cand || !r.o->category))) { why = "null argument"; return KBA_ERR_BAD_ARG; }
    const int ec = rank_entries_check(q->n_cand, q->max_near, q->max_middle, q->max_far, q->n_depth, q->depth, why);
    if (ec != KBA_OK) return ec;
    SelectReq& s = r.s;
    s.t = r.t; s.n_kf = q->n_kf; s.n_cand = q->n_cand; s.kf_slot = q->kf_slot; s.lm_slot = q->lm_slot; s.p = q->params;
    s.quantities_only = true;
    int rc = select_check(s, why);
    if (rc != KBA_OK) return rc;
    for (int e = 0; e < q->n_depth; ++e)  // the AddDepth heap of an entry lives in shared memory
        if (q->depth[e].ind < q->n_kf && std::min(q->depth[e].wanted, r.t->m_cnt[q->kf_slot[q->depth[e].ind]]) > kRankMaxCand) {
            why = "an AddDepth entry keeps more than 57344 landmarks"; return KBA_ERR_CAPACITY;
        }
    if (!r.t->rank) rc = rank_alloc(r.t, why);
    return rc;
}

// W checked requests of distinct tracks as the W windows of one launch sequence in two parts (include/kba_b200.h): the lists go
// up, the chain and the AddDepth costs run, the middle bins' sizes come down; the draw functions fill the draws, which go up with
// each window's output offsets; the heaps, the shuffle and the union run, the outputs come down.  A draw function that fails
// or is missing fails the call as request `bad`, for `why`.
static int rank_run(kba_handle* h, StoreStage& st, int W, RankReq* r, int& bad, std::string& why) {
    CU(cudaSetDevice(h->device));
    cudaStream_t s = h->stream;
    SelectGrid sg;
    RankGrid rg;
    size_t n_list = 0, N = 0, ND = 0;
    for (int w = 0; w < W; ++w) {
        const kba_rank_request& q = *r[w].q;
        n_list += (size_t)q.n_kf + q.n_cand; N += (size_t)q.n_cand; ND += (size_t)q.n_depth;
        sg.max_kf = std::max(sg.max_kf, q.n_kf); sg.max_cand = std::max(sg.max_cand, q.n_cand);
        sg.max_init = std::max(sg.max_init, std::max(std::max(q.n_kf, q.n_cand), r[w].t->n_cam));
        sg.max_meas = std::max(sg.max_meas, r[w].s.max_meas);
        rg.max_depth = std::max(rg.max_depth, q.n_depth);
    }
    rg.max_kf = sg.max_kf; rg.max_cand = sg.max_cand;
    // ---- staging up: select records | rank records | AddDepth entries | lists | flags, then (first draw, first output) per window |
    // draws; down: middle-bin sizes, then (n_sel, n_ground) per window | candidates | categories
    static_assert(sizeof(SelectArgs) % 8 == 0 && sizeof(RankArgs) % 8 == 0, "records keep the entries 8-byte aligned");
    const size_t o_rrec = sizeof(SelectArgs) * (size_t)(W - 1), o_depth = o_rrec + sizeof(RankArgs) * (size_t)(W - 1);
    const size_t o_lists = o_depth + 8 * ND, o_elig = o_lists + 4 * n_list, up_bytes = o_elig + N, o_p2 = (up_bytes + 7) & ~(size_t)7;
    const size_t o_res = (4 * (size_t)W + 7) & ~(size_t)7;
    unsigned char* uh = st.up.h;
    const unsigned char* ud = st.up.d;
    SelectLaunch sl;
    sl.rest = reinterpret_cast<const SelectArgs*>(ud);
    sl.n_win = W;
    RankLaunch rl;
    rl.rest = reinterpret_cast<const RankArgs*>(ud + o_rrec);
    rl.n_win = W;
    rl.n_mid = reinterpret_cast<int*>(st.out.d);
    rl.p2 = reinterpret_cast<const int*>(ud + o_p2);
    rl.res = reinterpret_cast<int*>(st.out.d + o_res);
    size_t li = 0, c0 = 0, d0 = 0;
    for (int w = 0; w < W; ++w) {
        const kba_rank_request& q = *r[w].q;
        kba_track* t = r[w].t;
        RankBufs& rb = *t->rank;
        int* lists_h = reinterpret_cast<int*>(uh + o_lists) + li;
        const int* lists_d = reinterpret_cast<const int*>(ud + o_lists) + li;
        memcpy(lists_h, q.kf_slot, 4 * (size_t)q.n_kf);
        if (q.n_cand) memcpy(lists_h + q.n_kf, q.lm_slot, 4 * (size_t)q.n_cand);
        if (q.elig) memcpy(uh + o_elig + c0, q.elig, (size_t)q.n_cand); else memset(uh + o_elig + c0, 0, (size_t)q.n_cand);
        for (int e = 0; e < q.n_depth; ++e) {
            int* de = reinterpret_cast<int*>(uh + o_depth) + 2 * (d0 + e);
            de[0] = q.depth[e].ind; de[1] = q.depth[e].wanted;
        }
        // the chain: its quantities go to the ranking's device block instead of the download
        const size_t L = (size_t)t->td.lm_cap;
        unsigned char* qd = rb.qty;
        SelectArgs a = t->select->a;
        a.td = t->td;
        a.kf_slot = lists_d; a.lm_slot = lists_d + q.n_kf; a.n_kf = q.n_kf; a.n_cand = q.n_cand;
        for (int k = 0; k < 3; ++k) a.leaf[k] = q.params->voxel_size[k];
        a.roi_far = q.params->roi_far; a.roi_middle = q.params->roi_middle;
        a.flow = reinterpret_cast<double*>(qd); a.seen = reinterpret_cast<int*>(qd + 8 * L); a.near_order = reinterpret_cast<int*>(qd + 12 * L);
        a.counters = reinterpret_cast<int*>(qd + 16 * L); a.n_near = a.counters + 1;
        a.cheiral = qd + 16 * L + 16; a.bin = reinterpret_cast<signed char*>(qd + 17 * L + 16);
        RankArgs ra;
        ra.td = t->td;
        ra.kf_slot = a.kf_slot; ra.lm_slot = a.lm_slot; ra.elig = ud + o_elig + c0;
        ra.depth = reinterpret_cast<const int*>(ud + o_depth) + 2 * d0;
        ra.n_kf = q.n_kf; ra.n_cand = q.n_cand; ra.n_depth = q.n_depth;
        ra.max_near = q.max_near; ra.max_middle = q.max_middle; ra.max_far = q.max_far;
        ra.cheiral = a.cheiral; ra.bin = a.bin; ra.near_order = a.near_order; ra.n_near = a.n_near; ra.flow = a.flow; ra.seen = a.seen;
        ra.cand_of = a.cand_of; ra.mark = rb.mark; ra.dcand = rb.dcand; ra.dcost = rb.dcost; ra.dcnt = rb.dcnt;
        ra.sel_slot = rb.sel_slot; ra.gp = rb.gp;
        if (w == 0) { sl.w0 = a; rl.w0 = ra; }
        else {
            memcpy(uh + sizeof(SelectArgs) * (size_t)(w - 1), &a, sizeof(SelectArgs));
            memcpy(uh + o_rrec + sizeof(RankArgs) * (size_t)(w - 1), &ra, sizeof(RankArgs));
        }
        li += (size_t)q.n_kf + q.n_cand; c0 += (size_t)q.n_cand; d0 += (size_t)q.n_depth;
    }
    // ---- part one: the chain's quantities, the middle bins' sizes and the AddDepth costs
    CU(cudaMemcpyAsync(st.up.d, st.up.h, up_bytes, cudaMemcpyHostToDevice, s));
    CU(cudaMemsetAsync(rl.n_mid, 0, 4 * (size_t)W, s));
    launch_select(sl, sg, s);
    launch_rank_prepare(rl, rg, s);
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(st.out.h, st.out.d, 4 * (size_t)W, cudaMemcpyDeviceToHost, s));
    CU(wait_stream(h));
    // ---- the draws, each window's output offset and the heaps' shared memory
    const int* n_mid = reinterpret_cast<const int*>(st.out.h);
    int* p2 = reinterpret_cast<int*>(uh + o_p2);
    int* draws = p2 + 2 * W;
    size_t n_draws = 0, n_out = 0;
    std::vector<int> bound(W);
    for (int w = 0; w < W; ++w) {
        const kba_rank_request& q = *r[w].q;
        const int nm = n_mid[w], D = std::max(nm - 1, 0), n = q.n_cand;
        long long b = std::min(q.max_near, n) + (long long)std::min(q.max_middle, nm) + std::min(q.max_far, n);
        // an AddDepth heap holds at most min(wanted, arena entries of its keyframe) elements, whatever the runs of the keyframe
        int heap = std::max(std::min(q.max_near, n), std::min(q.max_far, n));
        for (int e = 0; e < q.n_depth; ++e) {
            b += std::min(q.depth[e].wanted, n);
            if (q.depth[e].ind < q.n_kf) heap = std::max(heap, std::min(q.depth[e].wanted, r[w].t->m_cnt[q.kf_slot[q.depth[e].ind]]));
        }
        bound[w] = (int)std::min<long long>(b, n);
        rg.heap_ints = std::max(rg.heap_ints, heap);
        rg.mid_ints = std::max(rg.mid_ints, nm);
        p2[2 * w] = (int)n_draws; p2[2 * w + 1] = (int)n_out;
        n_out += (size_t)bound[w];
        if (D == 0) continue;
        if (!q.draw) why = "the middle bin needs " + std::to_string(D) + " draws and there is no draw function";
        else if (q.draw(q.draw_ctx, D, draws + n_draws) != 0) why = "the draw function failed";
        if (!why.empty()) {  // nothing is written; the slot maps go back to all -1 and no track keeps a ranking
            for (int v = 0; v < W; ++v) {
                r[v].t->rank->valid = false;
                cudaMemsetAsync(r[v].t->select->a.cand_of, 0xff, sizeof(int) * (size_t)r[v].t->td.lm_cap, s);
            }
            cudaStreamSynchronize(s);
            bad = w;
            return KBA_ERR_BAD_ARG;
        }
        n_draws += (size_t)D;
    }
    // ---- part two: heaps, shuffle, union
    const size_t p2_bytes = 8 * (size_t)W + 4 * n_draws;
    CU(cudaMemcpyAsync(st.up.d + o_p2, uh + o_p2, p2_bytes, cudaMemcpyHostToDevice, s));
    rl.out_cand = reinterpret_cast<int*>(st.out.d + o_res + 8 * (size_t)W);
    rl.out_cat = reinterpret_cast<signed char*>(st.out.d + o_res + 8 * (size_t)W + 4 * n_out);
    launch_rank(rl, rg, s);
    CU(cudaGetLastError());
    const size_t out_bytes = 8 * (size_t)W + 5 * n_out;
    CU(cudaMemcpyAsync(st.out.h + o_res, st.out.d + o_res, out_bytes, cudaMemcpyDeviceToHost, s));
    CU(wait_stream(h));
    // ---- scatter
    const int* res = reinterpret_cast<const int*>(st.out.h + o_res);
    const unsigned char* hc = st.out.h + o_res + 8 * (size_t)W;
    for (int w = 0; w < W; ++w) {
        kba_rank_out& o = *r[w].o;
        RankBufs& rb = *r[w].t->rank;
        const int n_sel = res[2 * w], off = p2[2 * w + 1];
        o.n_sel = n_sel; o.n_ground = res[2 * w + 1]; o.n_draws = std::max(n_mid[w] - 1, 0);
        if (n_sel) { memcpy(o.cand, hc + 4 * (size_t)off, 4 * (size_t)n_sel); memcpy(o.category, hc + 4 * n_out + off, (size_t)n_sel); }
        rb.kf.assign(r[w].q->kf_slot, r[w].q->kf_slot + r[w].q->n_kf);
        rb.n_sel = n_sel; rb.n_ground = o.n_ground; rb.gen = r[w].t->gen; rb.valid = true;
    }
    st.counts.h2d = (int64_t)(up_bytes + p2_bytes);
    st.counts.d2h = (int64_t)(4 * (size_t)W + out_bytes);
    return KBA_OK;
}

struct Rank {
    using Request = kba_rank_request;
    using Out = kba_rank_out;
    using Req = RankReq;
    static constexpr StoreCall slot = kRankCall;
    static constexpr const char* staging = "ranking";
    static bool sits_out(const Request& q) { return q.n_kf == 0; }
    static int sit_out_check(const Out&, std::string&) { return KBA_OK; }
    static void sat_out(Out*, bool) {}
    static Req make(kba_track* t, const Request& q, Out* o) {
        Req r;
        r.t = t; r.q = &q; r.o = o;
        return r;
    }
    static int check(Req& r, std::string& why) { return rank_check(r, why); }
    static void capacity(int n, kba_track* const* ts, size_t& up, size_t& down) {
        up = (sizeof(SelectArgs) + sizeof(RankArgs)) * (size_t)(n - 1) + 8 * (size_t)kRankMaxDepth * n + 8 * (size_t)n + 8;
        down = 16 * (size_t)n + 8;
        for (int i = 0; i < n; ++i) {
            up += 4 * (size_t)ts[i]->td.kf_cap + 9 * (size_t)ts[i]->td.lm_cap;  // lists, flags, draws
            down += 5 * (size_t)ts[i]->td.lm_cap;
        }
    }
    static int run(kba_handle* h, StoreStage& st, int W, Req* r, int& bad, std::string& why) { return rank_run(h, st, W, r, bad, why); }
};

int kba_track_rank_landmarks(kba_track* t, const kba_rank_request* req, kba_rank_out* out) {
    static const std::string who = "kba_track_rank_landmarks: ";
    if (!t || !req) return fail(KBA_ERR_BAD_ARG, who + "null argument");
    return store_call<Rank>(t->set, false, who, req, out);  // a null out fails in rank_check
}

int kba_track_group_rank_landmarks(kba_track_group* g, const kba_rank_request* req, kba_rank_out* out) {
    static const std::string who = "kba_track_group_rank_landmarks: ";
    if (!g || !req || !out) return fail(KBA_ERR_BAD_ARG, who + "null argument");
    return store_call<Rank>(g->set, true, who, req, out);
}

int kba_track_solve_ranked(kba_track* t, int32_t n_kf, const int32_t* kf_slot, const uint8_t* kf_fixed, const kba_window* sel,
                           const kba_options* opt, kba_result* res) {
    if (!t || !opt || !res) return fail(KBA_ERR_BAD_ARG, "null argument to kba_track_solve_ranked");
    TrackRequest q = track_request(n_kf, kf_slot, kf_fixed, 0, nullptr, sel, true);
    return set_solve(t->set, false, "kba_track_solve_ranked: ", &q, false, opt, res);
}

static int group_solve_ranked(kba_track_group* g, const kba_ranked_request* req, bool per_track, const kba_options* opts,
                              kba_result* res, const std::string& who) {
    if (!g || !req || !opts || !res) return fail(KBA_ERR_BAD_ARG, "null argument to " + who.substr(0, who.size() - 2));
    std::vector<TrackRequest> qs;
    for (size_t i = 0; i < g->set.tracks.size(); ++i)
        qs.push_back(track_request(req[i].n_kf, req[i].kf_slot, req[i].kf_fixed, 0, nullptr, req[i].sel, true));
    return set_solve(g->set, true, who, qs.data(), per_track, opts, res);
}
int kba_track_group_solve_ranked(kba_track_group* g, const kba_ranked_request* req, const kba_options* opt, kba_result* res) {
    return group_solve_ranked(g, req, false, opt, res, "kba_track_group_solve_ranked: ");
}
int kba_track_group_solve_ranked_opts(kba_track_group* g, const kba_ranked_request* req, const kba_options* opts, kba_result* res) {
    return group_solve_ranked(g, req, true, opts, res, "kba_track_group_solve_ranked_opts: ");
}

// ---------------------------------------------------------------------------------------------------------------------
// store writes of a track and of a group (include/kba_b200.h, kba_track_push_keyframe / kba_track_group_push_keyframes, the drops,
// landmark values and keyframe poses; kernels in kba_store.cu and kba_pack.cu): a single call is a one-track call of store_call.
// A call checks every request, then makes one upload, one launch sequence and one synchronisation; more only when its rows
// exceed the staging, which holds the tracks' rows of one push (up to 65536 each) or one window's landmarks (win_landmarks).
// ---------------------------------------------------------------------------------------------------------------------
static size_t align16(size_t b) { return (b + 15) & ~(size_t)15; }

// the writes have no outputs
struct NoOut {};
struct WriteCall {
    using Out = NoOut;
    static int sit_out_check(const Out&, std::string&) { return KBA_OK; }
    static void sat_out(Out*, bool) {}
};

struct PushReq {
    kba_track* t = nullptr;
    const kba_push_request* q = nullptr;
};

// every check of kba_track_push_keyframe, the arena's capacity decided from the host mirror: nothing is compacted for a push that
// cannot fit
static int push_check(const PushReq& r, std::string& why) {
    const kba_track* t = r.t;
    const kba_push_request& q = *r.q;
    if (!q.pose7 || q.n_meas < 0 || q.kf_slot < 0 || q.kf_slot >= t->td.kf_cap || (q.n_meas > 0 && (!q.lm_slot || !q.u || !q.v || !q.d))) {
        why = "null argument, negative size or keyframe slot out of range"; return KBA_ERR_BAD_ARG;
    }
    if (t->kf_live[q.kf_slot]) { why = "slot in use (drop it first)"; return KBA_ERR_BAD_ARG; }
    for (int i = 0; i < q.n_meas; ++i)
        if (q.lm_slot[i] < 0 || q.lm_slot[i] >= t->td.lm_cap || (q.cam && (q.cam[i] < 0 || q.cam[i] >= t->n_cam))) {
            why = "landmark slot / camera out of range"; return KBA_ERR_BAD_ARG;
        }
    long long live = 0;
    for (int k = 0; k < t->td.kf_cap; ++k) live += t->kf_live[k] ? t->m_cnt[k] : 0;
    if (live + q.n_meas > t->td.m_cap) { why = "measurement arena full"; return KBA_ERR_CAPACITY; }
    return KBA_OK;
}

// rows of one push staged per track: larger pushes go up in several flushes
constexpr int kPushStageRows = 1 << 16;

// the host mirror's part of one push of n_meas measurements into keyframe slot `slot` of track t: a track whose arena has no room
// left at its end compacts (its live keyframes in slot order into the other arena: a CompactTrack and its runs, appended to ct and
// runs), then the keyframe goes to the end of the arena.  Returns its append record (seg, n, src still to be set).
static StoreAppend append_plan(kba_track* t, int32_t slot, int32_t n_meas, const double* pose7, const double* plane4, bool cam_zero,
                               std::vector<CompactTrack>& ct, std::vector<CompactRun>& runs, int& max_run) {
    static const double kNoPlane[4] = {0., 0., 1., 0.};
    if (t->arena_used + n_meas > t->td.m_cap) {
        const int cur = t->arena_cur, other = 1 - cur;
        CompactTrack c;
        for (int j = 0; j < 2; ++j) { c.src[j] = (const unsigned*)t->arena_i[cur][j]; c.dst[j] = (unsigned*)t->arena_i[other][j]; }
        for (int j = 0; j < 3; ++j) { c.src[2 + j] = (const unsigned*)t->arena_f[cur][j]; c.dst[2 + j] = (unsigned*)t->arena_f[other][j]; }
        c.m_off = t->td.m_off; c.m_cnt = t->td.m_cnt;
        int used = 0;
        for (int k = 0; k < t->td.kf_cap; ++k) {
            const int n = t->m_cnt[k];
            if (!t->kf_live[k]) {  // a dropped keyframe's count is cleared
                if (n) { runs.push_back(CompactRun{(int)ct.size(), k, 0, t->m_off[k], 0, 0}); t->m_cnt[k] = 0; }
                continue;
            }
            if (n == 0) continue;
            runs.push_back(CompactRun{(int)ct.size(), k, t->m_off[k], used, n, 0});
            max_run = std::max(max_run, n);
            t->m_off[k] = used;
            used += n;
        }
        ct.push_back(c);
        t->arena_cur = other; t->arena_used = used;
        t->point_arena();
    }
    StoreAppend a;
    a.col[0] = (unsigned*)t->td.m_lm; a.col[1] = (unsigned*)t->td.m_cam;
    a.col[2] = (unsigned*)t->td.m_u; a.col[3] = (unsigned*)t->td.m_v; a.col[4] = (unsigned*)t->td.m_d;
    a.m_off = t->td.m_off; a.m_cnt = t->td.m_cnt; a.kf_pose = t->td.kf_pose; a.kf_plane = t->td.kf_plane;
    memcpy(a.pose, pose7, sizeof(a.pose));
    memcpy(a.plane, plane4 ? plane4 : kNoPlane, sizeof(a.plane));
    a.slot = slot; a.off = t->arena_used; a.cnt = n_meas; a.cam_zero = cam_zero ? 1 : 0;
    t->m_off[slot] = t->arena_used; t->m_cnt[slot] = n_meas; t->kf_live[slot] = 1;
    t->arena_used += n_meas;
    t->gen++;
    t->h2d_push += (int64_t)n_meas * 20 + 11 * 8;
    return a;
}

// W checked pushes of distinct tracks.  The host mirror decides every offset first: a track whose arena has no room left compacts
// (its live keyframes in slot order into the other arena, as runs of k_arena_compact), and each keyframe goes to the end of its
// track's arena (segments of k_store_append, which also write its layout, pose and plane).  The staging, flushed when its rows are
// full: compaction records | runs | segments | the five columns (lm, cam, u, v, d) of `stride` words; a segment's rows start at a
// column offset congruent to their arena offset modulo 4, so that the copies run on 16-byte vectors.
static int push_run(kba_handle* h, StoreStage& st, int W, const PushReq* r) {
    CU(cudaSetDevice(h->device));
    cudaStream_t s = h->stream;
    std::vector<CompactTrack> ct;
    std::vector<CompactRun> runs;
    std::vector<StoreAppend> app(W);
    int max_run = 0;
    for (int w = 0; w < W; ++w) {
        const kba_push_request& q = *r[w].q;
        app[w] = append_plan(r[w].t, q.kf_slot, q.n_meas, q.pose7, q.plane4, q.cam == nullptr, ct, runs, max_run);
    }
    // ---- segments, flushed when the staging's rows are full (the first flush carries the compactions)
    const size_t rec = align16(sizeof(CompactTrack) * ct.size()) + align16(sizeof(CompactRun) * runs.size()) +
                       align16(sizeof(StoreAppend) * (size_t)W);
    const int cap = (int)(((st.up.n - rec) / 20) & ~(size_t)3);
    std::vector<StoreAppend> segs;
    std::vector<int> seg_w;
    int used = 0, max_rows = 0;
    bool first = true;
    int64_t up = 0;
    auto flush = [&]() -> int {
        const size_t nct = first ? ct.size() : 0, nrun = first ? runs.size() : 0;
        const size_t o_run = align16(sizeof(CompactTrack) * nct), o_app = o_run + align16(sizeof(CompactRun) * nrun);
        const size_t o_col = o_app + align16(sizeof(StoreAppend) * segs.size());
        const int stride = (used + 3) & ~3;
        unsigned char* hb = st.up.h;
        if (nct) memcpy(hb, ct.data(), sizeof(CompactTrack) * nct);
        if (nrun) memcpy(hb + o_run, runs.data(), sizeof(CompactRun) * nrun);
        memcpy(hb + o_app, segs.data(), sizeof(StoreAppend) * segs.size());
        unsigned* col = reinterpret_cast<unsigned*>(hb + o_col);
        for (size_t i = 0; i < segs.size(); ++i) {
            const StoreAppend& a = segs[i];
            const kba_push_request& q = *r[seg_w[i]].q;
            if (a.n == 0) continue;
            const size_t b = 4 * (size_t)a.n;
            memcpy(col + a.src, q.lm_slot + a.seg, b);
            if (q.cam) memcpy(col + stride + a.src, q.cam + a.seg, b);
            memcpy(col + 2 * (size_t)stride + a.src, q.u + a.seg, b);
            memcpy(col + 3 * (size_t)stride + a.src, q.v + a.seg, b);
            memcpy(col + 4 * (size_t)stride + a.src, q.d + a.seg, b);
        }
        const size_t bytes = o_col + 20 * (size_t)stride;
        CU(cudaMemcpyAsync(st.up.d, hb, bytes, cudaMemcpyHostToDevice, s));
        const unsigned char* db = st.up.d;
        launch_store_push(reinterpret_cast<const CompactTrack*>(db), reinterpret_cast<const CompactRun*>(db + o_run), (int)nrun, max_run,
                          reinterpret_cast<const StoreAppend*>(db + o_app), (int)segs.size(), max_rows,
                          reinterpret_cast<const unsigned*>(db + o_col), stride, s);
        CU(cudaGetLastError());
        CU(wait_stream(h));  // the staging is reused by the next flush
        up += (int64_t)bytes;
        first = false; segs.clear(); seg_w.clear(); used = 0; max_rows = 0;
        return KBA_OK;
    };
    for (int w = 0; w < W; ++w) {
        const int n = app[w].cnt;
        for (int done = 0;;) {  // one segment per flush; a keyframe without measurements is one empty segment
            const int dst = app[w].off + done, src = used + ((dst - used) & 3);
            const int m = std::min(n - done, cap - src);
            if (m < 0 || (m == 0 && done < n)) {
                const int rc = flush();
                if (rc != KBA_OK) return rc;
                continue;
            }
            StoreAppend a = app[w];
            a.seg = done; a.n = m; a.src = src;
            segs.push_back(a); seg_w.push_back(w);
            used = src + m; max_rows = std::max(max_rows, m); done += m;
            if (done >= n) break;
        }
    }
    const int rc = flush();
    if (rc != KBA_OK) return rc;
    st.counts.h2d = up;
    st.counts.d2h = 0;
    return KBA_OK;
}

struct Push : WriteCall {
    using Request = kba_push_request;
    using Req = PushReq;
    static constexpr StoreCall slot = kPushCall;
    static constexpr const char* staging = "keyframe";
    static bool sits_out(const Request& q) { return q.kf_slot < 0; }
    static Req make(kba_track* t, const Request& q, Out*) { return PushReq{t, &q}; }
    static int check(Req& r, std::string& why) { return push_check(r, why); }
    static void capacity(int n, kba_track* const* ts, size_t& up, size_t& down) {  // every track pushing and compacting
        size_t kfs = 0, rows = 4 * (size_t)n + 8;
        for (int i = 0; i < n; ++i) { kfs += (size_t)ts[i]->td.kf_cap; rows += (size_t)std::min(ts[i]->td.m_cap, kPushStageRows); }
        up = align16(sizeof(CompactTrack) * n) + align16(sizeof(CompactRun) * kfs) + align16(sizeof(StoreAppend) * n) + 20 * rows;
        down = 0;
    }
    static int run(kba_handle* h, StoreStage& st, int W, Req* r, int&, std::string&) { return push_run(h, st, W, r); }
};

// a drop moves nothing: the arena space of the keyframe is reclaimed by the next compaction
struct DropReq {
    kba_track* t = nullptr;
    int32_t slot = -1;
};
struct Drop : WriteCall {
    using Request = int32_t;
    using Req = DropReq;
    static constexpr StoreCall slot = kPushCall;
    static constexpr const char* staging = "keyframe";
    static bool sits_out(const Request& q) { return q < 0; }
    static Req make(kba_track* t, const Request& q, Out*) { return DropReq{t, q}; }
    static int check(Req& r, std::string& why) {
        if (r.slot >= 0 && r.slot < r.t->td.kf_cap) return KBA_OK;
        why = "keyframe slot out of range"; return KBA_ERR_BAD_ARG;
    }
    static void capacity(int n, kba_track* const* ts, size_t& up, size_t& down) { Push::capacity(n, ts, up, down); }
    static int run(kba_handle*, StoreStage& st, int W, Req* r, int&, std::string&) {
        for (int w = 0; w < W; ++w) { r[w].t->kf_live[r[w].slot] = 0; r[w].t->gen++; }
        st.counts = Transfer{};
        return KBA_OK;
    }
};

// one landmark or keyframe write of track t: n rows of two arrays of widths wa, wb (either may be NULL) into dst_a, dst_b by slot
struct ScatterReq {
    kba_track* t = nullptr;
    int n = 0;
    const int32_t* slot = nullptr;
    const double* a = nullptr;
    const double* b = nullptr;
};

// rows per track of a scatter's staging: one window's landmarks
static size_t scatter_rows(const kba_track* t) { return (size_t)std::max(t->caps.win_landmarks, 64); }
static size_t scatter_records(int W) { return 2 * align16(sizeof(ScatterWin) * (size_t)W) + 16; }

// W checked writes of distinct tracks: the slots | rows of array a | rows of array b, with a window record per track and array;
// one k_scatter_rows launch per array, flushed when the staging's rows are full
static int scatter_run(kba_handle* h, StoreStage& st, int W, const ScatterReq* r, int wa, int wb, bool landmarks) {
    CU(cudaSetDevice(h->device));
    cudaStream_t s = h->stream;
    for (int w = 0; w < W; ++w) r[w].t->gen++;
    st.counts = Transfer{};
    bool any = false;
    for (int w = 0; w < W; ++w) any |= r[w].a || r[w].b;
    if (!any) return KBA_OK;
    struct Seg { int w, done, m; };
    std::vector<Seg> segs;
    const int cap = (int)((st.up.n - scatter_records(W)) / (4 + 8 * (size_t)(wa + wb)));
    int rows = 0;
    auto flush = [&]() -> int {
        std::vector<ScatterWin> win_a, win_b;
        int ra = 0, rb = 0, max_a = 0, max_b = 0;
        int r0 = 0;
        for (const Seg& g : segs) {
            const ScatterReq& q = r[g.w];
            const TrackDev& td = q.t->td;
            if (q.a) { ScatterWin x; x.dst = landmarks ? td.lm_pos : td.kf_pose; x.slot0 = r0; x.val0 = ra; x.n = g.m; win_a.push_back(x); ra += g.m; max_a = std::max(max_a, g.m); }
            if (q.b) { ScatterWin x; x.dst = landmarks ? td.lm_weight : td.kf_plane; x.slot0 = r0; x.val0 = rb; x.n = g.m; win_b.push_back(x); rb += g.m; max_b = std::max(max_b, g.m); }
            r0 += g.m;
        }
        const size_t o_b = align16(sizeof(ScatterWin) * win_a.size()), o_slot = o_b + align16(sizeof(ScatterWin) * win_b.size());
        const size_t o_va = o_slot + align16(4 * (size_t)r0), o_vb = o_va + 8 * (size_t)wa * ra, bytes = o_vb + 8 * (size_t)wb * rb;
        unsigned char* hb = st.up.h;
        memcpy(hb, win_a.data(), sizeof(ScatterWin) * win_a.size());
        memcpy(hb + o_b, win_b.data(), sizeof(ScatterWin) * win_b.size());
        int* slot_h = reinterpret_cast<int*>(hb + o_slot);
        double* va = reinterpret_cast<double*>(hb + o_va), *vb = reinterpret_cast<double*>(hb + o_vb);
        for (const Seg& g : segs) {
            const ScatterReq& q = r[g.w];
            memcpy(slot_h, q.slot + g.done, 4 * (size_t)g.m);
            slot_h += g.m;
            if (q.a) { memcpy(va, q.a + (size_t)wa * g.done, 8 * (size_t)wa * g.m); va += (size_t)wa * g.m; }
            if (q.b) { memcpy(vb, q.b + (size_t)wb * g.done, 8 * (size_t)wb * g.m); vb += (size_t)wb * g.m; }
        }
        CU(cudaMemcpyAsync(st.up.d, hb, bytes, cudaMemcpyHostToDevice, s));
        const unsigned char* db = st.up.d;
        const int* slot_d = reinterpret_cast<const int*>(db + o_slot);
        launch_scatter_rows(reinterpret_cast<const ScatterWin*>(db), (int)win_a.size(), max_a, slot_d,
                            reinterpret_cast<const double*>(db + o_va), wa, s);
        launch_scatter_rows(reinterpret_cast<const ScatterWin*>(db + o_b), (int)win_b.size(), max_b, slot_d,
                            reinterpret_cast<const double*>(db + o_vb), wb, s);
        CU(cudaGetLastError());
        CU(wait_stream(h));  // the staging is reused by the next flush
        st.counts.h2d += (int64_t)bytes;
        segs.clear(); rows = 0;
        return KBA_OK;
    };
    for (int w = 0; w < W; ++w) {
        if (!r[w].a && !r[w].b) continue;
        for (int done = 0; done < r[w].n;) {
            if (rows == cap) { const int rc = flush(); if (rc != KBA_OK) return rc; }
            const int m = std::min(r[w].n - done, cap - rows);
            segs.push_back(Seg{w, done, m});
            rows += m; done += m;
        }
    }
    return segs.empty() ? KBA_OK : flush();
}

// every check of kba_track_set_landmarks / kba_track_set_keyframe_poses: slots in range (a slot listed twice is written in an
// unspecified order, as it always was)
static int scatter_check(const ScatterReq& r, bool need_a, int cap_slots, const char* what, std::string& why) {
    if (r.n < 0 || (r.n > 0 && (!r.slot || (need_a && !r.a)))) { why = "null argument or negative size"; return KBA_ERR_BAD_ARG; }
    for (int i = 0; i < r.n; ++i)
        if (r.slot[i] < 0 || r.slot[i] >= cap_slots) { why = std::string(what) + " slot out of range"; return KBA_ERR_BAD_ARG; }
    return KBA_OK;
}

extern "C++" {  // templates have C++ linkage
template <class Q, bool Landmarks>
struct Scatter : WriteCall {
    using Request = Q;
    using Req = ScatterReq;
    static constexpr int wa = Landmarks ? 3 : 7, wb = Landmarks ? 1 : 4;
    static constexpr StoreCall slot = Landmarks ? kLandmarkWriteCall : kPoseWriteCall;
    static constexpr const char* staging = Landmarks ? "landmark" : "keyframe pose";
    static bool sits_out(const Request& q) { return q.n == 0; }
    static Req make(kba_track* t, const kba_landmark_write& q, Out*) { return ScatterReq{t, q.n, q.lm_slot, q.pos3, q.weight}; }
    static Req make(kba_track* t, const kba_pose_write& q, Out*) { return ScatterReq{t, q.n, q.kf_slot, q.pose7s, q.plane4s}; }
    static int check(Req& r, std::string& why) {
        return Landmarks ? scatter_check(r, false, r.t->td.lm_cap, "landmark", why) : scatter_check(r, true, r.t->td.kf_cap, "keyframe", why);
    }
    static void capacity(int n, kba_track* const* ts, size_t& up, size_t& down) {
        size_t rows = 0;
        for (int i = 0; i < n; ++i) rows += scatter_rows(ts[i]);
        up = scatter_records(n) + (4 + 8 * (size_t)(wa + wb)) * rows;
        down = 0;
    }
    static int run(kba_handle* h, StoreStage& st, int W, Req* r, int&, std::string&) {
        if (Landmarks)
            for (int w = 0; w < W; ++w) r[w].t->h2d_push += (int64_t)r[w].n * ((r[w].a ? 24 : 0) + (r[w].b ? 8 : 0) + 4);
        return scatter_run(h, st, W, r, wa, wb, Landmarks);
    }
};
}  // extern "C++"
using LandmarkWrite = Scatter<kba_landmark_write, true>;
using PoseWrite = Scatter<kba_pose_write, false>;

int kba_track_push_keyframe(kba_track* t, int32_t slot, const double* pose7, const double* plane4, int32_t n, const int32_t* lm,
                            const int32_t* cam, const float* u, const float* v, const float* d) {
    static const std::string who = "kba_track_push_keyframe: ";
    if (!t) return fail(KBA_ERR_BAD_ARG, who + "null argument");
    const kba_push_request q = {slot, n, pose7, plane4, lm, cam, u, v, d};
    return store_call<Push>(t->set, false, who, &q, nullptr);
}

int kba_track_group_push_keyframes(kba_track_group* g, const kba_push_request* req) {
    static const std::string who = "kba_track_group_push_keyframes: ";
    if (!g || !req) return fail(KBA_ERR_BAD_ARG, who + "null argument");
    return store_call<Push>(g->set, true, who, req, nullptr);
}

int kba_track_drop_keyframe(kba_track* t, int32_t slot) {
    static const std::string who = "kba_track_drop_keyframe: ";
    if (!t) return fail(KBA_ERR_BAD_ARG, who + "null argument");
    return store_call<Drop>(t->set, false, who, &slot, nullptr);
}

int kba_track_group_drop_keyframes(kba_track_group* g, const int32_t* kf_slot) {
    static const std::string who = "kba_track_group_drop_keyframes: ";
    if (!g || !kf_slot) return fail(KBA_ERR_BAD_ARG, who + "null argument");
    return store_call<Drop>(g->set, true, who, kf_slot, nullptr);
}

int kba_track_set_landmarks(kba_track* t, int32_t n, const int32_t* slot, const double* pos3, const double* weight) {
    static const std::string who = "kba_track_set_landmarks: ";
    if (!t) return fail(KBA_ERR_BAD_ARG, who + "null argument");
    const kba_landmark_write q = {n, 0, slot, pos3, weight};
    return store_call<LandmarkWrite>(t->set, false, who, &q, nullptr);
}

int kba_track_group_set_landmarks(kba_track_group* g, const kba_landmark_write* req) {
    static const std::string who = "kba_track_group_set_landmarks: ";
    if (!g || !req) return fail(KBA_ERR_BAD_ARG, who + "null argument");
    return store_call<LandmarkWrite>(g->set, true, who, req, nullptr);
}

int kba_track_set_keyframe_poses(kba_track* t, int32_t n, const int32_t* slot, const double* pose7s, const double* plane4s) {
    static const std::string who = "kba_track_set_keyframe_poses: ";
    if (!t) return fail(KBA_ERR_BAD_ARG, who + "null argument");
    const kba_pose_write q = {n, 0, slot, pose7s, plane4s};
    return store_call<PoseWrite>(t->set, false, who, &q, nullptr);
}

int kba_track_set_keyframe_pose(kba_track* t, int32_t slot, const double* pose7, const double* plane4) {
    static const double kNoPlane[4] = {0., 0., 1., 0.};
    return kba_track_set_keyframe_poses(t, 1, &slot, pose7, plane4 ? plane4 : kNoPlane);
}

int kba_track_group_set_keyframe_poses(kba_track_group* g, const kba_pose_write* req) {
    static const std::string who = "kba_track_group_set_keyframe_poses: ";
    if (!g || !req) return fail(KBA_ERR_BAD_ARG, who + "null argument");
    return store_call<PoseWrite>(g->set, true, who, req, nullptr);
}

// ---------------------------------------------------------------------------------------------------------------------
// limo's solve block as one call (include/kba_b200.h, kba_track_keyframe_solve and its group forms; kernels in kba_upkeep.cu,
// kba_kfsolve.cu, kba_select.cu, kba_rank.cu).  One upload and one launch sequence run the deactivation, updateLabels and the
// post-deactivation lists (k_kfs_labels) and the ranking's first part for every window; one download brings back what the host
// needs next: the draws' counts, the kept keyframes, and the outputs.  Then the draws, the ranking's second part, the shrubbery
// weights (k_kfs_weights) and the ranked solve.  Every output is staged here and written when the call succeeds.
// ---------------------------------------------------------------------------------------------------------------------
// the KBA_LABEL_* classes of a label in the request's class table
static int label_classes(const kba_kfsolve_request& q, int32_t label) {
    int c = 0;
    for (int i = 0; i < q.n_class; ++i)
        if (q.classes[i].label == label) c |= q.classes[i].classes;
    return c;
}

// the checks that need only the request and are not the deactivation's (upkeep_check)
static int kfsolve_check(const kba_track* t, const kba_kfsolve_request& q, const kba_kfsolve_out* o, std::string& why) {
    if (!o || !q.sel || !q.params || !o->kf_active || !o->kf_common || (q.n_trk > 0 && (!q.trk || !o->trk_outlier)) ||
        (q.n_class > 0 && !q.classes) || (q.n_outlier > 0 && !q.outlier_slot) ||
        (q.n_lm > 0 && (!o->lm_active || !o->lm_outlier || !o->lm_ground || !o->rank.cand || !o->rank.category))) {
        why = "null argument"; return KBA_ERR_BAD_ARG;
    }
    if (q.n_trk < 0 || q.n_class < 0 || q.n_outlier < 0) { why = "a negative size"; return KBA_ERR_BAD_ARG; }
    for (int i = 0; i < q.n_trk; ++i)
        if (q.trk[i].lm_slot < -1 || q.trk[i].lm_slot >= t->td.lm_cap) { why = "tracklet landmark slot out of range"; return KBA_ERR_BAD_ARG; }
    for (int i = 0; i < q.n_outlier; ++i)
        if (q.outlier_slot[i] < 0 || q.outlier_slot[i] >= t->td.lm_cap) { why = "outlier landmark slot out of range"; return KBA_ERR_BAD_ARG; }
    for (int k = 0; k < 3; ++k)
        if (!(q.params->voxel_size[k] > 0.0) || !std::isfinite(q.params->voxel_size[k])) {
            why = "voxel sizes must be finite and positive"; return KBA_ERR_BAD_ARG;
        }
    // the candidates are a subset of the listed landmarks: their bound is checked before anything runs
    return rank_entries_check(q.n_lm, q.max_near, q.max_middle, q.max_far, q.n_depth, q.depth, why);
}

static int kfs_bufs(kba_track* t, std::string& why) {
    if (t->kfs) return KBA_OK;
    std::unique_ptr<KfsBufs> kb(new KfsBufs());
    const size_t L = (size_t)t->td.lm_cap;
    if (kb->dev.alloc(&kb->lm_at, L) | kb->dev.alloc(&kb->last, L)) { why = "out of memory for the label buffers"; return KBA_ERR_CUDA; }
    cudaError_t e = cudaMemsetAsync(kb->lm_at, 0xff, sizeof(int) * L, t->set.h->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(t->set.h->stream);
    if (e != cudaSuccess) { why = std::string("label buffers: ") + cudaGetErrorString(e); return KBA_ERR_CUDA; }
    t->kfs = std::move(kb);
    return KBA_OK;
}

// offsets in a staging block, each aligned
struct Bump {
    size_t at = 0;
    size_t take(size_t bytes, size_t align = 8) { at = (at + align - 1) & ~(align - 1); const size_t o = at; at += bytes; return o; }
};

// one live request's place in the call's staging (byte offsets; `d_*` in the download block, `x_*` in its device-only part)
struct KfsWin {
    kba_track* t = nullptr;
    int i = 0;                             // track index in the set
    int max_meas = 0;
    size_t u_kf, u_lm, u_out, u_trk, u_gin, u_cls, u_depth;
    size_t d_cnt, d_common, d_post, d_kfa, d_lma, d_lmo, d_gr, d_tro;
    size_t x_fixed, x_cand, x_elig, x_shrub;
    size_t u_tag = 0, d_nlm = 0, d_index = 0;  // the camera step's: candidate tags, the list's length, the candidates' positions
    int kn = 0, ln = 0;                    // the keyframes and landmarks listed (the camera step's: after the push)
    int K = 0, N = 0, bound = 0, p_out = 0;
    std::vector<int> kf, fixed;
};

// the refused call's cleanup after the ranking's first part ran: the slot maps back to all -1, no track keeps a ranking
static void kfs_abandon(cudaStream_t s, const std::vector<KfsWin>& ws) {
    for (const KfsWin& w : ws) {
        w.t->rank->valid = false;
        cudaMemsetAsync(w.t->select->a.cand_of, 0xff, sizeof(int) * (size_t)w.t->td.lm_cap, s);
    }
    cudaStreamSynchronize(s);
}

// one keyframe solve of the tracks of s (group = false: a single call), req[i] / out[i] / res[i] track i's, in the phases the
// camera step (set_camera_step) shares: the request checks (check), the staging's layout and lists (stage), the argument records
// (records), the first part's launches (launch_first: deactivation, labels and lists, the ranking's first part), and after its
// download the rest (rest: the checks on the kept keyframes, the draws, the ranking's second part, the weights, the solve and the
// outputs).  In the camera step (cs), each request's landmark list is the candidate bound, compacted by k_cs_lists into the list
// the deactivation and k_kfs_labels read, and its keyframe list may end with the frame's pending slot (kn: the keyframes listed).
extern "C++" {  // member templates have C++ linkage
struct KfsCall {
    TrackSet& s;
    bool group;
    const std::string& who;
    const kba_kfsolve_request* req;
    bool per_track;
    const kba_options* opts;
    kba_kfsolve_out* out;
    kba_result* res;
    bool cs = false;
    std::vector<KfsWin> ws;
    int W = 0, max_trk = 0;
    Bump up, dn, dx;
    size_t o_up_rec = 0, o_kfs = 0, o_sel = 0, o_rank = 0, o_cs = 0, o_mid = 0, rec_end = 0, up1 = 0, o_p2 = 0, down1 = 0, o_x = 0, o_res = 0;
    UpkeepGrid ug;
    SelectGrid sg;
    RankGrid rg;
    StoreStage* st = nullptr;
    UpkeepLaunch ul;
    Transfer sum;

    KfsCall(TrackSet& s_, bool group_, const std::string& who_, const kba_kfsolve_request* req_, bool per_track_, const kba_options* opts_,
            kba_kfsolve_out* out_, kba_result* res_)
        : s(s_), group(group_), who(who_), req(req_), per_track(per_track_), opts(opts_), out(out_), res(res_) {}

    // the options of the tracks live(i) names, before any request
    template <class Live>
    int check_options(Live live) {
        SolveTotals tot;
        std::string owhy;
        const int orc = solve_options_check((int)s.tracks.size(), opts, per_track, "track ", live, tot, owhy);
        return orc != KBA_OK ? fail(orc, who + owhy) : KBA_OK;
    }

    // every check of track i's request that needs only the request; the scratch of each step at its first use.  The last
    // kf_pending keyframes of the list are not pushed yet (the camera step's kf_new, which its frame step checks).
    int check(int i, int kf_pending) {
        kba_track* t = s.tracks[i];
        const kba_kfsolve_request& q = req[i];
        std::string why;
        int rc = kfsolve_check(t, q, out + i, why);
        if (rc == KBA_OK) {
            const kba_deactivate_request dq{q.n_kf - kf_pending, q.n_lm, q.min_connecting, q.min_window, q.max_window, 0, q.kf_slot, q.lm_slot};
            kba_deactivate_out dout{out[i].kf_active, out[i].kf_common, out[i].lm_active};
            UpkeepReq ur = upkeep_req(t, dq, &dout);
            rc = upkeep_check(ur, why);
            if (rc == KBA_OK && !t->select) rc = select_alloc(t, why);
            if (rc == KBA_OK && !t->rank) rc = rank_alloc(t, why);
            if (rc == KBA_OK) rc = kfs_bufs(t, why);
            KfsWin w;
            w.t = t; w.i = i; w.max_meas = ur.max_meas; w.kn = q.n_kf; w.ln = q.n_lm;
            ws.push_back(w);
        }
        return rc != KBA_OK ? fail(rc, who + track_prefix(group, i) + why) : KBA_OK;
    }

    // the layout (records | AddDepth entries | int lists | byte lists, then the draws' block; out = the first download | device-only
    // lists | the ranking's outputs), the staging grown to it, and every window's lists in the host staging
    int stage() {
        W = (int)ws.size();
        o_up_rec = up.take(sizeof(UpkeepArgs) * (size_t)(W - 1)); o_kfs = up.take(sizeof(KfsArgs) * (size_t)W);
        o_sel = up.take(sizeof(SelectArgs) * (size_t)W); o_rank = up.take(sizeof(RankArgs) * (size_t)W);
        if (cs) o_cs = up.take(sizeof(CsArgs) * (size_t)W);
        rec_end = up.at;
        o_mid = dn.take(4 * (size_t)W);
        size_t sum_lm = 0, max_draws = 0;
        for (KfsWin& w : ws) {
            const kba_kfsolve_request& q = req[w.i];
            const size_t K = (size_t)q.n_kf, L = (size_t)q.n_lm, O = (size_t)q.n_outlier, T = (size_t)q.n_trk;
            w.u_depth = up.take(8 * (size_t)q.n_depth);
            w.u_kf = up.take(4 * K, 4); w.u_lm = up.take(4 * L, 4); w.u_out = up.take(4 * O, 4); w.u_trk = up.take(4 * T, 4);
            if (cs) w.u_tag = up.take(4 * L, 4);
            w.d_cnt = dn.take(8); w.d_common = dn.take(4 * K, 4); w.d_post = dn.take(4 * K, 4);
            if (cs) { w.d_nlm = dn.take(4, 4); w.d_index = dn.take(4 * L, 4); }
            w.x_cand = dx.take(4 * L);
            sum_lm += L; max_draws += L > 0 ? L - 1 : 0;
            ug.max_kf = std::max(ug.max_kf, q.n_kf); ug.max_lm = std::max(ug.max_lm, q.n_lm); ug.max_meas = std::max(ug.max_meas, w.max_meas);
            sg.max_init = std::max(sg.max_init, std::max(std::max(q.n_kf, q.n_lm), w.t->n_cam));
            rg.max_depth = std::max(rg.max_depth, q.n_depth);
            max_trk = std::max(max_trk, q.n_trk);
        }
        for (KfsWin& w : ws) {  // the byte lists after every window's ints
            const kba_kfsolve_request& q = req[w.i];
            const size_t K = (size_t)q.n_kf, L = (size_t)q.n_lm, T = (size_t)q.n_trk;
            w.u_gin = up.take(L, 1); w.u_cls = up.take(T, 1);
            w.d_kfa = dn.take(K, 1); w.d_lma = dn.take(L, 1); w.d_lmo = dn.take(L, 1); w.d_gr = dn.take(L, 1); w.d_tro = dn.take(T, 1);
            w.x_fixed = dx.take(K, 1); w.x_elig = dx.take(L, 1); w.x_shrub = dx.take(T, 1);
        }
        sg.max_kf = ug.max_kf; sg.max_cand = ug.max_lm; sg.max_meas = ug.max_meas;
        rg.max_kf = sg.max_kf; rg.max_cand = sg.max_cand;
        up1 = up.at; o_p2 = up.take(8 * (size_t)W + 4 * max_draws); down1 = dn.at;
        o_x = (down1 + 7) & ~(size_t)7; o_res = o_x + ((dx.at + 7) & ~(size_t)7);
        const size_t out_need = o_res + 8 * (size_t)W + 5 * sum_lm;
        std::unique_ptr<StoreStage>& stage = s.stage[kKfSolveCall];
        if (!stage || stage->up.n < up.at || stage->out.n < out_need) {  // grow-only: a call no larger than an earlier one allocates nothing
            std::unique_ptr<StoreStage> fresh(new StoreStage());
            if (fresh->alloc(std::max(up.at, stage ? stage->up.n : 0), std::max(out_need, stage ? stage->out.n : 0)))
                return fail(KBA_ERR_CUDA, who + "out of memory for the keyframe solve staging");
            stage = std::move(fresh);
        }
        st = stage.get();
        unsigned char* uh = st->up.h;
        for (KfsWin& w : ws) {
            const kba_kfsolve_request& q = req[w.i];
            memcpy(uh + w.u_kf, q.kf_slot, 4 * (size_t)q.n_kf);
            if (q.n_lm) memcpy(uh + w.u_lm, q.lm_slot, 4 * (size_t)q.n_lm);
            if (q.n_outlier) memcpy(uh + w.u_out, q.outlier_slot, 4 * (size_t)q.n_outlier);
            if (q.lm_ground) memcpy(uh + w.u_gin, q.lm_ground, (size_t)q.n_lm); else memset(uh + w.u_gin, 0, (size_t)q.n_lm);
            int* ts = reinterpret_cast<int*>(uh + w.u_trk);
            for (int i = 0; i < q.n_trk; ++i) {
                const int c = label_classes(q, q.trk[i].label);
                ts[i] = q.trk[i].lm_slot;
                uh[w.u_cls + i] = (unsigned char)(((q.trk[i].is_outlier || (c & KBA_LABEL_OUTLIER)) ? kKfsMarked : 0) |
                                                  ((c & KBA_LABEL_SHRUBBERY) ? kKfsShrub : 0) | ((c & KBA_LABEL_GROUND) ? kKfsGround : 0));
            }
            int* de = reinterpret_cast<int*>(uh + w.u_depth);
            for (int e = 0; e < q.n_depth; ++e) { de[2 * e] = q.depth[e].ind; de[2 * e + 1] = q.depth[e].wanted; }
        }
        return KBA_OK;
    }

    // every window's argument records, on the keyframes it lists now (kn); cs: the camera step's list records, created[v] the
    // creation's flags of window v's frame (null: not selected)
    int records(const std::vector<const unsigned char*>* created = nullptr) {
        cudaStream_t st_s = s.h->stream;
        unsigned char* uh = st->up.h, *od = st->out.d;
        const unsigned char* ud = st->up.d;
        ul.rest = reinterpret_cast<const UpkeepArgs*>(ud + o_up_rec);
        ul.n_win = W;
        KfsArgs* kfs_h = reinterpret_cast<KfsArgs*>(uh + o_kfs);
        SelectArgs* sel_h = reinterpret_cast<SelectArgs*>(uh + o_sel);
        RankArgs* rank_h = reinterpret_cast<RankArgs*>(uh + o_rank);
        for (int v = 0; v < W; ++v) {
            KfsWin& w = ws[v];
            kba_track* t = w.t;
            const kba_kfsolve_request& q = req[w.i];
            const int* n_lm_d = nullptr;
            if (cs) {
                CsArgs c;
                c.lm_slot = reinterpret_cast<int*>(st->up.d + w.u_lm); c.ground = st->up.d + w.u_gin;
                c.tag = reinterpret_cast<const int*>(ud + w.u_tag); c.created = (*created)[v];
                c.n_cand = q.n_lm; c.selected = c.created != nullptr;
                c.index = reinterpret_cast<int*>(od + w.d_index); c.n_lm = reinterpret_cast<int*>(od + w.d_nlm);
                reinterpret_cast<CsArgs*>(uh + o_cs)[v] = c;
                n_lm_d = c.n_lm;
            }
            // the deactivation
            UpkeepBufs& ub = *t->upkeep;
            if (ub.stamp >= 0xfffffff0u) {  // the stamps wrap: the map starts over from all 0
                CU(cudaMemsetAsync(ub.map, 0, sizeof(unsigned long long) * (size_t)t->td.lm_cap, st_s));
                ub.stamp = 0;
            }
            UpkeepArgs a;
            a.td = t->td;
            a.kf_slot = reinterpret_cast<const int*>(ud + w.u_kf); a.lm_slot = reinterpret_cast<const int*>(ud + w.u_lm);
            a.n_kf = w.kn; a.n_lm = q.n_lm; a.n_lm_d = n_lm_d;
            a.stamp = ub.stamp + 1; ub.stamp += 2;
            a.map = ub.map;
            a.min_connecting = q.min_connecting; a.min_window = q.min_window; a.max_window = q.max_window;
            a.kf_common = reinterpret_cast<int*>(od + w.d_common); a.kf_active = od + w.d_kfa; a.lm_active = od + w.d_lma;
            if (v == 0) ul.w0 = a;
            else memcpy(uh + o_up_rec + sizeof(UpkeepArgs) * (size_t)(v - 1), &a, sizeof(UpkeepArgs));
            // the labels and the post-deactivation lists
            KfsArgs k;
            k.kf_slot = a.kf_slot; k.lm_slot = a.lm_slot; k.kf_active = a.kf_active; k.lm_active = a.lm_active;
            k.ground_in = ud + w.u_gin; k.out_slot = reinterpret_cast<const int*>(ud + w.u_out);
            k.trk_slot = reinterpret_cast<const int*>(ud + w.u_trk); k.trk_cls = ud + w.u_cls;
            k.n_kf = w.kn; k.n_lm = q.n_lm; k.n_lm_d = n_lm_d; k.n_out = q.n_outlier; k.n_trk = q.n_trk;
            k.lm_at = t->kfs->lm_at; k.last = t->kfs->last;
            k.lm_out = od + w.d_lmo; k.ground = od + w.d_gr; k.trk_out = od + w.d_tro; k.shrub = od + o_x + w.x_shrub;
            k.kf_post = reinterpret_cast<int*>(od + w.d_post); k.fixed = od + o_x + w.x_fixed;
            k.cand = reinterpret_cast<int*>(od + o_x + w.x_cand); k.elig = od + o_x + w.x_elig;
            k.counts = reinterpret_cast<int*>(od + w.d_cnt);
            k.sel = reinterpret_cast<SelectArgs*>(st->up.d + o_sel) + v; k.rank = reinterpret_cast<RankArgs*>(st->up.d + o_rank) + v;
            k.lm_weight = t->td.lm_weight; k.shrub_weight = q.shrubbery_weight;
            kfs_h[v] = k;
            // the ranking's chain on the device-built lists; k_kfs_labels writes its n_kf and n_cand
            const size_t L = (size_t)t->td.lm_cap;
            unsigned char* qd = t->rank->qty;
            SelectArgs sa = t->select->a;
            sa.td = t->td;
            sa.kf_slot = k.kf_post; sa.lm_slot = k.cand; sa.n_kf = 0; sa.n_cand = 0;
            for (int c = 0; c < 3; ++c) sa.leaf[c] = q.params->voxel_size[c];
            sa.roi_far = q.params->roi_far; sa.roi_middle = q.params->roi_middle;
            sa.flow = reinterpret_cast<double*>(qd); sa.seen = reinterpret_cast<int*>(qd + 8 * L); sa.near_order = reinterpret_cast<int*>(qd + 12 * L);
            sa.counters = reinterpret_cast<int*>(qd + 16 * L); sa.n_near = sa.counters + 1;
            sa.cheiral = qd + 16 * L + 16; sa.bin = reinterpret_cast<signed char*>(qd + 17 * L + 16);
            sel_h[v] = sa;
            RankArgs ra;
            ra.td = t->td;
            ra.kf_slot = sa.kf_slot; ra.lm_slot = sa.lm_slot; ra.elig = k.elig;
            ra.depth = reinterpret_cast<const int*>(ud + w.u_depth);
            ra.n_kf = 0; ra.n_cand = 0; ra.n_depth = q.n_depth;
            ra.max_near = q.max_near; ra.max_middle = q.max_middle; ra.max_far = q.max_far;
            ra.cheiral = sa.cheiral; ra.bin = sa.bin; ra.near_order = sa.near_order; ra.n_near = sa.n_near; ra.flow = sa.flow; ra.seen = sa.seen;
            RankBufs& rb = *t->rank;
            ra.cand_of = sa.cand_of; ra.mark = rb.mark; ra.dcand = rb.dcand; ra.dcost = rb.dcost; ra.dcnt = rb.dcnt;
            ra.sel_slot = rb.sel_slot; ra.gp = rb.gp;
            rank_h[v] = ra;
            t->rank->valid = false;  // replaced by this call's, or none if it is refused
        }
        return KBA_OK;
    }

    // the first part's launch sequence (cs: k_cs_lists first), enqueued after the upload of the records and lists
    cudaError_t launch_first() {
        cudaStream_t st_s = s.h->stream;
        const unsigned char* ud = st->up.d;
        cudaError_t e = cudaMemsetAsync(st->out.d + o_mid, 0, 4 * (size_t)W, st_s);
        if (e != cudaSuccess) return e;
        if (cs) launch_cs_lists(reinterpret_cast<const CsArgs*>(ud + o_cs), W, st_s);
        SelectLaunch sl;
        sl.all = reinterpret_cast<const SelectArgs*>(ud + o_sel); sl.n_win = W;
        RankLaunch rl;
        rl.all = reinterpret_cast<const RankArgs*>(ud + o_rank); rl.n_win = W;
        rl.n_mid = reinterpret_cast<int*>(st->out.d + o_mid);
        launch_deactivate(ul, ug, st_s);
        launch_kfs_labels(reinterpret_cast<const KfsArgs*>(ud + o_kfs), W, st_s);
        launch_select(sl, sg, st_s);
        launch_rank_prepare(rl, rg, st_s);
        return cudaGetLastError();
    }

    // after the first download: the checks on the kept keyframes, the draws, the ranking's second part, the ranked solve's checks,
    // the shrubbery weights, the solve and the outputs.  Every refusal comes before the store is written.
    int rest() {
        kba_handle* h = s.h;
        cudaStream_t st_s = h->stream;
        const int n = (int)s.tracks.size();
        unsigned char* uh = st->up.h, *od = st->out.d;
        const unsigned char* ud = st->up.d;
        const unsigned char* oh = st->out.h;
        const int* n_mid = reinterpret_cast<const int*>(oh + o_mid);
        int* p2 = reinterpret_cast<int*>(uh + o_p2);
        int* draws = p2 + 2 * W;
        size_t n_draws = 0, n_out = 0;
        std::vector<TrackRequest> qs(n);
        for (int v = 0; v < W; ++v) {
            KfsWin& w = ws[v];
            const kba_kfsolve_request& q = req[w.i];
            const int* cnt = reinterpret_cast<const int*>(oh + w.d_cnt);
            w.K = cnt[0]; w.N = cnt[1];
            if (cs) w.ln = *reinterpret_cast<const int*>(oh + w.d_nlm);
            std::string why;
            int rc = KBA_OK;
            if (w.K == 0) { why = "no keyframes or a negative size"; rc = KBA_ERR_BAD_ARG; }
            if (rc == KBA_OK) {
                const int* post = reinterpret_cast<const int*>(oh + w.d_post);
                w.kf.assign(post, post + w.K);
                w.fixed.assign(w.K, 0);
                w.fixed[0] = 1;
                for (int e = 0; e < q.n_depth && rc == KBA_OK; ++e)  // the AddDepth heap of an entry lives in shared memory
                    if (q.depth[e].ind < w.K && std::min(q.depth[e].wanted, w.t->m_cnt[w.kf[q.depth[e].ind]]) > kRankMaxCand) {
                        why = "an AddDepth entry keeps more than 57344 landmarks"; rc = KBA_ERR_CAPACITY;
                    }
            }
            if (rc == KBA_OK) {
                // the solve's keyframe checks; the ranking's ground candidates are not known yet: on a window without any
                kba_window sel0 = *q.sel;
                sel0.n_gp = 0;
                std::vector<uint8_t> f8(w.fixed.begin(), w.fixed.end());
                TrackRequest q0 = track_request(w.K, w.kf.data(), f8.data(), 0, nullptr, &sel0, true);
                rc = track_check(w.t, q0, why);
            }
            if (rc == KBA_OK) {
                const int nm = n_mid[v], D = std::max(nm - 1, 0), N = w.N;
                long long b = std::min(q.max_near, N) + (long long)std::min(q.max_middle, nm) + std::min(q.max_far, N);
                int heap = std::max(std::min(q.max_near, N), std::min(q.max_far, N));
                for (int e = 0; e < q.n_depth; ++e) {
                    b += std::min(q.depth[e].wanted, N);
                    if (q.depth[e].ind < w.K) heap = std::max(heap, std::min(q.depth[e].wanted, w.t->m_cnt[w.kf[q.depth[e].ind]]));
                }
                w.bound = (int)std::min<long long>(b, N);
                rg.heap_ints = std::max(rg.heap_ints, heap);
                rg.mid_ints = std::max(rg.mid_ints, nm);
                p2[2 * v] = (int)n_draws; p2[2 * v + 1] = (int)n_out;
                w.p_out = (int)n_out;
                n_out += (size_t)w.bound;
                if (D > 0) {
                    if (!q.draw) { why = "the middle bin needs " + std::to_string(D) + " draws and there is no draw function"; rc = KBA_ERR_BAD_ARG; }
                    else if (q.draw(q.draw_ctx, D, draws + n_draws) != 0) { why = "the draw function failed"; rc = KBA_ERR_BAD_ARG; }
                    n_draws += (size_t)D;
                }
            }
            if (rc != KBA_OK) {
                kfs_abandon(st_s, ws);
                return fail(rc, who + track_prefix(group, w.i) + why);
            }
        }
        // ---- the ranking's second part
        RankLaunch rl;
        rl.all = reinterpret_cast<const RankArgs*>(ud + o_rank); rl.n_win = W;
        rl.n_mid = reinterpret_cast<int*>(od + o_mid);
        const size_t p2_bytes = 8 * (size_t)W + 4 * n_draws;
        CU(cudaMemcpyAsync(st->up.d + o_p2, uh + o_p2, p2_bytes, cudaMemcpyHostToDevice, st_s));
        rl.p2 = reinterpret_cast<const int*>(ud + o_p2);
        rl.res = reinterpret_cast<int*>(od + o_res);
        rl.out_cand = reinterpret_cast<int*>(od + o_res + 8 * (size_t)W);
        rl.out_cat = reinterpret_cast<signed char*>(od + o_res + 8 * (size_t)W + 4 * n_out);
        launch_rank(rl, rg, st_s);
        CU(cudaGetLastError());
        const size_t down2 = 8 * (size_t)W + 5 * n_out;
        CU(cudaMemcpyAsync(st->out.h + o_res, st->out.d + o_res, down2, cudaMemcpyDeviceToHost, st_s));
        CU(wait_stream(h));
        sum.h2d += (int64_t)p2_bytes; sum.d2h += (int64_t)down2;
        const int* rres = reinterpret_cast<const int*>(oh + o_res);
        for (int v = 0; v < W; ++v) {
            KfsWin& w = ws[v];
            RankBufs& rb = *w.t->rank;
            rb.kf = w.kf; rb.n_sel = rres[2 * v]; rb.n_ground = rres[2 * v + 1]; rb.gen = w.t->gen; rb.valid = true;
        }
        // ---- the ranked solve's checks, the shrubbery weights, the solve
        std::vector<std::vector<uint8_t>> fixed8(n);
        for (const KfsWin& w : ws) {
            fixed8[w.i].assign(w.fixed.begin(), w.fixed.end());
            qs[w.i] = track_request(w.K, w.kf.data(), fixed8[w.i].data(), 0, nullptr, req[w.i].sel, true);
            TrackRequest q = qs[w.i];
            std::string why;
            const int rc = ranked_check(w.t, q, why);
            if (rc != KBA_OK) return fail(rc, who + track_prefix(group, w.i) + why);
        }
        launch_kfs_weights(reinterpret_cast<const KfsArgs*>(ud + o_kfs), W, max_trk, st_s);
        CU(cudaGetLastError());
        for (const KfsWin& w : ws) { w.t->gen++; w.t->rank->gen = w.t->gen; }  // the weights do not enter the ranking
        int rc = set_solve(s, group, who, qs.data(), per_track, opts, res);
        if (rc != KBA_OK) return rc;
        sum.h2d += s.last->h2d; sum.d2h += s.last->d2h;
        // ---- the outputs
        const unsigned char* hc = oh + o_res + 8 * (size_t)W;
        for (int v = 0; v < W; ++v) {
            const KfsWin& w = ws[v];
            const kba_kfsolve_request& q = req[w.i];
            kba_kfsolve_out& o = out[w.i];
            memcpy(o.kf_active, oh + w.d_kfa, (size_t)w.kn); memcpy(o.kf_common, oh + w.d_common, 4 * (size_t)w.kn);
            if (w.ln) {
                memcpy(o.lm_active, oh + w.d_lma, (size_t)w.ln); memcpy(o.lm_outlier, oh + w.d_lmo, (size_t)w.ln);
                memcpy(o.lm_ground, oh + w.d_gr, (size_t)w.ln);
            }
            if (q.n_trk) memcpy(o.trk_outlier, oh + w.d_tro, (size_t)q.n_trk);
            const int n_sel = rres[2 * v];
            o.rank.n_sel = n_sel; o.rank.n_ground = rres[2 * v + 1]; o.rank.n_draws = std::max(n_mid[v] - 1, 0);
            if (n_sel) { memcpy(o.rank.cand, hc + 4 * (size_t)w.p_out, 4 * (size_t)n_sel); memcpy(o.rank.category, hc + 4 * n_out + w.p_out, (size_t)n_sel); }
        }
        st->counts = sum;
        s.last = &st->counts;
        return KBA_OK;
    }
};
}

static int set_keyframe_solve(TrackSet& s, bool group, const std::string& who, const kba_kfsolve_request* req, bool per_track,
                              const kba_options* opts, kba_kfsolve_out* out, kba_result* res) {
    const int n = (int)s.tracks.size();
    auto sits_out = [&](int i) { return group && req[i].n_kf == 0; };
    KfsCall c(s, group, who, req, per_track, opts, out, res);
    int rc = c.check_options([&](int i) { return !sits_out(i); });
    for (int i = 0; i < n && rc == KBA_OK; ++i)
        if (!sits_out(i)) rc = c.check(i, 0);
    if (rc != KBA_OK) return rc;
    if (c.ws.empty()) {  // no upload, no launch
        for (int i = 0; i < n; ++i) idle_result(res[i]);
        s.last = &kNoTransfer;
        return KBA_OK;
    }
    kba_handle* h = s.h;
    CU(cudaSetDevice(h->device));
    if ((rc = c.stage()) != KBA_OK || (rc = c.records()) != KBA_OK) return rc;
    // ---- one upload, one launch sequence (deactivation, labels and lists, the ranking's first part), one download
    StoreStage& st = *c.st;
    CU(cudaMemcpyAsync(st.up.d, st.up.h, c.up1, cudaMemcpyHostToDevice, h->stream));
    CU(c.launch_first());
    CU(cudaMemcpyAsync(st.out.h, st.out.d, c.down1, cudaMemcpyDeviceToHost, h->stream));
    CU(wait_stream(h));
    c.sum.h2d = (int64_t)c.up1; c.sum.d2h = (int64_t)c.down1;
    return c.rest();
}

int kba_track_keyframe_solve(kba_track* t, const kba_kfsolve_request* req, const kba_options* opt, kba_kfsolve_out* out, kba_result* res) {
    static const std::string who = "kba_track_keyframe_solve: ";
    if (!t || !req || !opt || !out || !res) return fail(KBA_ERR_BAD_ARG, who + "null argument");
    return set_keyframe_solve(t->set, false, who, req, false, opt, out, res);
}

static int group_keyframe_solve(kba_track_group* g, const kba_kfsolve_request* req, bool per_track, const kba_options* opts,
                                kba_kfsolve_out* out, kba_result* res, const std::string& who) {
    if (!g || !req || !opts || !out || !res) return fail(KBA_ERR_BAD_ARG, who + "null argument");
    return set_keyframe_solve(g->set, true, who, req, per_track, opts, out, res);
}
int kba_track_group_keyframe_solve(kba_track_group* g, const kba_kfsolve_request* req, const kba_options* opt, kba_kfsolve_out* out,
                                   kba_result* res) {
    return group_keyframe_solve(g, req, false, opt, out, res, "kba_track_group_keyframe_solve: ");
}
int kba_track_group_keyframe_solve_opts(kba_track_group* g, const kba_kfsolve_request* req, const kba_options* opts,
                                        kba_kfsolve_out* out, kba_result* res) {
    return group_keyframe_solve(g, req, true, opts, out, res, "kba_track_group_keyframe_solve_opts: ");
}

// ---------------------------------------------------------------------------------------------------------------------
// limo's frame step as one store call (include/kba_b200.h, kba_track_frame_step and its group forms; kernels in kba_framestep.cu,
// kba_motion.cu, kba_keyframe.cu, kba_store.cu, kba_create.cu).  One upload stages every window's frame once; one launch
// sequence gathers the adjusted frames' selected runs (k_fs_gather), adjusts their poses and computes the flow from the staged
// columns; one download brings back what the host's verdict needs.  The selected windows then append the staged columns (the
// adjusted pose read from device memory) and create their landmarks: one more upload of records and one more download.
// ---------------------------------------------------------------------------------------------------------------------
// KeyframeSelectionSchemePose's angle: calcQuaternionDiff of the facade (mini_eigen.hpp), the angle of AngleAxisd(q1.inverse() *
// q0), in its operation order (limo_b200/keyframe_selector.py states the same), on the host: atan2 has no bit-exact device twin
static double quaternion_diff(const double* p0, const double* p1) {
    const double w0 = p0[0], x0 = p0[1], y0 = p0[2], z0 = p0[3];
    const double w1 = p1[0], x1 = p1[1], y1 = p1[2], z1 = p1[3];
    const double n = w1 * w1 + x1 * x1 + y1 * y1 + z1 * z1;
    const double aw = w1 / n, ax = -x1 / n, ay = -y1 / n, az = -z1 / n;
    const double qw = aw * w0 - ax * x0 - ay * y0 - az * z0;
    const double qx = aw * x0 + ax * w0 + ay * z0 - az * y0;
    const double qy = aw * y0 - ax * z0 + ay * w0 + az * x0;
    const double qz = aw * z0 + ax * y0 - ay * x0 + az * w0;
    const double sn = std::sqrt(qx * qx + qy * qy + qz * qz);
    return sn != 0.0 ? 2.0 * std::atan2(sn, std::fabs(qw)) : 0.0;
}

// one live request's place in the call (byte offsets into the staging)
struct StepWin {
    kba_track* t = nullptr;
    int i = 0;                             // track index in the set
    const kba_frame_step_request* q = nullptr;
    int n_runs = 0, sel_runs = 0, sel_meas = 0, rounds = 0, max_meas = 0;
    bool adjusted = false;                 // a pose-only frame of the launch: adjust set and a run selected
    int a = -1;                            // its index among the adjusted frames
    int src = 0, flag0 = 0;                // its rows of the staged columns, its first run flag
    size_t u_list = 0;                     // kf_slot | kf_new | new_slot
    size_t d_pose = 0, d_flow = 0, d_match = 0, d_create = 0;
    bool selected = false;
    double angle = 0.;
    unsigned char verdict[3] = {0, 0, 0};
    // the lidar form: the rows of each camera's measurements (a view each), in request order, camera by camera
    std::vector<int> cam_rows, cam_off;    // cam_off[n_cam + 1]: camera c's rows are cam_rows[cam_off[c] .. cam_off[c + 1])
};

// every check of one request that needs only the request; allocates the track's upkeep and creation scratch at their first use
static int step_check(kba_track* t, const kba_frame_step_request& q, const kba_frame_step_out* o, const kba_options* opt,
                      const kba_frame_lidar* lid, StepWin& w, std::string& why) {
    if (!o || !q.kf_slot || !q.pose7 || (q.n_meas > 0 && (!q.lm_slot || !q.u || !q.v || (!q.d && !lid) || !q.run_sel)) ||
        (q.n_new > 0 && (!q.new_slot || !o->pos || !o->flags))) {
        why = "null argument"; return KBA_ERR_BAD_ARG;
    }
    if (q.n_kf < 1 || q.n_meas < 0 || q.n_new < 0) { why = "no keyframes or a negative size"; return KBA_ERR_BAD_ARG; }
    if (q.n_kf + 1 > t->td.kf_cap || q.n_new > t->td.lm_cap) { why = "more keyframes or landmarks than the track's slots"; return KBA_ERR_CAPACITY; }
    if (q.kf_new < 0 || q.kf_new >= t->td.kf_cap) { why = "kf_new out of range"; return KBA_ERR_BAD_ARG; }
    if (t->kf_live[q.kf_new]) { why = "kf_new in use (drop it first)"; return KBA_ERR_BAD_ARG; }
    if (q.n_meas > t->caps.win_observations) { why = "more measurements than win_observations"; return KBA_ERR_CAPACITY; }
    if (q.adjust) {
        const int rc = options_check(opt, why);
        if (rc != KBA_OK) return rc;
        if (q.speed_weight > 0 && !(q.speed_dt > 0)) { why = "speed prior: dt <= 0"; return KBA_ERR_BAD_ARG; }
    }
    const cudaError_t e = cudaSetDevice(t->set.h->device);
    if (e != cudaSuccess) { why = std::string("cudaSetDevice: ") + cudaGetErrorString(e); return KBA_ERR_CUDA; }
    int rc = upkeep_bufs(t, why);
    if (rc == KBA_OK && !t->create) rc = create_alloc(t, why);
    if (rc == KBA_OK) rc = check_slot_lists(t, q.n_kf, q.kf_slot, q.n_new, q.new_slot, w.max_meas, why);
    if (rc != KBA_OK) return rc;
    // the run contract, as the flow and pose-only calls check it
    SlotStamps& st = t->stamps;
    st.next();
    w.n_runs = w.sel_runs = w.sel_meas = 0;
    for (int i = 0; i < q.n_meas; ++i) {
        const int sl = q.lm_slot[i], c = q.cam ? q.cam[i] : 0;
        if (sl < 0 || sl >= t->td.lm_cap) { why = "landmark slot out of range"; return KBA_ERR_BAD_ARG; }
        if (c < 0 || c >= t->n_cam) { why = "camera out of range"; return KBA_ERR_BAD_ARG; }
        if (i > 0 && sl == q.lm_slot[i - 1]) {
            if (c <= (q.cam ? q.cam[i - 1] : 0)) { why = "camera not ascending inside a run"; return KBA_ERR_BAD_ARG; }
        } else {
            if (st.lm[sl] == st.cur) { why = "landmark slot reappears after its run"; return KBA_ERR_BAD_ARG; }
            st.lm[sl] = st.cur;
            w.sel_runs += q.run_sel[w.n_runs] ? 1 : 0;
            ++w.n_runs;
        }
        w.sel_meas += q.run_sel[w.n_runs - 1] ? 1 : 0;
    }
    w.adjusted = q.adjust && w.sel_runs > 0;
    if (w.adjusted && w.sel_runs > t->caps.win_landmarks) { why = "more selected landmarks than win_landmarks"; return KBA_ERR_CAPACITY; }
    long long live = 0;
    for (int k = 0; k < t->td.kf_cap; ++k) live += t->kf_live[k] ? t->m_cnt[k] : 0;
    if (live + q.n_meas > t->td.m_cap) { why = "measurement arena full"; return KBA_ERR_CAPACITY; }
    w.rounds = opt->num_trim_rounds;  // k_reset_state's rule on the frame's landmark count, as frame_check
    if (w.rounds < 0) w.rounds = (w.sel_runs > opt->min_landmarks_for_trimming) ? opt->num_rounds_option : 0;
    if (w.rounds > 6) w.rounds = 6;
    w.max_meas = std::max(w.max_meas, q.n_meas);  // the creation lists the new keyframe too
    if (!lid) return KBA_OK;
    // the lidar form: the frame's cloud, and one view per camera that measures something
    if (!lid->T_cam_lidar || !lid->opt) { why = "null T_cam_lidar or lidar options"; return KBA_ERR_BAD_ARG; }
    if (lid->n_points < 0 || lid->stride < 3) { why = "cloud: negative n_points or stride < 3"; return KBA_ERR_BAD_ARG; }
    if (lid->n_points > 0 && !lid->points) { why = "cloud: null points"; return KBA_ERR_BAD_ARG; }
    w.cam_off.assign(t->n_cam + 1, 0);
    for (int i = 0; i < q.n_meas; ++i) ++w.cam_off[(q.cam ? q.cam[i] : 0) + 1];
    for (int c = 0; c < t->n_cam; ++c) w.cam_off[c + 1] += w.cam_off[c];
    w.cam_rows.resize((size_t)q.n_meas);
    std::vector<int> at(w.cam_off.begin(), w.cam_off.end() - 1);
    for (int i = 0; i < q.n_meas; ++i) w.cam_rows[at[q.cam ? q.cam[i] : 0]++] = i;
    return KBA_OK;
}

// what a call adds to the frame step's phases (the camera step's solve block, set_camera_step): its checks and staging after the
// frame step's checks, its upload with the frame step's first upload, whether it runs after the verdicts, and its launch sequence
// right after the push's and the creation's kernels, ahead of the second download.  Its transfers are its own to count.
struct StepHook {
    virtual int checked() = 0;
    virtual cudaError_t upload(cudaStream_t s) = 0;
    virtual bool due(const std::vector<StepWin>& ws) = 0;
    // created[v]: the creation's flags in device memory of ws[v]'s frame, null when it is not selected
    virtual cudaError_t launch(const std::vector<const unsigned char*>& created, cudaStream_t s) = 0;
};

// one frame step of the tracks of s (group = false: a single call), req[i] / out[i] / res[i] / lid[i] track i's; lid null: the
// requests' d columns are the depths, else the lidar kernels extract them from lid[i]'s cloud into the staged d column
static int set_frame_step(TrackSet& s, bool group, const std::string& who, const kba_frame_step_request* req, bool per_track,
                          const kba_options* opts, kba_frame_step_out* out, kba_result* res, const kba_frame_lidar* lid,
                          StepHook* hook = nullptr) {
    const int n = (int)s.tracks.size();
    std::vector<StepWin> ws;
    for (int i = 0; i < n; ++i) {
        if (group && req[i].n_kf == 0) continue;
        StepWin w;
        w.t = s.tracks[i]; w.i = i; w.q = &req[i];
        std::string why;
        const int rc = step_check(w.t, req[i], out + i, &opts[per_track ? i : 0], lid ? lid + i : nullptr, w, why);
        if (rc != KBA_OK) return fail(rc, who + track_prefix(group, i) + why);
        ws.push_back(std::move(w));
    }
    if (hook) {
        const int rc = hook->checked();
        if (rc != KBA_OK) return rc;
    }
    // the lidar views (cloud v is ws[v]'s), those of the frames whose depths are downloaded first: their features lead the
    // feature order, so the download is the first n_copy depths in that order
    LidarPlan plan((int)ws.size());
    std::vector<int> lid_order;
    int n_copy = 0;
    int64_t cloud_bytes = 0;
    if (lid) {
        for (int pass = 0; pass < 2; ++pass)
            for (int v = 0; v < (int)ws.size(); ++v)
                if ((lid[ws[v].i].depth_out != nullptr) == (pass == 0) && ws[v].q->n_meas > 0) lid_order.push_back(v);
        for (int v : lid_order) {
            const StepWin& w = ws[v];
            const kba_frame_lidar& l = lid[w.i];
            const kba_lidar_cloud cl{l.points, l.n_points, l.stride};
            if (l.depth_out) n_copy += w.q->n_meas;
            cloud_bytes += 4 * (int64_t)l.n_points * l.stride;
            for (int c = 0; c < w.t->n_cam; ++c) {
                const int m = w.cam_off[c + 1] - w.cam_off[c];
                if (m > 0 && plan.add(v, cl, l.T_cam_lidar + 7 * c, w.t->cam_intr.data() + 3 * c, l.opt + c, m) != KBA_OK)
                    return fail(KBA_ERR_CAPACITY, who + track_prefix(group, w.i) +
                                                      "the call's lidar cells, (view, point) pairs or features exceed 32-bit indexing");
            }
        }
    }
    for (int i = 0; i < n; ++i) idle_result(res[i]);  // written below for the adjusted frames
    if (ws.empty()) {  // no upload, no launch
        s.last = &kNoTransfer;
        return KBA_OK;
    }
    kba_handle* h = s.h;
    CU(cudaSetDevice(h->device));
    cudaStream_t cs = h->stream;
    TrackSolver& sv = s.solver;
    if (motion_alloc(sv.motion, n, s.tracks.data()) != KBA_OK) return fail(KBA_ERR_CUDA, who + "out of memory for the pose-only buffers");
    MotionBufs& mb = *sv.motion;
    const int W = (int)ws.size();
    // ---- layout.  up: step records | flow records | frame descriptors | solver options | columns lm, cam, u, v, d | lists | run
    // flags, then the second phase's records; down: frame results | iteration records | flow records | kf_last poses | match
    // indices | rejections, then the creations' positions | flags
    int A = 0, N = 0, Rn = 0, log_cap = 0, R_all = 0;
    size_t n_lists = 0, n_new = 0, kf_caps = 0;
    FlowGrid fg;
    for (StepWin& w : ws) {
        const kba_frame_step_request& q = *w.q;
        w.src = N; w.flag0 = R_all;
        N += q.n_meas; R_all += w.n_runs;
        n_lists += (size_t)q.n_kf + 1 + q.n_new; n_new += (size_t)q.n_new; kf_caps += (size_t)w.t->td.kf_cap;
        fg.max_last = std::max(fg.max_last, w.t->m_cnt[q.kf_slot[q.n_kf - 1]]);
        if (w.adjusted) {
            w.a = A++; Rn += w.sel_runs;
            const kba_result& r = res[w.i];
            if (r.iterations) log_cap = std::max(log_cap, std::min(r.iterations_capacity, kIterLogCap));
        }
    }
    Bump up, dn;
    const size_t o_step = up.take(sizeof(StepArgs) * (size_t)W), o_flow = up.take(sizeof(FlowArgs) * (size_t)W);
    const size_t o_fd = up.take(sizeof(FrameDesc) * (size_t)A), o_sp = up.take(sizeof(SolveParams) * (size_t)A);
    // the lidar form replaces the d column's upload by the lidar views' parameters and one feature index per measurement; the
    // columns then come last, so that the d column, which the lidar kernels write, is the first region past the upload
    size_t o_cols = lid ? 0 : up.take(20 * (size_t)N, 4), o_lpack = 0, o_idx = 0, o_dep = 0;
    if (lid) { o_lpack = up.take(plan.pack_bytes()); o_idx = up.take(4 * (size_t)N, 4); }
    for (StepWin& w : ws) w.u_list = up.take(4 * ((size_t)w.q->n_kf + 1 + w.q->n_new), 4);
    const size_t o_flags = up.take((size_t)R_all, 1);
    if (lid) o_cols = up.take(20 * (size_t)N, 4);
    const size_t up1 = lid ? o_cols + 16 * (size_t)N : up.at;
    const size_t o_fr = dn.take(sizeof(FrameRes) * (size_t)A), o_log = dn.take(sizeof(IterRecord) * (size_t)A * log_cap);
    const size_t o_fres = dn.take(sizeof(FlowRes) * (size_t)W), o_pose = dn.take(56 * (size_t)W);
    const size_t o_match = dn.take(4 * (size_t)N, 4);
    if (lid) o_dep = dn.take(4 * (size_t)n_copy, 4);
    const size_t o_rej = dn.take((size_t)Rn, 1), down1 = dn.at;
    // the second phase at its largest: every window selected and compacting
    Bump up2 = up, dn2 = dn;
    up2.take(0);
    const size_t up2_0 = up2.at;
    up2.take((sizeof(StoreAppend) + sizeof(CreateArgs) + sizeof(CompactTrack)) * (size_t)W + sizeof(CompactRun) * kf_caps);
    dn2.take(0);
    const size_t dn2_0 = dn2.at;
    dn2.take(25 * n_new);
    std::unique_ptr<StoreStage>& stage = s.stage[kFrameStepCall];
    if (!stage || stage->up.n < up2.at || stage->out.n < dn2.at) {  // grow-only: a call no larger than an earlier one allocates nothing
        std::unique_ptr<StoreStage> fresh(new StoreStage());
        if (fresh->alloc(std::max(up2.at, stage ? stage->up.n : 0), std::max(dn2.at, stage ? stage->out.n : 0)))
            return fail(KBA_ERR_CUDA, who + "out of memory for the frame step staging");
        stage = std::move(fresh);
    }
    StoreStage& st = *stage;
    unsigned char* uh = st.up.h, *od = st.out.d;
    const unsigned char* ud = st.up.d;
    LidarWs lws;
    if (!plan.par.empty() && lidar_workspace(h, plan, 0, lws) != KBA_OK) return fail(KBA_ERR_CUDA, who + "out of memory for the lidar workspace");
    // ---- staging: the columns, lists and flags once; the records of the gather, the adjustment and the flow
    unsigned* cols_h = reinterpret_cast<unsigned*>(uh + o_cols);
    const unsigned* cols_d = reinterpret_cast<const unsigned*>(ud + o_cols);
    StepArgs* step_h = reinterpret_cast<StepArgs*>(uh + o_step);
    FlowArgs* flow_h = reinterpret_cast<FlowArgs*>(uh + o_flow);
    FrameDesc* fd = reinterpret_cast<FrameDesc*>(uh + o_fd);
    SolveParams* sp = reinterpret_cast<SolveParams*>(uh + o_sp);
    const size_t m_cols = MotionBufs::al(sizeof(FrameDesc) * (size_t)mb.frames_cap) + MotionBufs::al(sizeof(SolveParams) * (size_t)mb.frames_cap);
    const size_t m_lm = m_cols + MotionBufs::al(4 * ((size_t)Rn + A)), m_stride = MotionBufs::al(4 * (size_t)std::max(N, 1));
    int mo = 0, ro = 0, rso = 0;
    for (int v = 0; v < W; ++v) {
        StepWin& w = ws[v];
        kba_track* t = w.t;
        const kba_frame_step_request& q = *w.q;
        const size_t m = (size_t)q.n_meas, b = 4 * m;
        if (m) {
            memcpy(cols_h + w.src, q.lm_slot, b);
            if (q.cam) memcpy(cols_h + N + w.src, q.cam, b); else memset(cols_h + N + w.src, 0, b);
            memcpy(cols_h + 2 * (size_t)N + w.src, q.u, b);
            memcpy(cols_h + 3 * (size_t)N + w.src, q.v, b);
            if (!lid) memcpy(cols_h + 4 * (size_t)N + w.src, q.d, b);
            memcpy(uh + o_flags + w.flag0, q.run_sel, (size_t)w.n_runs);
        }
        int* lh = reinterpret_cast<int*>(uh + w.u_list);
        memcpy(lh, q.kf_slot, 4 * (size_t)q.n_kf);
        lh[q.n_kf] = q.kf_new;
        if (q.n_new) memcpy(lh + q.n_kf + 1, q.new_slot, 4 * (size_t)q.n_new);
        w.d_pose = o_pose + 56 * (size_t)v; w.d_flow = o_fres + sizeof(FlowRes) * (size_t)v; w.d_match = o_match + 4 * (size_t)w.src;
        const int kf_last = q.kf_slot[q.n_kf - 1];
        StepArgs sa;
        sa.src = w.src; sa.n_meas = q.n_meas; sa.flag0 = w.flag0; sa.adjust = w.adjusted ? 1 : 0;
        sa.kf_pose = t->td.kf_pose + 7 * (size_t)kf_last; sa.last_pose = reinterpret_cast<double*>(od + w.d_pose);
        if (w.adjusted) {
            sa.meas_off = mo; sa.rs_off = rso;
            FrameDesc& d = fd[w.a];
            d.n_meas = w.sel_meas; d.n_runs = w.sel_runs; d.meas_off = mo; d.run_off = ro; d.rs_off = rso; d.rounds_total = w.rounds;
            sp[w.a] = make_params(&opts[per_track ? w.i : 0]);
            d.lm_pos = t->td.lm_pos; d.lm_weight = t->td.lm_weight;
            d.cam16 = t->set.solver.batch->bd.cam + (size_t)t->set.solver.batch->desc_h[0].cam_off * kCamStride; d.n_cam = t->n_cam; d.pad = 0;
            memcpy(d.pose7, q.pose7, sizeof(d.pose7));
            d.speed_weight = q.speed_weight; d.speed_dt = q.speed_dt;
            memcpy(d.speed_v_before, q.speed_v_before, sizeof(d.speed_v_before));
            memcpy(d.speed_T_origin_before, q.speed_T_origin_before, sizeof(d.speed_T_origin_before));
            mo += w.sel_meas; ro += w.sel_runs; rso += w.sel_runs + 1;
        }
        step_h[v] = sa;
        UpkeepBufs& ub = *t->upkeep;
        if (ub.stamp >= 0xfffffff0u) {  // the stamps wrap: the map starts over from all 0
            CU(cudaMemsetAsync(ub.map, 0, sizeof(unsigned long long) * (size_t)t->td.lm_cap, cs));
            ub.stamp = 0;
        }
        FlowArgs fa;
        fa.td = t->td;
        fa.kf_last = kf_last; fa.n_meas = q.n_meas;
        fa.lm_slot = reinterpret_cast<const int*>(cols_d + w.src); fa.cam = reinterpret_cast<const int*>(cols_d + N + w.src);
        fa.u = reinterpret_cast<const float*>(cols_d + 2 * (size_t)N + w.src); fa.v = reinterpret_cast<const float*>(cols_d + 3 * (size_t)N + w.src);
        fa.min_median_flow = q.min_median_flow;
        fa.stamp = ++ub.stamp;
        fa.map = ub.map;
        fa.res = reinterpret_cast<FlowRes*>(od + w.d_flow);
        fa.match = reinterpret_cast<int*>(od + w.d_match);
        flow_h[v] = fa;
    }
    std::vector<kba_lidar_cloud> clouds;
    LidarStaged lf;
    if (lid) {
        plan.pack(uh + o_lpack);
        int* idx = reinterpret_cast<int*>(uh + o_idx);
        for (int v : lid_order) {
            const StepWin& w = ws[v];
            for (int r : w.cam_rows) *idx++ = w.src + r;
        }
        for (const StepWin& w : ws) clouds.push_back(kba_lidar_cloud{lid[w.i].points, lid[w.i].n_points, lid[w.i].stride});
        lf.u = reinterpret_cast<const float*>(cols_d + 2 * (size_t)N); lf.v = reinterpret_cast<const float*>(cols_d + 3 * (size_t)N);
        lf.idx = reinterpret_cast<const int*>(ud + o_idx);
        lf.d = reinterpret_cast<float*>(st.up.d + o_cols + 16 * (size_t)N);
        lf.n_copy = n_copy; lf.copy = reinterpret_cast<float*>(od + o_dep);
    }
    StepLaunch gl;
    gl.win = reinterpret_cast<const StepArgs*>(ud + o_step);
    gl.cols = cols_d; gl.stride = N; gl.run_sel = ud + o_flags; gl.n_win = W;
    unsigned char* md = mb.up.d;
    for (int c = 0; c < 5; ++c) gl.dst[c] = reinterpret_cast<unsigned*>(md + m_lm + (size_t)c * m_stride);
    gl.run_start = reinterpret_cast<int*>(md + m_cols);
    MotionArgs ma;
    ma.fd = reinterpret_cast<const FrameDesc*>(ud + o_fd);
    ma.sp = reinterpret_cast<const SolveParams*>(ud + o_sp);
    ma.run_start = gl.run_start;
    ma.lm_slot = reinterpret_cast<const int*>(gl.dst[0]); ma.cam = reinterpret_cast<const int*>(gl.dst[1]);
    ma.u = reinterpret_cast<const float*>(gl.dst[2]); ma.v = reinterpret_cast<const float*>(gl.dst[3]); ma.d = reinterpret_cast<const float*>(gl.dst[4]);
    ma.run_pw = mb.run_pw; ma.run_active = mb.run_active; ma.run_rej = mb.run_rej; ma.trim_val = mb.trim_val; ma.log = mb.log;
    ma.total_runs = Rn; ma.log_cap = log_cap;
    ma.res = reinterpret_cast<FrameRes*>(od + o_fr);
    ma.res_log = reinterpret_cast<IterRecord*>(od + o_log);
    ma.res_rej = od + o_rej;
    FlowLaunch fl;
    fl.w0 = flow_h[0];
    fl.rest = reinterpret_cast<const FlowArgs*>(ud + o_flow) + 1;
    fl.n_win = W;
    // ---- one upload, one launch sequence, one download, one synchronisation
    auto reset_maps = [&]() {  // as flow_run: after a failed sequence the maps go back to all 0
        for (const StepWin& w : ws) cudaMemsetAsync(w.t->upkeep->map, 0, sizeof(unsigned long long) * (size_t)w.t->td.lm_cap, cs);
        cudaStreamSynchronize(cs);
    };
    cudaError_t e = hook ? hook->upload(cs) : cudaSuccess;
    if (e == cudaSuccess && !plan.par.empty()) e = lidar_copy_clouds(plan, clouds.data(), lws, cs);
    if (e == cudaSuccess) e = cudaMemcpyAsync(st.up.d, uh, up1, cudaMemcpyHostToDevice, cs);
    if (e == cudaSuccess && !plan.par.empty()) e = launch_lidar_staged(plan, lws, ud + o_lpack, lf, cs);  // the d column
    if (e == cudaSuccess) {
        launch_frame_step_gather(gl, cs);
        e = cudaEventRecord(mb.ev0, cs);
    }
    if (e == cudaSuccess) {
        if (A > 0) launch_adjust_pose(ma, A, cs);
        e = cudaEventRecord(mb.ev1, cs);
    }
    if (e == cudaSuccess) {
        launch_frame_flow(fl, fg, cs);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(st.out.h, od, down1, cudaMemcpyDeviceToHost, cs);
    if (e == cudaSuccess) e = wait_stream(h);
    if (e != cudaSuccess) {
        reset_maps();
        return fail(KBA_ERR_CUDA, who + "frame step: " + cudaGetErrorString(e));
    }
    float ms = 0.f;
    if (A > 0) {
        h->counters.launches_total += 1;
        CU(cudaEventElapsedTime(&ms, mb.ev0, mb.ev1));
    }
    // ---- the verdicts (KeyframeSelector::select({frame}, active keyframes): flow and (pose or time))
    const unsigned char* oh = st.out.h;
    const FrameRes* fr = reinterpret_cast<const FrameRes*>(oh + o_fr);
    std::vector<int> sel;
    for (int v = 0; v < W; ++v) {
        StepWin& w = ws[v];
        const kba_frame_step_request& q = *w.q;
        const FlowRes& f = *reinterpret_cast<const FlowRes*>(oh + w.d_flow);
        const double* pose = w.adjusted ? fr[w.a].pose : q.pose7;
        w.angle = quaternion_diff(pose, reinterpret_cast<const double*>(oh + w.d_pose));
        w.verdict[0] = q.n_meas > 0 && f.usable;
        w.verdict[1] = w.angle > q.critical_quaternion_diff;
        w.verdict[2] = q.stamp - q.stamp_last > q.time_difference_ns;
        w.selected = w.verdict[0] && (w.verdict[1] || w.verdict[2]);
        if (w.selected) sel.push_back(v);
    }
    int64_t up_bytes = (int64_t)up1 + cloud_bytes, down_bytes = (int64_t)down1;
    const bool hooked = hook && hook->due(ws);
    // ---- the push and the creation of the selected windows: one upload of records, one launch sequence, one download
    if (!sel.empty() || hooked) {
        const int S = (int)sel.size();
        std::vector<CompactTrack> ct;
        std::vector<CompactRun> runs;
        std::vector<StoreAppend> app(S);
        std::vector<CreateArgs> cr(S);
        int max_run = 0, max_rows = 0;
        CreateGrid cg;
        Bump dc;
        dc.at = dn2_0;
        for (int j = 0; j < S; ++j) {
            StepWin& w = ws[sel[j]];
            kba_track* t = w.t;
            const kba_frame_step_request& q = *w.q;
            StoreAppend& a = app[j];
            a = append_plan(t, q.kf_new, q.n_meas, q.pose7, q.plane4, false, ct, runs, max_run);
            a.seg = 0; a.n = q.n_meas; a.src = w.src;
            if (w.adjusted) a.pose_src = reinterpret_cast<const double*>(od + o_fr) + (size_t)w.a * (sizeof(FrameRes) / sizeof(double));
            max_rows = std::max(max_rows, q.n_meas);
            CreateArgs c = t->create->a;
            c.td = t->td;
            c.kf_slot = reinterpret_cast<const int*>(ud + w.u_list); c.lm_slot = c.kf_slot + q.n_kf + 1;
            c.n_kf = q.n_kf + 1; c.kf_new = q.n_kf; c.n_new = q.n_new;
            w.d_create = dc.take(24 * (size_t)q.n_new);
            c.pos = reinterpret_cast<double*>(od + w.d_create);
            cr[j] = c;
            t->gen++;
            cg.max_kf = std::max(cg.max_kf, c.n_kf); cg.max_new = std::max(cg.max_new, q.n_new);
            cg.max_init = std::max(cg.max_init, std::max(q.n_new, c.n_kf * t->n_cam));
            cg.max_meas = std::max(cg.max_meas, w.max_meas);
        }
        for (int j = 0; j < S; ++j) cr[j].flags = od + dc.take((size_t)ws[sel[j]].q->n_new, 1);
        Bump u2;
        u2.at = up2_0;
        const size_t o_app = u2.take(sizeof(StoreAppend) * (size_t)S), o_cr = u2.take(sizeof(CreateArgs) * (size_t)S);
        const size_t o_ct = u2.take(sizeof(CompactTrack) * ct.size()), o_run = u2.take(sizeof(CompactRun) * runs.size());
        memcpy(uh + o_app, app.data(), sizeof(StoreAppend) * (size_t)S);
        memcpy(uh + o_cr, cr.data(), sizeof(CreateArgs) * (size_t)S);
        if (!ct.empty()) memcpy(uh + o_ct, ct.data(), sizeof(CompactTrack) * ct.size());
        if (!runs.empty()) memcpy(uh + o_run, runs.data(), sizeof(CompactRun) * runs.size());
        CreateLaunch cl;
        if (S > 0) cl.w0 = cr[0];
        cl.rest = reinterpret_cast<const CreateArgs*>(ud + o_cr) + 1;
        cl.n_win = S;
        if (S > 0) {
            e = cudaMemcpyAsync(st.up.d + up2_0, uh + up2_0, u2.at - up2_0, cudaMemcpyHostToDevice, cs);
            if (e == cudaSuccess) {
                launch_store_push(reinterpret_cast<const CompactTrack*>(ud + o_ct), reinterpret_cast<const CompactRun*>(ud + o_run),
                                  (int)runs.size(), max_run, reinterpret_cast<const StoreAppend*>(ud + o_app), S, max_rows, cols_d, N, cs);
                launch_create(cl, cg, cs);
                e = cudaGetLastError();
            }
        }
        if (e == cudaSuccess && hooked) {
            std::vector<const unsigned char*> created(ws.size(), nullptr);
            for (int j = 0; j < S; ++j) created[sel[j]] = cr[j].flags;
            e = hook->launch(created, cs);
        }
        if (e == cudaSuccess && S > 0) e = cudaMemcpyAsync(st.out.h + dn2_0, od + dn2_0, dc.at - dn2_0, cudaMemcpyDeviceToHost, cs);
        if (e == cudaSuccess) e = wait_stream(h);
        if (e != cudaSuccess) {
            // as create_run: the slot -> request maps go back to all -1
            for (int j = 0; j < S; ++j)
                cudaMemsetAsync(ws[sel[j]].t->create->a.req_of, 0xff, sizeof(int) * (size_t)ws[sel[j]].t->td.lm_cap, cs);
            cudaStreamSynchronize(cs);
            return fail(KBA_ERR_CUDA, who + "frame step push: " + cudaGetErrorString(e));
        }
        up_bytes += (int64_t)(u2.at - up2_0);
        down_bytes += (int64_t)(dc.at - dn2_0);
        for (int j = 0; j < S; ++j) {
            const StepWin& w = ws[sel[j]];
            const size_t m = (size_t)w.q->n_new;
            if (m) {
                memcpy(out[w.i].pos, st.out.h + w.d_create, 24 * m);
                memcpy(out[w.i].flags, st.out.h + (reinterpret_cast<const unsigned char*>(cr[j].flags) - od), m);
            }
        }
    }
    // ---- outputs
    if (n_copy) {
        const float* dep = reinterpret_cast<const float*>(oh + o_dep);
        for (int v : lid_order) {
            const StepWin& w = ws[v];
            float* d = lid[w.i].depth_out;
            if (!d) break;  // the downloaded frames come first
            for (int r : w.cam_rows) d[r] = *dep++;
        }
    }
    const IterRecord* lg = reinterpret_cast<const IterRecord*>(oh + o_log);
    const unsigned char* rj = oh + o_rej;
    for (const StepWin& w : ws) {
        kba_frame_step_out& o = out[w.i];
        const FlowRes& f = *reinterpret_cast<const FlowRes*>(oh + w.d_flow);
        o.n_matched = f.n_matched;
        o.flow_sum = f.flow_sum;
        o.mean_flow_sq = mean_flow_sq(f);
        if (o.match && w.q->n_meas) memcpy(o.match, oh + w.d_match, 4 * (size_t)w.q->n_meas);
        o.angle = w.angle;
        o.usable_flow = w.verdict[0]; o.usable_pose = w.verdict[1]; o.usable_time = w.verdict[2];
        o.selected = w.selected ? 1 : 0;
        if (w.adjusted)
            frame_result(fr[w.a], lg + (size_t)w.a * log_cap, log_cap, rj + fd[w.a].run_off, w.sel_runs, ms, res[w.i]);
    }
    st.counts.h2d = up_bytes;
    st.counts.d2h = down_bytes;
    s.last = &st.counts;
    return KBA_OK;
}

int kba_track_frame_step(kba_track* t, const kba_frame_step_request* req, const kba_options* opt, kba_frame_step_out* out, kba_result* res) {
    static const std::string who = "kba_track_frame_step: ";
    if (!t || !req || !opt || !out || !res) return fail(KBA_ERR_BAD_ARG, who + "null argument");
    return set_frame_step(t->set, false, who, req, false, opt, out, res, nullptr);
}
int kba_track_frame_step_lidar(kba_track* t, const kba_frame_step_request* req, const kba_frame_lidar* lid, const kba_options* opt,
                               kba_frame_step_out* out, kba_result* res) {
    static const std::string who = "kba_track_frame_step_lidar: ";
    if (!t || !req || !lid || !opt || !out || !res) return fail(KBA_ERR_BAD_ARG, who + "null argument");
    return set_frame_step(t->set, false, who, req, false, opt, out, res, lid);
}

// lidar: a _lidar form, which needs lid
static int group_frame_step(kba_track_group* g, const kba_frame_step_request* req, bool per_track, const kba_options* opts,
                            kba_frame_step_out* out, kba_result* res, const std::string& who, bool lidar, const kba_frame_lidar* lid) {
    if (!g || !req || !opts || !out || !res || (lidar && !lid)) return fail(KBA_ERR_BAD_ARG, who + "null argument");
    return set_frame_step(g->set, true, who, req, per_track, opts, out, res, lid);
}
int kba_track_group_frame_step(kba_track_group* g, const kba_frame_step_request* req, const kba_options* opt, kba_frame_step_out* out,
                               kba_result* res) {
    return group_frame_step(g, req, false, opt, out, res, "kba_track_group_frame_step: ", false, nullptr);
}
int kba_track_group_frame_step_opts(kba_track_group* g, const kba_frame_step_request* req, const kba_options* opts,
                                    kba_frame_step_out* out, kba_result* res) {
    return group_frame_step(g, req, true, opts, out, res, "kba_track_group_frame_step_opts: ", false, nullptr);
}
int kba_track_group_frame_step_lidar(kba_track_group* g, const kba_frame_step_request* req, const kba_frame_lidar* lid,
                                     const kba_options* opt, kba_frame_step_out* out, kba_result* res) {
    return group_frame_step(g, req, false, opt, out, res, "kba_track_group_frame_step_lidar: ", true, lid);
}
int kba_track_group_frame_step_lidar_opts(kba_track_group* g, const kba_frame_step_request* req, const kba_frame_lidar* lid,
                                          const kba_options* opts, kba_frame_step_out* out, kba_result* res) {
    return group_frame_step(g, req, true, opts, out, res, "kba_track_group_frame_step_lidar_opts: ", true, lid);
}

// ---------------------------------------------------------------------------------------------------------------------
// limo's camera callback as one store call (include/kba_b200.h, kba_track_camera_step and its group forms; kernels in
// kba_camerastep.cu and those of the two calls it joins).  The frame step's phases (set_frame_step) run with the solve block's
// (KfsCall) hooked in: the solve's lists go up with the frame's, and once the verdicts are known its records go up with the push's,
// k_cs_lists builds the post-push landmark lists right after the creation, and the solve block's first part follows in the same
// launch sequence.  The solve block's rest runs after the frame step's outputs are written.
// ---------------------------------------------------------------------------------------------------------------------
struct CameraStep : StepHook {
    const kba_camera_step_request* req;
    bool group;
    const std::string& who;
    KfsCall& c;
    std::vector<kba_kfsolve_request>& kq;
    std::vector<std::vector<int32_t>>& kf;
    std::vector<char> may_solve;
    int64_t lists_up = 0;                 // the solve's lists in the first upload

    CameraStep(const kba_camera_step_request* r, bool g, const std::string& w, KfsCall& c_, std::vector<kba_kfsolve_request>& kq_,
               std::vector<std::vector<int32_t>>& kf_)
        : req(r), group(g), who(w), c(c_), kq(kq_), kf(kf_) {}

    // after the frame step's checks (kf_slot, n_kf, kf_new and new_slot are valid): the policy, the tags and the solve block's
    // request checks on the candidate bound, then its staging
    int checked() override {
        const int n = (int)c.s.tracks.size();
        for (int i = 0; i < n; ++i) {
            const kba_camera_step_request& q = req[i];
            if (!may_solve[i]) continue;
            const kba_frame_step_request& f = q.step;
            std::string why;
            int rc = KBA_OK;
            if (q.n_cand < 0) { why = "a negative size"; rc = KBA_ERR_BAD_ARG; }
            else if (q.n_cand > 0 && (!q.lm_slot || !q.lm_new)) { why = "null argument"; rc = KBA_ERR_BAD_ARG; }
            std::vector<char> named((size_t)f.n_new, 0);
            for (int j = 0; j < q.n_cand && rc == KBA_OK; ++j) {
                const int k = q.lm_new[j];
                if (k < kCsActive || k >= f.n_new) { why = "candidate tag out of range"; rc = KBA_ERR_BAD_ARG; }
                else if (k >= 0 && (named[k] || q.lm_slot[j] != f.new_slot[k])) {
                    why = "a new landmark's tag named twice or not at its new_slot"; rc = KBA_ERR_BAD_ARG;
                } else if (k >= 0) named[k] = 1;
            }
            if (rc != KBA_OK) return fail(rc, who + track_prefix(group, i) + why);
            kf[i].assign(f.kf_slot, f.kf_slot + f.n_kf);
            kf[i].push_back(f.kf_new);
            kba_kfsolve_request& k = kq[i];
            k.n_kf = f.n_kf + 1; k.n_lm = q.n_cand;
            k.min_connecting = q.min_connecting; k.min_window = q.min_window; k.max_window = q.max_window;
            k.n_trk = q.n_trk; k.kf_slot = kf[i].data(); k.lm_slot = q.lm_slot; k.lm_ground = q.lm_ground; k.trk = q.trk;
            k.classes = q.classes; k.n_class = q.n_class; k.n_outlier = q.n_outlier; k.outlier_slot = q.outlier_slot;
            k.shrubbery_weight = q.shrubbery_weight; k.params = q.params;
            k.max_near = q.max_near; k.max_middle = q.max_middle; k.max_far = q.max_far;
            k.n_depth = q.n_depth; k.depth = q.depth; k.draw = q.draw; k.draw_ctx = q.draw_ctx; k.sel = q.sel;
            if ((rc = c.check(i, 1)) != KBA_OK) return rc;
            KfsWin& w = c.ws.back();
            w.max_meas = std::max(w.max_meas, f.n_meas);  // kf_new, the newest keyframe if the frame is pushed
        }
        if (c.ws.empty()) return KBA_OK;
        const int rc = c.stage();
        if (rc != KBA_OK) return rc;
        for (const KfsWin& w : c.ws)
            if (kq[w.i].n_lm) memcpy(c.st->up.h + w.u_tag, req[w.i].lm_new, 4 * (size_t)kq[w.i].n_lm);
        return KBA_OK;
    }

    // the lists, ahead of the records (which wait for the verdicts)
    cudaError_t upload(cudaStream_t s) override {
        if (c.ws.empty()) return cudaSuccess;
        lists_up = (int64_t)(c.up1 - c.rec_end);
        return cudaMemcpyAsync(c.st->up.d + c.rec_end, c.st->up.h + c.rec_end, c.up1 - c.rec_end, cudaMemcpyHostToDevice, s);
    }

    std::vector<int> step_of;             // c.ws[v]'s window in the frame step

    // the solve rule: the windows that solve are kept, with the keyframes they list now
    bool due(const std::vector<StepWin>& ws) override {
        std::vector<int> win_of(c.s.tracks.size(), -1);
        for (int v = 0; v < (int)ws.size(); ++v) win_of[ws[v].i] = v;
        std::vector<KfsWin> keep;
        for (KfsWin& w : c.ws) {
            const StepWin& sw = ws[win_of[w.i]];
            if (req[w.i].solve == KBA_STEP_SOLVE_IF_SELECTED && !sw.selected) continue;
            w.kn = sw.q->n_kf + (sw.selected ? 1 : 0);
            keep.push_back(w);
            step_of.push_back(win_of[w.i]);
        }
        c.ws.swap(keep);
        c.W = (int)c.ws.size();
        return c.W > 0;
    }

    cudaError_t launch(const std::vector<const unsigned char*>& created, cudaStream_t s) override {
        std::vector<const unsigned char*> cr(c.ws.size());
        for (size_t v = 0; v < c.ws.size(); ++v) cr[v] = created[step_of[v]];
        if (c.records(&cr) != KBA_OK) return cudaErrorUnknown;
        cudaError_t e = cudaMemcpyAsync(c.st->up.d, c.st->up.h, c.rec_end, cudaMemcpyHostToDevice, s);
        if (e == cudaSuccess) e = c.launch_first();
        if (e == cudaSuccess) e = cudaMemcpyAsync(c.st->out.h, c.st->out.d, c.down1, cudaMemcpyDeviceToHost, s);
        return e;
    }
};

static int set_camera_step(TrackSet& s, bool group, const std::string& who, const kba_camera_step_request* req, const kba_frame_lidar* lid,
                           bool per_track, const kba_options* opts_adjust, const kba_options* opts_solve, kba_camera_step_out* out,
                           kba_result* res_adjust, kba_result* res_solve) {
    const int n = (int)s.tracks.size();
    std::vector<kba_frame_step_request> fq(n);
    std::vector<kba_frame_step_out> fo(n);
    std::vector<kba_kfsolve_request> kq(n);
    std::vector<kba_kfsolve_out> ko(n);
    std::vector<std::vector<int32_t>> kf(n);
    KfsCall c(s, group, who, kq.data(), per_track, opts_solve, ko.data(), res_solve);
    c.cs = true;
    CameraStep cs(req, group, who, c, kq, kf);
    cs.may_solve.assign(n, 0);
    for (int i = 0; i < n; ++i) {
        fq[i] = req[i].step; fo[i] = out[i].step; ko[i] = out[i].solve;
        if (group && req[i].step.n_kf == 0) continue;
        if (req[i].solve > KBA_STEP_SOLVE_IF_SELECTED) return fail(KBA_ERR_BAD_ARG, who + track_prefix(group, i) + "unknown solve policy");
        if (req[i].solve != KBA_STEP_SOLVE_NEVER) {
            if (!out[i].lm_index && req[i].n_cand > 0) return fail(KBA_ERR_BAD_ARG, who + track_prefix(group, i) + "null argument");
            cs.may_solve[i] = 1;
        }
    }
    int rc = c.check_options([&](int i) { return cs.may_solve[i] != 0; });
    if (rc != KBA_OK) return rc;
    rc = set_frame_step(s, group, who, fq.data(), per_track, opts_adjust, fo.data(), res_adjust, lid, &cs);
    if (rc != KBA_OK) return rc;
    // the frame step is done: its outputs are the caller's whatever the solve block does
    Transfer sum = *s.last;
    sum.h2d += cs.lists_up;
    for (int i = 0; i < n; ++i) {
        if (group && req[i].step.n_kf == 0) continue;
        out[i].step = fo[i];
        out[i].solved = 0;
    }
    if (c.W == 0) {  // no track solves
        for (int i = 0; i < n; ++i) idle_result(res_solve[i]);
        if (c.st) {
            c.st->counts = sum;
            s.last = &c.st->counts;
        }
        return KBA_OK;
    }
    c.sum.h2d = sum.h2d + (int64_t)c.rec_end; c.sum.d2h = sum.d2h + (int64_t)c.down1;
    rc = c.rest();
    if (rc != KBA_OK) return rc;
    for (const KfsWin& w : c.ws) {
        kba_camera_step_out& o = out[w.i];
        o.solve = ko[w.i];  // the ranking's counts
        o.solved = 1;
        o.n_lm = w.ln;
        if (req[w.i].n_cand) memcpy(o.lm_index, c.st->out.h + w.d_index, 4 * (size_t)req[w.i].n_cand);
    }
    return KBA_OK;
}

int kba_track_camera_step(kba_track* t, const kba_camera_step_request* req, const kba_frame_lidar* lid, const kba_options* opt_adjust,
                          const kba_options* opt_solve, kba_camera_step_out* out, kba_result* res_adjust, kba_result* res_solve) {
    static const std::string who = "kba_track_camera_step: ";
    if (!t || !req || !opt_adjust || !opt_solve || !out || !res_adjust || !res_solve) return fail(KBA_ERR_BAD_ARG, who + "null argument");
    return set_camera_step(t->set, false, who, req, lid, false, opt_adjust, opt_solve, out, res_adjust, res_solve);
}

static int group_camera_step(kba_track_group* g, const kba_camera_step_request* req, const kba_frame_lidar* lid, bool per_track,
                             const kba_options* opts_adjust, const kba_options* opts_solve, kba_camera_step_out* out, kba_result* res_adjust,
                             kba_result* res_solve, const std::string& who) {
    if (!g || !req || !opts_adjust || !opts_solve || !out || !res_adjust || !res_solve) return fail(KBA_ERR_BAD_ARG, who + "null argument");
    return set_camera_step(g->set, true, who, req, lid, per_track, opts_adjust, opts_solve, out, res_adjust, res_solve);
}
int kba_track_group_camera_step(kba_track_group* g, const kba_camera_step_request* req, const kba_frame_lidar* lid, const kba_options* opt_adjust,
                                const kba_options* opt_solve, kba_camera_step_out* out, kba_result* res_adjust, kba_result* res_solve) {
    return group_camera_step(g, req, lid, false, opt_adjust, opt_solve, out, res_adjust, res_solve, "kba_track_group_camera_step: ");
}
int kba_track_group_camera_step_opts(kba_track_group* g, const kba_camera_step_request* req, const kba_frame_lidar* lid,
                                     const kba_options* opts_adjust, const kba_options* opts_solve, kba_camera_step_out* out,
                                     kba_result* res_adjust, kba_result* res_solve) {
    return group_camera_step(g, req, lid, true, opts_adjust, opts_solve, out, res_adjust, res_solve, "kba_track_group_camera_step_opts: ");
}

// ---------------------------------------------------------------------------------------------------------------------
// snapshots of the stored window (include/kba_b200.h, kba_track_save / kba_track_load / kba_track_clone / kba_track_group_save;
// kernels in kba_store.cu).  A snapshot is assembled as an image in device memory: the host uploads each image's head (header,
// cameras, keyframe lists), k_copy_spans copies the heads, poses, planes and landmark values into the images, k_arena_compact the
// live keyframes' runs.  A load goes the other way from an image: k_store_append writes the runs and the keyframe layout,
// k_copy_spans the poses, planes and landmark values.  A single save is a one-track call of store_call.
// ---------------------------------------------------------------------------------------------------------------------
static int64_t align8(int64_t b) { return (b + 7) & ~(int64_t)7; }

// byte offsets of a snapshot's arrays, from its counts (n_cam, K live keyframes, M entries, L landmark slots); col is the bytes of
// one measurement column
struct SnapLayout {
    int64_t cam_intr = 0, cam_pose = 0, kf_slot = 0, kf_count = 0, kf_pose = 0, kf_plane = 0, meas = 0, col = 0, lm_pos = 0,
            lm_weight = 0, end = 0;
    SnapLayout() = default;
    SnapLayout(int64_t n_cam, int64_t K, int64_t M, int64_t L) {
        cam_intr = sizeof(kba_snapshot_header); cam_pose = cam_intr + 24 * n_cam;
        kf_slot = cam_pose + 56 * n_cam; kf_count = kf_slot + align8(4 * K); kf_pose = kf_count + align8(4 * K);
        kf_plane = kf_pose + 56 * K; meas = kf_plane + 32 * K; col = align8(4 * M);
        lm_pos = meas + 5 * col; lm_weight = lm_pos + 24 * L; end = lm_weight + 8 * L;
    }
    void sections(kba_snapshot_header& hd) const {
        hd.cam_offset = cam_intr; hd.cam_bytes = kf_slot - cam_intr; hd.kf_offset = kf_slot; hd.kf_bytes = meas - kf_slot;
        hd.meas_offset = meas; hd.meas_bytes = lm_pos - meas; hd.lm_offset = lm_pos; hd.lm_bytes = end - lm_pos;
    }
};

// what a snapshot of t holds: its live keyframe slots (ascending), their counts, and the layout
struct SnapContent {
    std::vector<int> slot, cnt;
    int M = 0, L = 0;
    SnapLayout lay;
};
static SnapContent snap_content(const kba_track* t) {
    SnapContent c;
    for (int k = 0; k < t->td.kf_cap; ++k)
        if (t->kf_live[k]) { c.slot.push_back(k); c.cnt.push_back(t->m_cnt[k]); c.M += t->m_cnt[k]; }
    c.L = t->td.lm_cap;
    c.lay = SnapLayout(t->n_cam, (int64_t)c.slot.size(), c.M, c.L);
    return c;
}

static kba_snapshot_header snap_header(const kba_track* t, const SnapContent& c) {
    kba_snapshot_header hd;
    memset(&hd, 0, sizeof(hd));
    hd.magic = KBA_SNAPSHOT_MAGIC; hd.format_version = KBA_SNAPSHOT_VERSION; hd.writer_version = KBA_VERSION_MAJOR * 100 + KBA_VERSION_MINOR;
    hd.n_cam = t->n_cam; hd.caps = t->caps; hd.n_keyframes = (int32_t)c.slot.size(); hd.n_entries = c.M; hd.lm_cap = c.L;
    c.lay.sections(hd);
    return hd;
}

// the staging of a track's snapshots at its capacities: every keyframe slot live, a full arena
static SnapLayout snap_capacity(const kba_track* t) { return SnapLayout(t->n_cam, t->td.kf_cap, t->td.m_cap, t->td.lm_cap); }
static size_t snap_spans(int64_t K) { return 8 + 2 * (size_t)K; }  // head, 5 column pads, positions, weights; pose and plane per keyframe
static size_t save_records(int W, size_t kfs, size_t spans) {
    return align16(sizeof(CompactTrack) * W) + align16(sizeof(CompactRun) * kfs) + align16(sizeof(CopySpan) * spans) + 16;
}
static size_t load_records(int64_t K) { return align16(sizeof(StoreAppend) * (size_t)K) + align16(sizeof(CopySpan) * snap_spans(K)); }

static const unsigned* words(const void* p) { return reinterpret_cast<const unsigned*>(p); }

struct SaveReq {
    kba_track* t = nullptr;
    void* buf = nullptr;
    int64_t bytes = 0;
    SnapContent c;
};

// the images of W saves in st.out.d, image w at img[w]: one upload of the records and heads, k_copy_spans, k_arena_compact (no
// synchronisation).  The upload: CompactTrack [W] | runs | spans | 16 zero bytes (the columns' padding) | the heads.
static int snap_gather(kba_handle* h, StoreStage& st, int W, const SaveReq* r, std::vector<int64_t>& img, int64_t& up) {
    CU(cudaSetDevice(h->device));
    cudaStream_t s = h->stream;
    size_t n_run = 0, n_span = 0;
    int64_t heads = 0;
    img.assign(W, 0);
    for (int w = 0; w < W; ++w) {
        for (int n : r[w].c.cnt) n_run += n > 0;
        n_span += snap_spans((int64_t)r[w].c.slot.size());
        heads += r[w].c.lay.kf_pose;
        if (w > 0) img[w] = img[w - 1] + r[w - 1].c.lay.end;  // every size is a multiple of 8
    }
    const size_t o_run = align16(sizeof(CompactTrack) * W), o_span = o_run + align16(sizeof(CompactRun) * n_run);
    const size_t o_zero = o_span + align16(sizeof(CopySpan) * n_span), o_head = o_zero + 16;
    unsigned char* hb = st.up.h;
    const unsigned char* ub = st.up.d;
    unsigned char* ob = st.out.d;
    memset(hb + o_zero, 0, 16 + (size_t)heads);
    CompactTrack* ct = reinterpret_cast<CompactTrack*>(hb);
    CompactRun* runs = reinterpret_cast<CompactRun*>(hb + o_run);
    CopySpan* spans = reinterpret_cast<CopySpan*>(hb + o_span);
    size_t nr = 0, ns = 0;
    int max_run = 0;
    long long max_words = 0;
    auto span = [&](const void* src, void* dst, long long n) {
        spans[ns].src = words(src); spans[ns].dst = reinterpret_cast<unsigned*>(dst); spans[ns].n = n; ++ns;
        max_words = std::max(max_words, n);
    };
    int64_t o_h = (int64_t)o_head;
    for (int w = 0; w < W; ++w) {
        const kba_track* t = r[w].t;
        const SnapContent& c = r[w].c;
        const SnapLayout& L = c.lay;
        const int K = (int)c.slot.size();
        unsigned char* hd = hb + o_h;  // the head: header | cameras | slots | counts (padding zero)
        const kba_snapshot_header head = snap_header(t, c);
        memcpy(hd, &head, sizeof(head));
        memcpy(hd + L.cam_intr, t->cam_intr.data(), 24 * (size_t)t->n_cam);
        memcpy(hd + L.cam_pose, t->cam_pose.data(), 56 * (size_t)t->n_cam);
        memcpy(hd + L.kf_slot, c.slot.data(), 4 * (size_t)K);
        memcpy(hd + L.kf_count, c.cnt.data(), 4 * (size_t)K);
        unsigned char* im = ob + img[w];
        span(ub + o_h, im, L.kf_pose / 4);
        for (int i = 0; i < K; ++i) {
            span(t->td.kf_pose + 7 * (size_t)c.slot[i], im + L.kf_pose + 56 * (int64_t)i, 14);
            span(t->td.kf_plane + 4 * (size_t)c.slot[i], im + L.kf_plane + 32 * (int64_t)i, 8);
        }
        for (int q = 0; q < 5; ++q)  // an odd column ends in a word of padding
            span(ub + o_zero, im + L.meas + q * L.col + 4 * (int64_t)c.M, (L.col - 4 * (int64_t)c.M) / 4);
        span(t->td.lm_pos, im + L.lm_pos, 6 * (long long)c.L);
        span(t->td.lm_weight, im + L.lm_weight, 2 * (long long)c.L);
        CompactTrack& x = ct[w];
        x = CompactTrack{};
        for (int j = 0; j < 2; ++j) x.src[j] = words(t->arena_i[t->arena_cur][j]);
        for (int j = 0; j < 3; ++j) x.src[2 + j] = words(t->arena_f[t->arena_cur][j]);
        for (int q = 0; q < 5; ++q) x.dst[q] = reinterpret_cast<unsigned*>(im + L.meas + q * L.col);
        for (int i = 0, dst = 0; i < K; dst += c.cnt[i], ++i) {
            if (c.cnt[i] == 0) continue;
            runs[nr++] = CompactRun{w, c.slot[i], t->m_off[c.slot[i]], dst, c.cnt[i], 0};
            max_run = std::max(max_run, c.cnt[i]);
        }
        o_h += L.kf_pose;
    }
    up = o_h;
    CU(cudaMemcpyAsync(st.up.d, hb, (size_t)up, cudaMemcpyHostToDevice, s));
    launch_copy_spans(reinterpret_cast<const CopySpan*>(ub + o_span), (int)ns, max_words, s);
    launch_store_push(reinterpret_cast<const CompactTrack*>(ub), reinterpret_cast<const CompactRun*>(ub + o_run), (int)nr, max_run,
                      nullptr, 0, 0, nullptr, 0, s);
    CU(cudaGetLastError());
    return KBA_OK;
}

// W checked saves: the images, one download, one synchronisation, each image into its caller's buffer
static int save_run(kba_handle* h, StoreStage& st, int W, const SaveReq* r) {
    std::vector<int64_t> img;
    int64_t up = 0;
    int rc = snap_gather(h, st, W, r, img, up);
    if (rc != KBA_OK) return rc;
    const int64_t total = img[W - 1] + r[W - 1].c.lay.end;
    CU(cudaMemcpyAsync(st.out.h, st.out.d, (size_t)total, cudaMemcpyDeviceToHost, h->stream));
    CU(wait_stream(h));
    for (int w = 0; w < W; ++w) memcpy(r[w].buf, st.out.h + img[w], (size_t)r[w].c.lay.end);
    st.counts.h2d = up;
    st.counts.d2h = total;
    return KBA_OK;
}

// the staging of the snapshot call for tracks ts[0..n) at their capacities; a single track's also holds a load's records and image
static void snap_stage_bytes(int n, kba_track* const* ts, size_t& up, size_t& down) {
    size_t kfs = 0, spans = 0, heads = 0, images = 0;
    for (int i = 0; i < n; ++i) {
        const SnapLayout c = snap_capacity(ts[i]);
        kfs += (size_t)ts[i]->td.kf_cap; spans += snap_spans(ts[i]->td.kf_cap); heads += (size_t)c.kf_pose; images += (size_t)c.end;
    }
    up = save_records(n, kfs, spans) + heads;
    if (n == 1) up = std::max(up, load_records(ts[0]->td.kf_cap) + images);
    down = images;
}

static int snap_stage(TrackSet& s, const std::string& who, StoreStage*& st) {
    std::unique_ptr<StoreStage>& p = s.stage[kSnapshotCall];
    if (!p) {
        size_t up = 0, down = 0;
        snap_stage_bytes((int)s.tracks.size(), s.tracks.data(), up, down);
        std::unique_ptr<StoreStage> fresh(new StoreStage());
        if (fresh->alloc(up, down)) return fail(KBA_ERR_CUDA, who + "out of memory for the snapshot staging");
        p = std::move(fresh);
    }
    st = p.get();
    return KBA_OK;
}

struct SnapshotWrite {
    void* buf;
    int64_t bytes;
};
struct Save : WriteCall {
    using Request = SnapshotWrite;
    using Req = SaveReq;
    static constexpr StoreCall slot = kSnapshotCall;
    static constexpr const char* staging = "snapshot";
    static bool sits_out(const Request& q) { return q.buf == nullptr; }
    static Req make(kba_track* t, const Request& q, Out*) {
        SaveReq r;
        r.t = t; r.buf = q.buf; r.bytes = q.bytes; r.c = snap_content(t);
        return r;
    }
    static int check(Req& r, std::string& why) {
        if (!r.buf) { why = "null buffer"; return KBA_ERR_BAD_ARG; }
        if (r.bytes < r.c.lay.end) {
            why = "a buffer of " + std::to_string(r.bytes) + " bytes, the snapshot has " + std::to_string(r.c.lay.end);
            return KBA_ERR_CAPACITY;
        }
        return KBA_OK;
    }
    static void capacity(int n, kba_track* const* ts, size_t& up, size_t& down) { snap_stage_bytes(n, ts, up, down); }
    static int run(kba_handle* h, StoreStage& st, int W, Req* r, int&, std::string&) { return save_run(h, st, W, r); }
};

// every structural field of a snapshot from outside the program, before anything is allocated: hd, the slots, the counts
static int snap_check(const unsigned char* b, int64_t bytes, kba_snapshot_header& hd, std::vector<int>& slot, std::vector<int>& cnt,
                      std::string& why) {
    why = "";
    if (bytes < (int64_t)sizeof(hd)) { why = "truncated buffer: shorter than the header"; return KBA_ERR_BAD_ARG; }
    memcpy(&hd, b, sizeof(hd));
    if (hd.magic != KBA_SNAPSHOT_MAGIC) why = "magic";
    else if (hd.format_version != KBA_SNAPSHOT_VERSION) why = "format_version " + std::to_string(hd.format_version) + " (this library reads 1)";
    else if (hd.reserved_ != 0) why = "reserved_";
    else if (hd.n_cam < 1 || (int64_t)hd.n_cam > bytes / 80) why = "n_cam";
    else if (hd.lm_cap < 1 || hd.lm_cap != hd.caps.max_landmarks) why = "lm_cap (caps.max_landmarks)";
    else if (hd.n_keyframes < 0 || hd.n_keyframes > hd.caps.max_keyframes) why = "n_keyframes";
    else if (hd.n_entries < 0 || hd.n_entries > hd.caps.max_measurements) why = "n_entries";
    if (!why.empty()) { why = "snapshot header: " + why; return KBA_ERR_BAD_ARG; }
    const SnapLayout L(hd.n_cam, hd.n_keyframes, hd.n_entries, hd.lm_cap);
    kba_snapshot_header want = hd;
    L.sections(want);
    const char* names[] = {"cam_offset", "cam_bytes", "kf_offset", "kf_bytes", "meas_offset", "meas_bytes", "lm_offset", "lm_bytes"};
    const int64_t got[] = {hd.cam_offset, hd.cam_bytes, hd.kf_offset, hd.kf_bytes, hd.meas_offset, hd.meas_bytes, hd.lm_offset, hd.lm_bytes};
    const int64_t exp[] = {want.cam_offset, want.cam_bytes, want.kf_offset, want.kf_bytes, want.meas_offset, want.meas_bytes,
                           want.lm_offset, want.lm_bytes};
    for (int i = 0; i < 8; ++i)
        if (got[i] != exp[i]) {
            why = std::string("snapshot header: ") + names[i] + " " + std::to_string(got[i]) + ", the counts give " + std::to_string(exp[i]);
            return KBA_ERR_BAD_ARG;
        }
    if (L.end > bytes) {
        why = "truncated buffer: " + std::to_string(bytes) + " bytes, the sections end at " + std::to_string(L.end);
        return KBA_ERR_BAD_ARG;
    }
    const int K = hd.n_keyframes, M = hd.n_entries;
    slot.resize(K); cnt.resize(K);
    memcpy(slot.data(), b + L.kf_slot, 4 * (size_t)K);
    memcpy(cnt.data(), b + L.kf_count, 4 * (size_t)K);
    int64_t sum = 0;
    for (int i = 0; i < K; ++i) {
        if (slot[i] < 0 || slot[i] >= hd.caps.max_keyframes || (i > 0 && slot[i] <= slot[i - 1])) {
            why = "keyframe slot " + std::to_string(i) + ": not ascending in [0, caps.max_keyframes)"; return KBA_ERR_BAD_ARG;
        }
        if (cnt[i] < 0) { why = "keyframe count " + std::to_string(i) + " negative"; return KBA_ERR_BAD_ARG; }
        sum += cnt[i];
    }
    if (sum != M) { why = "keyframe counts sum to " + std::to_string(sum) + ", n_entries is " + std::to_string(M); return KBA_ERR_BAD_ARG; }
    std::vector<int32_t> col(M);
    memcpy(col.data(), b + L.meas, 4 * (size_t)M);
    for (int i = 0; i < M; ++i)
        if (col[i] < 0 || col[i] >= hd.lm_cap) { why = "measurement " + std::to_string(i) + ": landmark slot out of [0, lm_cap)"; return KBA_ERR_BAD_ARG; }
    memcpy(col.data(), b + L.meas + L.col, 4 * (size_t)M);
    for (int i = 0; i < M; ++i)
        if (col[i] < 0 || col[i] >= hd.n_cam) { why = "measurement " + std::to_string(i) + ": camera out of [0, n_cam)"; return KBA_ERR_BAD_ARG; }
    return KBA_OK;
}

// caps given at a load or clone must hold the snapshot's content
static int snap_caps_check(const kba_track_caps* caps, const std::vector<int>& slot, int M, int L, std::string& why) {
    if (!caps) return KBA_OK;
    if (!slot.empty() && caps->max_keyframes <= slot.back()) why = "caps.max_keyframes does not hold keyframe slot " + std::to_string(slot.back());
    else if (caps->max_landmarks < L) why = "caps.max_landmarks below the snapshot's " + std::to_string(L) + " landmark slots";
    else if (caps->max_measurements < M) why = "caps.max_measurements below the snapshot's " + std::to_string(M) + " arena entries";
    return why.empty() ? KBA_OK : KBA_ERR_CAPACITY;
}

// a new track on h with caps and cameras, its store written from a snapshot image: host_img (uploaded with the records) or, when
// null, dev_img in device memory of h's device, which h's stream may read.  slot, cnt: the image's live keyframes; L its slots.
static int snap_create(kba_handle* h, const kba_track_caps& caps, int n_cam, const double* intr, const double* pose, const std::vector<int>& slot,
                       const std::vector<int>& cnt, int L, const unsigned char* host_img, const unsigned char* dev_img, const std::string& who,
                       kba_track** out) {
    const int K = (int)slot.size();
    int M = 0;
    for (int n : cnt) M += n;
    const SnapLayout lay(n_cam, K, M, L);
    kba_track* t = nullptr;
    int rc = kba_track_create(h, &caps, n_cam, intr, pose, &t);
    if (rc != KBA_OK) return rc;
    std::unique_ptr<kba_track, void (*)(kba_track*)> guard(t, kba_track_destroy);
    StoreStage* st = nullptr;
    rc = snap_stage(t->set, who, st);
    if (rc != KBA_OK) return rc;
    cudaStream_t s = h->stream;
    const size_t o_span = align16(sizeof(StoreAppend) * (size_t)K), o_img = load_records(K);
    unsigned char* hb = st->up.h;
    const unsigned char* ub = st->up.d;
    if (host_img) { memcpy(hb + o_img, host_img, (size_t)lay.end); dev_img = ub + o_img; }
    StoreAppend* app = reinterpret_cast<StoreAppend*>(hb);
    CopySpan* spans = reinterpret_cast<CopySpan*>(hb + o_span);
    TrackDev& td = t->td;
    int ns = 0, max_rows = 0;
    long long max_words = 0;
    auto span = [&](const void* src, void* dst, long long n) {
        spans[ns].src = words(src); spans[ns].dst = reinterpret_cast<unsigned*>(dst); spans[ns].n = n; ++ns;
        max_words = std::max(max_words, n);
    };
    for (int i = 0, off = 0; i < K; off += cnt[i], ++i) {
        StoreAppend a;  // the record's pose and plane are 0: the spans below write the snapshot's after it
        a.col[0] = (unsigned*)td.m_lm; a.col[1] = (unsigned*)td.m_cam; a.col[2] = (unsigned*)td.m_u; a.col[3] = (unsigned*)td.m_v;
        a.col[4] = (unsigned*)td.m_d;
        a.m_off = td.m_off; a.m_cnt = td.m_cnt; a.kf_pose = td.kf_pose; a.kf_plane = td.kf_plane;
        a.slot = slot[i]; a.off = off; a.cnt = cnt[i]; a.seg = 0; a.n = cnt[i]; a.src = off; a.cam_zero = 0;
        app[i] = a;
        max_rows = std::max(max_rows, cnt[i]);
        span(dev_img + lay.kf_pose + 56 * (int64_t)i, td.kf_pose + 7 * (size_t)slot[i], 14);
        span(dev_img + lay.kf_plane + 32 * (int64_t)i, td.kf_plane + 4 * (size_t)slot[i], 8);
        t->m_off[slot[i]] = off; t->m_cnt[slot[i]] = cnt[i]; t->kf_live[slot[i]] = 1;
    }
    span(dev_img + lay.lm_pos, td.lm_pos, 6 * (long long)L);
    span(dev_img + lay.lm_weight, td.lm_weight, 2 * (long long)L);
    const size_t up = host_img ? o_img + (size_t)lay.end : o_img;
    CU(cudaMemcpyAsync(st->up.d, hb, up, cudaMemcpyHostToDevice, s));
    launch_store_push(nullptr, nullptr, 0, 0, reinterpret_cast<const StoreAppend*>(ub), K, max_rows, words(dev_img + lay.meas),
                      (int)(lay.col / 4), s);
    launch_copy_spans(reinterpret_cast<const CopySpan*>(ub + o_span), ns, max_words, s);
    CU(cudaGetLastError());
    CU(wait_stream(h));
    t->arena_used = M;
    st->counts.h2d = (int64_t)up; st->counts.d2h = 0;
    t->set.last = &st->counts;
    *out = guard.release();
    return KBA_OK;
}

int kba_track_snapshot_size(const kba_track* t, int64_t* bytes) {
    if (!t || !bytes) return fail(KBA_ERR_BAD_ARG, "kba_track_snapshot_size: null argument");
    *bytes = snap_content(t).lay.end;
    return KBA_OK;
}

int kba_track_group_snapshot_sizes(kba_track_group* g, int64_t* bytes) {
    if (!g || !bytes) return fail(KBA_ERR_BAD_ARG, "kba_track_group_snapshot_sizes: null argument");
    for (size_t i = 0; i < g->set.tracks.size(); ++i) bytes[i] = snap_content(g->set.tracks[i]).lay.end;
    return KBA_OK;
}

int kba_track_save(kba_track* t, void* buf, int64_t bytes) {
    static const std::string who = "kba_track_save: ";
    if (!t) return fail(KBA_ERR_BAD_ARG, who + "null argument");
    const SnapshotWrite q = {buf, bytes};
    return store_call<Save>(t->set, false, who, &q, nullptr);
}

int kba_track_group_save(kba_track_group* g, void* const* bufs, const int64_t* bytes) {
    static const std::string who = "kba_track_group_save: ";
    if (!g || !bufs || !bytes) return fail(KBA_ERR_BAD_ARG, who + "null argument");
    std::vector<SnapshotWrite> q(g->set.tracks.size());
    for (size_t i = 0; i < q.size(); ++i) q[i] = SnapshotWrite{bufs[i], bytes[i]};
    return store_call<Save>(g->set, true, who, q.data(), nullptr);
}

int kba_track_load(kba_handle* h, const void* buf, int64_t bytes, const kba_track_caps* caps, kba_track** out) {
    static const std::string who = "kba_track_load: ";
    if (!h || !buf || !out) return fail(KBA_ERR_BAD_ARG, who + "null argument");
    const unsigned char* b = static_cast<const unsigned char*>(buf);
    kba_snapshot_header hd;
    std::vector<int> slot, cnt;
    std::string why;
    int rc = snap_check(b, bytes, hd, slot, cnt, why);
    if (rc == KBA_OK) rc = snap_caps_check(caps, slot, hd.n_entries, hd.lm_cap, why);
    if (rc != KBA_OK) return fail(rc, who + why);
    const SnapLayout L(hd.n_cam, hd.n_keyframes, hd.n_entries, hd.lm_cap);
    std::vector<double> intr(3 * (size_t)hd.n_cam), pose(7 * (size_t)hd.n_cam);
    memcpy(intr.data(), b + L.cam_intr, 8 * intr.size());
    memcpy(pose.data(), b + L.cam_pose, 8 * pose.size());
    return snap_create(h, caps ? *caps : hd.caps, hd.n_cam, intr.data(), pose.data(), slot, cnt, hd.lm_cap, b, nullptr, who, out);
}

int kba_track_clone(kba_track* src, kba_handle* h, const kba_track_caps* caps, kba_track** out) {
    static const std::string who = "kba_track_clone: ";
    if (!src || !h || !out) return fail(KBA_ERR_BAD_ARG, who + "null argument");
    SaveReq r;
    r.t = src; r.c = snap_content(src);
    std::string why;
    const int rc = snap_caps_check(caps, r.c.slot, r.c.M, r.c.L, why);
    if (rc != KBA_OK) return fail(rc, who + why);
    kba_handle* hs = src->set.h;
    if (hs->device != h->device) {  // across devices: a save and a load
        std::vector<unsigned char> buf((size_t)r.c.lay.end);
        const int rs = kba_track_save(src, buf.data(), (int64_t)buf.size());
        if (rs != KBA_OK) return rs;
        return kba_track_load(h, buf.data(), (int64_t)buf.size(), caps, out);
    }
    StoreStage* st = nullptr;
    int rs = snap_stage(src->set, who, st);
    if (rs != KBA_OK) return rs;
    std::vector<int64_t> img;
    int64_t up = 0;
    rs = snap_gather(hs, *st, 1, &r, img, up);
    if (rs != KBA_OK) return rs;
    st->counts.h2d = up; st->counts.d2h = 0;
    src->set.last = &st->counts;
    if (hs->stream != h->stream) {  // h's stream reads the image after src's stream wrote it
        cudaEvent_t ev = nullptr;
        CU(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
        cudaError_t e = cudaEventRecord(ev, hs->stream);
        if (e == cudaSuccess) e = cudaStreamWaitEvent(h->stream, ev, 0);
        cudaEventDestroy(ev);
        if (e != cudaSuccess) return fail(KBA_ERR_CUDA, who + cudaGetErrorString(e));
    }
    return snap_create(h, caps ? *caps : src->caps, src->n_cam, src->cam_intr.data(), src->cam_pose.data(), r.c.slot, r.c.cnt, r.c.L,
                       nullptr, st->out.d, who, out);
}

}  // extern "C"
