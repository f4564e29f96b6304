// kba_kernels.h -- host-visible launch interface of kba_kernels.cu
#pragma once
#include <vector>

#include <cuda_runtime.h>

#include "kba_b200.h"
#include "kba_device.cuh"

namespace kba {

// KBA_LAUNCH_CHECK=1 (debugging): every kernel launch is followed by cudaGetLastError() and a failing one is named on stderr.
// Off by default: kba_batch_solve checks once per solve.
int launch_check_enabled();
void launch_check_report(const char* kernel, cudaError_t e);
#define LCHK(name)                                                                       \
    do {                                                                                 \
        if (kba::launch_check_enabled()) {                                               \
            const cudaError_t lchk_e_ = cudaGetLastError();                              \
            if (lchk_e_ != cudaSuccess) kba::launch_check_report(name, lchk_e_);         \
        }                                                                                \
    } while (0)

struct Counters {
    long long launches_total = 0;
    long long launches_jacobian = 0, launches_prep = 0, launches_schur = 0, launches_solve = 0, launches_backsub = 0,
              launches_cost = 0, launches_update = 0, launches_trim = 0;
    double ms_jacobian = 0.0;
    long long jacobian_obs = 0;
};

// cross-rank reduction hook of the sharded solve: all-reduce of `count` doubles on stream s (op 0 = sum, 1 = max; send == recv
// allowed); returns 0 on success.  Implemented in kba_shard.cu over NCCL (one process per GPU) and in process (several handles
// of one process on one device).
struct Exchange {
    int (*allreduce)(void* user, const double* send, double* recv, long long count, int op, cudaStream_t s) = nullptr;
    void (*abort)(void* user) = nullptr;  // this rank leaves the collective on an error: release the ranks waiting for it
    void* user = nullptr;
    int rank = 0, world = 1;
    bool capturable = true;               // the all-reduce may be captured into a CUDA graph (no host step at enqueue time)
};

struct LaunchCfg {
    Plan plan;                // what the batch runs (kba_plan.h); BatchDev holds the fields the kernels read
    Knobs knobs;              // read when the batch was created
    int sm_count = 132;       // SMs of the device the batch runs on (strided_grid: waves of CTAs)
    int max_rank = 0;         // largest observation rank in the batch (multi-camera rigs)
    bool time_jacobian = false;
    cudaEvent_t* ev_pool = nullptr;  // pairs of events bracketing each residual/Jacobian launch
    int ev_cap = 0;
    int* ev_used = nullptr;
    Exchange xchg;  // used when BatchDev::sharded
    struct WinDescHost { int nr_cap = 0, n_kf = 0; } shard_win;  // shapes of the sharded window (host copy)
};

// window arrays exactly as the caller passes them (landmark-major CSR in the caller's landmark order), batch-flat on the
// device: input of the packing kernels (kba_pack.cu)
struct PackRaw {
    const int* lm_ptr = nullptr;      // [tot_lm + n_win]
    const int* obs_kf = nullptr;      // [tot_obs]
    const int* obs_cam = nullptr;
    const float* obs_u = nullptr, *obs_v = nullptr, *obs_d = nullptr;
    const double* lm_pos = nullptr;   // [tot_lm*3]
    const double* lm_weight = nullptr;
    const int* gp_lm = nullptr;       // [tot_gp] caller landmark index
    int* lm_inv = nullptr;            // [tot_lm] scratch: caller index -> sorted position
    int* obs_orig = nullptr;          // [tot_obs] optional: sorted slot -> caller observation index
};
// device-resident track store of a persistent sliding window (kba_track_*, include/kba_b200.h): keyframe poses / planes,
// the measurements of every pushed keyframe in one arena, landmark positions / weights by caller-assigned slot
struct TrackDev {
    double* kf_pose = nullptr;   // [kf_cap*7]
    double* kf_plane = nullptr;  // [kf_cap*4]
    int* m_off = nullptr;        // [kf_cap] first measurement of the keyframe in the arena
    int* m_cnt = nullptr;        // [kf_cap]
    int* m_lm = nullptr;         // [m_cap] landmark slot
    int* m_cam = nullptr;        // [m_cap] camera index
    float* m_u = nullptr, *m_v = nullptr, *m_d = nullptr;
    double* lm_pos = nullptr;    // [lm_cap*3]
    double* lm_weight = nullptr; // [lm_cap]
    int* sel_index = nullptr;    // [lm_cap] position of the landmark in the current selection, -1 otherwise (all -1 between solves)
    int* cursor = nullptr;       // [lm window capacity] scratch
    long long* key = nullptr;    // [obs window capacity] scratch: (keyframe index, arena index) of each gathered observation
    int* n_depth = nullptr;      // [1] gathered observations with a lidar depth (d > 0): the depth residual blocks of the window
    int kf_cap = 0, lm_cap = 0, m_cap = 0;
};
// per-solve selection, device copies of the caller's small lists
struct TrackSel {
    const int* kf_slot = nullptr;    // [n_kf] ascending keyframe id
    const unsigned char* kf_fixed = nullptr;
    const int* lm_slot = nullptr;    // [n_lm] ascending landmark id
    int n_kf = 0, n_lm = 0, max_meas = 0;  // n_kf = n_lm = 0: the window is idle (WinDesc::idle)
    int auto_scale = 0;              // 1: scale-regulariser weight by the reference rule (cpp:703-716) from the gathered window
    const int* gp_cand = nullptr;    // [n_cand] candidate ground points (index into lm_slot, ascending), attached by k_track_ground
    int n_cand = 0;                  // 0: the window's ground-plane lists (if any) came from the host
};
// grid sizes of the gather / write-back launches: maxima over the windows of the batch
struct TrackGrid {
    int max_kf = 0, max_lm = 0, max_meas = 0;
    int any_cand = 0;                // some window attaches its ground points on the device
};
// builds the raw CSR of every window w of batch `bd` (its PackRaw inputs) from track store tds[w] and selection sels[w]
// (device arrays of bd.n_win entries); desc[w].n_obs is written on the device
void launch_track_gather(const BatchDev& bd, const PackRaw& raw_out, const TrackDev* tds, const TrackSel* sels, const TrackGrid& g,
                         cudaStream_t s);
// rows of `width` doubles into store slots, for n windows (tracks) in one launch: row r of window w is row val0 + r of `val`, its
// slot slot[slot0 + r], written to dst[slot * width ..]
struct ScatterWin {
    double* dst = nullptr;
    int slot0 = 0, val0 = 0, n = 0, pad = 0;
};
void launch_scatter_rows(const ScatterWin* wins, int n_win, int max_rows, const int* slot, const double* val, int width, cudaStream_t s);

// ---- store writes of a track group (kba_track_group_push_keyframes, kba_store.cu) ---------------------------------------
// One staged segment of a pushed keyframe: rows src .. src + n of the staged columns (lm, cam, u, v, d, 4 bytes each) go to arena
// entries off + seg .. of the track's current arena; the keyframe's layout (m_off = off, m_cnt = cnt), pose and plane are written
// with it.  cam_zero: no camera column, every measurement is camera 0.
struct StoreAppend {
    unsigned* col[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};  // the current arena: lm, cam, u, v, d
    int* m_off = nullptr;
    int* m_cnt = nullptr;
    double* kf_pose = nullptr;
    double* kf_plane = nullptr;
    double pose[7] = {0, 0, 0, 0, 0, 0, 0};
    double plane[4] = {0, 0, 0, 0};
    const double* pose_src = nullptr;  // [7] or null: the pose is read from device memory (a frame step's adjusted pose), not `pose`
    int slot = 0, off = 0, cnt = 0, seg = 0, n = 0, src = 0, cam_zero = 0, pad = 0;
};
// one track's compaction: its live keyframes' runs copied from one arena into the other.  m_off null: the runs are copied out
// of the store (into a snapshot) and no layout is written.
struct CompactTrack {
    const unsigned* src[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
    unsigned* dst[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
    int* m_off = nullptr;
    int* m_cnt = nullptr;
};
// one keyframe slot of a compaction: n entries from src to dst, then m_off[slot] = dst, m_cnt[slot] = n (n = 0: a dropped slot's
// count cleared, dst its unchanged offset)
struct CompactRun {
    int track = 0, slot = 0, src = 0, dst = 0, n = 0, pad = 0;
};
// the compaction runs (if any), then the appends, on stream s: cols = the staged columns, 5 x stride entries
void launch_store_push(const CompactTrack* ct, const CompactRun* runs, int n_runs, int max_run, const StoreAppend* app, int n_app,
                       int max_rows, const unsigned* cols, int stride, cudaStream_t s);
// n words from src to dst: the parts of a snapshot that are not arena runs (header and keyframe lists, poses, planes, landmark
// values), between a store and a snapshot image in device memory, for many tracks in one launch (k_copy_spans, kba_store.cu)
struct CopySpan {
    const unsigned* src = nullptr;
    unsigned* dst = nullptr;
    long long n = 0;
};
void launch_copy_spans(const CopySpan* spans, int n_spans, long long max_words, cudaStream_t s);

// results of every window w back into track store tds[w]
void launch_track_writeback(const BatchDev& bd, const TrackDev* tds, const TrackSel* sels, const TrackGrid& g, cudaStream_t s);

// ---- landmark selection on a track's store (kba_track_select_landmarks / kba_track_group_select_landmarks, kba_select.cu) ----
// One window = one request: active keyframe slots (ascending timestamp), candidate landmark slots (ascending id).  Scratch is the
// track's, sized for its capacities at its first selection; the outputs point into one device block that goes down in one copy.
struct SelectArgs {
    TrackDev td;
    const int* kf_slot = nullptr;   // [n_kf]
    const int* lm_slot = nullptr;   // [n_cand]
    const double* cam_pose7 = nullptr;  // [n_cam * 7] the track's cameras
    int n_kf = 0, n_cand = 0, n_cam = 0;
    double leaf[3] = {0., 0., 0.}, roi_far = 0., roi_middle = 0.;
    // scratch
    int* cand_of = nullptr;         // [lm_cap] slot -> candidate, all -1 between calls
    double* kf_T = nullptr;         // [kf_cap * 12] transforms of the listed keyframes
    double* cam_T = nullptr;        // [kMaxCam * 12]
    double* path = nullptr;         // [kf_cap * 3] keyframe positions seen from the newest keyframe
    float* pt = nullptr;            // [lm_cap * 3] cloud points by candidate
    int* cnt = nullptr;             // [lm_cap] arena entries per candidate
    int* cursor = nullptr;          // [lm_cap]
    int* obs_off = nullptr;         // [lm_cap] first key of a near candidate's observations
    int* in_list = nullptr;         // [lm_cap] cloud points (candidate indices), in arrival order
    long long* vkey = nullptr;      // [lm_cap] voxel index by cloud position
    int* sorted = nullptr;          // [lm_cap] cloud positions in (voxel index, label) order
    int* near_flag = nullptr;       // [lm_cap] by sorted position: a near voxel starts here
    long long* okey = nullptr;      // [m_cap] (keyframe position, arena index) of the near candidates' observations
    unsigned* bounds = nullptr;     // [6] order-preserving min xyz, max xyz of the cloud
    int* counters = nullptr;        // [3] cloud points, near voxels, gathered observations
    // outputs [n_cand]
    unsigned char* cheiral = nullptr;
    signed char* bin = nullptr;
    int* near_order = nullptr;
    int* n_near = nullptr;          // = counters + 1
    double* flow = nullptr;
    int* seen = nullptr;
};
// W windows in one launch sequence, window = grid z.  Window 0's arguments travel in the launch parameters, as a one-track
// selection's always did, so that it uploads its lists and nothing else; windows 1 .. W-1 read theirs from a device array that
// goes up in the same copy as the lists.
struct SelectLaunch {
    SelectArgs w0;
    const SelectArgs* rest = nullptr;  // [n_win - 1]
    const SelectArgs* all = nullptr;   // [n_win] or null: every window's record in device memory (w0, rest unused), for records that
                                       // an earlier kernel of the same sequence completes (k_kfs_labels)
    int n_win = 0;
};
// grid sizes: maxima over the windows (threads beyond their own window's sizes exit)
struct SelectGrid {
    int max_kf = 0, max_cand = 0, max_init = 0;  // max_init: of max(n_cand, n_kf, n_cam)
    int max_meas = 0;                            // arena entries of a listed keyframe
};
void launch_select(const SelectLaunch& l, const SelectGrid& g, cudaStream_t s);

// ---- landmark creation of push() on a track's store (kba_track_create_landmarks / kba_track_group_create_landmarks, kba_create.cu) ----
// One window = one request: the active keyframe slots (ascending id, kf_new the one just pushed) and the slots of the landmarks to
// create.  Scratch is the track's, sized for its capacities at its first creation; the outputs point into one device block.
struct CreateArgs {
    TrackDev td;
    const int* kf_slot = nullptr;     // [n_kf]
    const int* lm_slot = nullptr;     // [n_new]
    const double* cam_intr = nullptr; // [n_cam * 3] the track's cameras: f, cx, cy
    const double* cam_pose7 = nullptr;// [n_cam * 7]
    int n_kf = 0, kf_new = 0, n_new = 0, n_cam = 0;
    // scratch
    int* req_of = nullptr;            // [lm_cap] slot -> request index, all -1 between calls
    double* ray_T = nullptr;          // [kf_cap * n_cam * 12] (cam * kf).inverse() of every listed keyframe and camera
    double* intr_inv = nullptr;       // [n_cam * 9] Camera::intrin_inv
    int* cnt = nullptr;               // [lm_cap] arena entries per request
    int* cursor = nullptr;            // [lm_cap]
    int* off = nullptr;               // [lm_cap] first key of a request's entries
    long long* key = nullptr;         // [m_cap] (keyframe position, arena index) of every gathered entry
    int* total = nullptr;             // [1] gathered entries
    // outputs [n_new]
    double* pos = nullptr;            // [3 * n_new]
    unsigned char* flags = nullptr;
};
// W windows in one launch sequence, window = grid z; window 0's arguments travel in the launch parameters (as SelectLaunch)
struct CreateLaunch {
    CreateArgs w0;
    const CreateArgs* rest = nullptr;  // [n_win - 1]
    int n_win = 0;
};
struct CreateGrid {
    int max_kf = 0, max_new = 0, max_init = 0;  // max_init: of max(n_new, n_kf * n_cam)
    int max_meas = 0;                           // arena entries of a listed keyframe
};
void launch_create(const CreateLaunch& l, const CreateGrid& g, cudaStream_t s);

// ---- window upkeep on a track's store (kba_track_deactivate_keyframes / kba_track_depth_costs and their group forms,
// kba_upkeep.cu) ----
// One window = one request: the active keyframe slots (ascending id) and a landmark list (deactivation: the active landmarks;
// depth costs: the eligible ones, ascending id).  The slot map is the track's; an entry is (stamp << 32) | payload and counts only
// when its stamp is this call's, so the map needs no clearing between calls.
struct UpkeepArgs {
    TrackDev td;
    const int* kf_slot = nullptr;          // [n_kf]
    const int* lm_slot = nullptr;          // [n_lm]
    int n_kf = 0, n_lm = 0;
    const int* n_lm_d = nullptr;           // or null: the deactivation reads n_lm from here (k_cs_lists writes it), n_lm its bound
    int min_connecting = 0, min_window = 0, max_window = 0;
    unsigned stamp = 0;                    // deactivation uses stamp (newest keyframe) and stamp + 1 (surviving keyframes)
    unsigned long long* map = nullptr;     // [lm_cap] scratch, by slot
    // deactivation outputs
    int* kf_common = nullptr;              // [n_kf]
    unsigned char* kf_active = nullptr;    // [n_kf]
    unsigned char* lm_active = nullptr;    // [n_lm]
    // depth-cost outputs: keyframe k's pairs at base_k = sum over k' < k of min(n_lm, arena entries of k')
    int* cnt = nullptr;                    // [n_kf] pairs of keyframe k
    int* cand = nullptr;                   // [B]
    double* cost = nullptr;                // [B]
};
// W windows in one launch sequence, window = grid z; window 0's arguments travel in the launch parameters (as SelectLaunch)
struct UpkeepLaunch {
    UpkeepArgs w0;
    const UpkeepArgs* rest = nullptr;      // [n_win - 1]
    int n_win = 0;
};
struct UpkeepGrid {
    int max_kf = 0, max_lm = 0;
    int max_meas = 0;                      // arena entries of a listed keyframe
};
void launch_deactivate(const UpkeepLaunch& l, const UpkeepGrid& g, cudaStream_t s);
void launch_depth_costs(const UpkeepLaunch& l, const UpkeepGrid& g, cudaStream_t s);

// ---- the flow scheme of keyframe selection on a track's store (kba_track_frame_flow / kba_track_group_frame_flow,
// kba_keyframe.cu) ----
// One window = one request: the new frame's measurements (runs by landmark slot, cameras ascending inside a run) against the
// stored keyframe kf_last.  The slot map is the track's upkeep map (UpkeepArgs): kf_last's runs are marked with the call's stamp
// and their first entry, so the map needs no clearing between calls.
struct FlowRes {                           // one window's download record, 24 bytes
    double flow_sum, mean_flow_sq;
    int n_matched, usable;
};
struct FlowArgs {
    TrackDev td;
    int kf_last = 0, n_meas = 0;
    const int* lm_slot = nullptr;          // [n_meas]
    const int* cam = nullptr;              // [n_meas]
    const float* u = nullptr, *v = nullptr;  // [n_meas]
    double min_median_flow = 0;
    unsigned stamp = 0;
    unsigned long long* map = nullptr;     // [lm_cap] scratch, by slot
    FlowRes* res = nullptr;
    int* match = nullptr;                  // [n_meas] index into kf_last's entries, -1: no match
};
struct FlowLaunch {
    FlowArgs w0;
    const FlowArgs* rest = nullptr;        // [n_win - 1]
    int n_win = 0;
};
struct FlowGrid {
    int max_last = 0;                      // arena entries of the largest kf_last
};
void launch_frame_flow(const FlowLaunch& l, const FlowGrid& g, cudaStream_t s);

// ---- free landmark slots of a track's store (kba_track_reclaim_landmarks / kba_track_group_reclaim_landmarks, kba_reclaim.cu) ----
// One window = one request: the slot range [lo, hi) and the track's live keyframe slots.  The slot map is the track's upkeep map:
// every arena entry of a live keyframe is marked with the call's stamp, the unmarked slots of the range are the free ones.
constexpr int kReclaimChunk = 1024;        // slots of the range per block of k_rc_count / k_rc_write (256 threads, 4 slots each)
struct ReclaimArgs {
    TrackDev td;
    const int* kf_live = nullptr;          // [n_live] live keyframe slots
    int n_live = 0, lo = 0, hi = 0;
    unsigned stamp = 0;
    unsigned long long* map = nullptr;     // [lm_cap] scratch, by slot
    int* blk = nullptr;                    // [ceil(lm_cap / kReclaimChunk)] scratch: free slots per chunk of the range
    // outputs
    int* n_free = nullptr;                 // [1]
    int* free_slot = nullptr;              // [hi - lo]
    double* pos = nullptr;                 // [3 * (hi - lo)] or null
    double* weight = nullptr;              // [hi - lo] or null
};
struct ReclaimLaunch {
    ReclaimArgs w0;
    const ReclaimArgs* rest = nullptr;     // [n_win - 1]
    int n_win = 0;
};
struct ReclaimGrid {
    int max_live = 0, max_meas = 0;        // live keyframes of a window, arena entries of a live keyframe
    int max_range = 0;                     // hi - lo
};
void launch_reclaim(const ReclaimLaunch& l, const ReclaimGrid& g, cudaStream_t s);

// ---- the ranked selection on a track's store (kba_track_rank_landmarks / kba_track_group_rank_landmarks, kba_rank.cu) ----
// One window = one request, run after launch_select on the same lists.  The first part (launch_rank_prepare) counts the middle
// bin and computes the AddDepth costs; the host then downloads the counts and uploads the draws; the second part (launch_rank)
// replays the partial sorts, shuffles the middle bin and compacts the union into the track's ranked list.
constexpr int kRankMaxCand = 57344;        // candidates of a request: the middle bin and every heap live in shared memory, 4 B each
constexpr int kRankMaxDepth = 1024;        // AddDepth entries of a request: one block each
struct RankArgs {
    TrackDev td;
    const int* kf_slot = nullptr;          // [n_kf]
    const int* lm_slot = nullptr;          // [n_cand]
    const unsigned char* elig = nullptr;   // [n_cand]
    const int* depth = nullptr;            // [2 * n_depth] (ind, wanted)
    int n_kf = 0, n_cand = 0, n_depth = 0;
    int max_near = 0, max_middle = 0, max_far = 0;
    // the selection chain's quantities (the SelectArgs outputs of the same window), on the device only
    const unsigned char* cheiral = nullptr;
    const signed char* bin = nullptr;
    const int* near_order = nullptr;
    const int* n_near = nullptr;
    const double* flow = nullptr;
    const int* seen = nullptr;
    // scratch
    int* cand_of = nullptr;                // SelectArgs::cand_of: slot -> candidate for the call, all -1 again at its end
    int* mark = nullptr;                   // [lm_cap] by candidate: bit 0 near, 1 middle, 2 far, 3 AddDepth
    int* dcand = nullptr;                  // [m_cap] listed keyframe k's i-th eligible landmark (candidate) at m_off[kf_slot[k]] + i
    double* dcost = nullptr;               // [m_cap] ... and its cost
    int* dcnt = nullptr;                   // [kf_cap] eligible landmarks of listed keyframe k
    // the track's ranking
    int* sel_slot = nullptr;               // [lm_cap] ranked landmark slots
    int* gp = nullptr;                     // [lm_cap] ranked ground candidates, indices into sel_slot
};
// W windows in one launch sequence, window = grid z; window 0's arguments travel in the launch parameters (as SelectLaunch).
// n_mid, p2 and the outputs are shared by the windows, indexed by window.
struct RankLaunch {
    RankArgs w0;
    const RankArgs* rest = nullptr;        // [n_win - 1]
    const RankArgs* all = nullptr;         // [n_win] or null: as SelectLaunch::all
    int n_win = 0;
    int* n_mid = nullptr;                  // [n_win] middle-bin sizes (zeroed before launch_rank_prepare)
    const int* p2 = nullptr;               // [2 * n_win] (first draw, first output) of each window, then the draws end to end
    int* res = nullptr;                    // [2 * n_win] n_sel, n_ground of each window
    int* out_cand = nullptr;               // outputs of window w from its first output on
    signed char* out_cat = nullptr;
};
struct RankGrid {
    int max_kf = 0, max_cand = 0, max_depth = 0;
    int mid_ints = 1;                      // dynamic shared memory of k_rk_heap, in ints: the largest middle bin
    int heap_ints = 1;                     // ... and the largest near, far or AddDepth heap
};
void launch_rank_prepare(const RankLaunch& l, const RankGrid& g, cudaStream_t s);
void launch_rank(const RankLaunch& l, const RankGrid& g, cudaStream_t s);

// ---- limo's solve block on a track's store (kba_track_keyframe_solve and its group forms, kba_kfsolve.cu) ----
// One window = one request, one CTA.  k_kfs_labels runs between launch_deactivate and launch_select of the same sequence: updateLabels
// over the deactivation's outputs, the post-deactivation keyframe list and the ranking's candidates, whose counts it writes into the
// window's SelectArgs / RankArgs records (launched with `all`).  k_kfs_weights writes the shrubbery weights once the call's checks
// have passed.
constexpr unsigned char kKfsMarked = 1, kKfsShrub = 2, kKfsGround = 4;  // trk_cls: outlier (is_outlier or label), shrubbery, ground
struct KfsArgs {
    const int* kf_slot = nullptr;          // [n_kf] the request's keyframes
    const int* lm_slot = nullptr;          // [n_lm] the request's landmarks
    const unsigned char* kf_active = nullptr;  // [n_kf] the deactivation's outputs
    const unsigned char* lm_active = nullptr;  // [n_lm]
    const unsigned char* ground_in = nullptr;  // [n_lm] or null
    const int* out_slot = nullptr;         // [n_out] the caller's outlier set
    const int* trk_slot = nullptr;         // [n_trk] slot or -1
    const unsigned char* trk_cls = nullptr;    // [n_trk] kKfs* bits
    int n_kf = 0, n_lm = 0, n_out = 0, n_trk = 0;
    const int* n_lm_d = nullptr;           // or null: n_lm is read from here (k_cs_lists writes it), the field is its bound
    int* lm_at = nullptr;                  // [lm_cap] scratch, -1 between calls
    int* last = nullptr;                   // [lm_cap] scratch
    unsigned char* lm_out = nullptr;       // [n_lm] outputs
    unsigned char* ground = nullptr;       // [n_lm]
    unsigned char* trk_out = nullptr;      // [n_trk]
    unsigned char* shrub = nullptr;        // [n_trk]
    int* kf_post = nullptr;                // [n_kf] the kept keyframes, then their fixation
    unsigned char* fixed = nullptr;        // [n_kf]
    int* cand = nullptr;                   // [n_lm] the candidates' slots and AddDepth eligibility
    unsigned char* elig = nullptr;         // [n_lm]
    int* counts = nullptr;                 // [2] kept keyframes, candidates
    SelectArgs* sel = nullptr;             // the window's records: n_kf, n_cand written
    RankArgs* rank = nullptr;
    double* lm_weight = nullptr;           // the store's weights
    double shrub_weight = 0.;
};
void launch_kfs_labels(const KfsArgs* args, int n_win, cudaStream_t s);
void launch_kfs_weights(const KfsArgs* args, int n_win, int max_trk, cudaStream_t s);

// ---- limo's camera callback on a track's store (kba_track_camera_step and its group forms, kba_camerastep.cu) ----
// One CTA per solving window, between the push's creation kernels and the solve block's first part (launch_deactivate,
// launch_kfs_labels, ...) of the same sequence: the candidate list staged as the solve block's landmark list is compacted in
// place, in list order, to the landmarks the push leaves active, and its length goes to n_lm, which the deactivation and
// k_kfs_labels read (UpkeepArgs::n_lm_d, KfsArgs::n_lm_d).
constexpr int kCsActive = -2, kCsMeasured = -1;  // tags: active before the frame; measured by it (listed iff it is selected)
struct CsArgs {
    int* lm_slot = nullptr;                // [n_cand] the candidates in, the solve's list out (in place)
    unsigned char* ground = nullptr;       // [n_cand] their is_ground_plane, compacted alongside
    const int* tag = nullptr;              // [n_cand] kCsActive, kCsMeasured or k >= 0: new_slot[k], listed iff created
    const unsigned char* created = nullptr;  // [n_new] the creation's flags (bit 0: created); null when the frame is not selected
    int n_cand = 0;
    int selected = 0;
    int* index = nullptr;                  // [n_cand] out: each candidate's position in the list, or -1
    int* n_lm = nullptr;                   // out: the list's length
};
void launch_cs_lists(const CsArgs* args, int n_win, cudaStream_t s);

// ---- evaluation of stored windows at the store's state (kba_track_evaluate / kba_track_group_evaluate, kba_evaluate.cu) ----
// Run after launch_track_gather on the same batch, in place of the packing and the solve: the outputs of window w go to its
// regions of one output block (EvalOut), in the window's own order, so that one copy brings every window's outputs down.
struct EvalWin {                           // window w's regions, in entries of each array
    int obs0;                              // observations: obs_*, res (3 per entry), rho (2 per entry)
    int lm0;                               // landmarks: trim and rej, group g at g * n_lm_total + lm0
    int gp0;                               // ground-plane residuals
    int part0, n_part;                     // cost partials of k_ev_obs: one per 64 landmarks
    int n_lm_total;                        // landmark entries of the whole block
};
struct EvalHead {                          // one window's record of the block, 64 bytes
    int n_obs, n_gp, failed, pad;
    double cost[6];                        // reprojection, depth, ground plane, scale regulariser, plane chain, total
};
struct EvalOut {
    EvalHead* head;                        // [n_win]
    double* res, *rho, *trim, *gp_w, *gp_r;
    int* obs_lm, *obs_kf, *obs_cam, *gp_lm, *gp_kf;
    unsigned char* rej;
    double* part;                          // [3 * partials] scratch (not downloaded)
};
void launch_evaluate(const BatchDev& bd, const PackRaw& raw, const EvalWin* wins, const EvalOut& o, int max_lm, cudaStream_t s);

// ---- motion-only frames against a track's store (kba_track_adjust_pose / kba_track_group_adjust_pose, kba_motion.cu) ----
// One frame = one free pose against constant landmarks read from a store by slot: its measurements come in runs, one run per
// landmark (the landmarks of the equivalent window, in the caller's order).
struct FrameDesc {
    int n_meas, n_runs;
    int meas_off;               // first measurement of the frame in the call's staged arrays
    int run_off;                // first run of the frame in the work / result arrays
    int rs_off;                 // first entry of the frame's run_start list (n_runs + 1 entries, frame-local measurement indices)
    int rounds_total;           // trimming rounds, resolved on the host (k_reset_state's rule on MotionArgs::sp of the frame)
    const double* lm_pos;       // the track's store: positions [lm_cap*3] and weights by slot
    const double* lm_weight;
    const double* cam16;        // the track's staged cameras (kCamStride doubles each)
    int n_cam, pad;
    double pose7[7];
    double speed_weight, speed_dt;
    double speed_v_before[3];
    double speed_T_origin_before[7];
};
// what one frame hands back (the frame's slot of the result block; its rejections and iteration records follow elsewhere in it)
struct FrameRes {
    double pose[7];
    int n_solves, log_n, done, pad;
    SolveSummary solves[8];
};
struct MotionArgs {
    const FrameDesc* fd;        // [n_frames]
    const SolveParams* sp;      // [n_frames] solver options of each frame
    const int* lm_slot;         // [total measurements] staged per call
    const int* cam;
    const float* u, *v, *d;
    const int* run_start;
    double* run_pw;             // [4 * total runs] work: landmark position and weight of every run
    unsigned char* run_active;  // [total runs] work
    unsigned char* run_rej;     // [total runs] work
    double* trim_val;           // [2 * total runs] work: per-run maximum raw residual (depth, reprojection)
    IterRecord* log;            // [n_frames * kIterLogCap] work
    FrameRes* res;              // [n_frames]
    IterRecord* res_log;        // [n_frames * log_cap]
    unsigned char* res_rej;     // [total runs]
    int log_cap, total_runs;
};
void launch_adjust_pose(const MotionArgs& a, int n_frames, cudaStream_t s);

// ---- limo's frame step on a track's store (kba_track_frame_step and its group forms, kba_framestep.cu) ----
// One window = one request, one CTA of k_fs_gather, which runs ahead of k_adjust_pose and the flow kernels in the same sequence:
// it copies kf_last's stored pose into the download and, for a frame that is adjusted, gathers the measurements of its selected
// runs from the staged columns into the pose-only kernel's input (MotionArgs' lm_slot .. d and run_start at meas_off / rs_off),
// keeping their order with a block-wide ballot scan.  The host knows the gathered sizes from its checks and writes the FrameDesc.
struct StepArgs {
    int src = 0, n_meas = 0;               // the window's rows of the staged columns
    int flag0 = 0;                         // its first run flag
    int adjust = 0;                        // 1: gather the selected runs
    int meas_off = 0, rs_off = 0;          // where they go: MotionArgs' columns, run_start
    const double* kf_pose = nullptr;       // [7] kf_last's stored pose
    double* last_pose = nullptr;           // [7] its copy in the download
};
struct StepLaunch {
    const StepArgs* win = nullptr;         // [n_win]
    const unsigned* cols = nullptr;        // the staged columns lm, cam, u, v, d, `stride` words each
    int stride = 0;
    const unsigned char* run_sel = nullptr;  // every window's run flags, end to end
    unsigned* dst[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};  // MotionArgs' lm_slot, cam, u, v, d
    int* run_start = nullptr;              // MotionArgs' run_start
    int n_win = 0;
};
void launch_frame_step_gather(const StepLaunch& l, cudaStream_t s);

// ---- lidar depth (kba_lidar.cu, compiled with -fmad=false) ----
// The host halves of kba_lidar_depth_batch, shared with the frame step's lidar form (kba_track_frame_step_lidar): a plan of the
// call's views -- their parameters in the kernels' single precision and the offsets of their cells, sorted point records, blocks
// and features --, the handle's grow-only workspace for the used clouds and the scratch, and one launch sequence (memset, count,
// scan, fill and feature kernels).  The batch's feature pass reads packed (u, v) pairs and writes depths in feature order; the
// frame step's reads feature k as staged measurement idx[k]: u, v from the staged columns, its depth into the staged d column.
// Both are one template of k_lidar_feature, so the depths are the same bit for bit.
struct LidarParams {
    float R[9], t[3], f, cx, cy;
    int width, height, cells_x, cells_y;
    float hw, hh, offx, offy, bw;
    int hist_min_count, min_points;
    float depth_min, depth_max, local_tol, crossnorm_min, viewray_min;
    int local_enabled;
    // where the view's data sits in the call's concatenated device arrays
    long long cloud_off;       // floats, into the clouds
    int n_points, stride;
    int cell_off;              // cells_x * cells_y + 1 entries of counts, cursors and starts
    int sort_off;              // n_points sorted point records
};
struct LidarPlan {
    std::vector<LidarParams> par;                // one per view
    std::vector<int> blk_off{0}, feat_off{0};    // prefixes over the views: blocks of 256 points, features
    std::vector<long long> cloud_off;            // per cloud: floats into the workspace's clouds; -1: no view names it
    long long cells = 0, pairs = 0, blocks = 0, feats = 0;
    size_t b_clouds = 0;
    explicit LidarPlan(int n_clouds) : cloud_off(n_clouds, -1) {}
    // a view of n_feat features on cloud c (checked by the caller) with options o; KBA_ERR_CAPACITY when the call's cells,
    // (view, point) pairs or 2 * features pass INT32_MAX
    int add(int c, const kba_lidar_cloud& cl, const double* T_cam_lidar, const double* intr, const kba_lidar_options* o, int n_feat);
    size_t pack_bytes() const;                   // what the launch reads from d_pack: view parameters | block | feature prefix
    void pack(void* dst) const;
};
struct LidarWs {                                 // the plan's part of the handle's workspace
    float* clouds = nullptr;
    int* cnt = nullptr, *cur = nullptr, *start = nullptr;
    void* sorted = nullptr;
    void* extra = nullptr;                       // the caller's `extra` bytes, 256-byte aligned
};
int lidar_workspace(kba_handle* h, const LidarPlan& p, size_t extra, LidarWs& ws);
// one copy per cloud a view names, from the caller's memory into the workspace
cudaError_t lidar_copy_clouds(const LidarPlan& p, const kba_lidar_cloud* clouds, const LidarWs& ws, cudaStream_t s);
struct LidarStaged {                             // the frame step's features: feature k is staged measurement idx[k]
    const float* u = nullptr, *v = nullptr;      // the staged columns
    const int* idx = nullptr;                    // [feats] measurement rows, view by view
    float* d = nullptr;                          // the staged d column: d[idx[k]] = depth
    int n_copy = 0;                              // the first n_copy features' depths also go to copy[k] (the download)
    float* copy = nullptr;
};
cudaError_t launch_lidar_staged(const LidarPlan& p, const LidarWs& ws, const void* d_pack, const LidarStaged& f, cudaStream_t s);

cudaError_t configure_pack();
void launch_pack(const BatchDev& bd, const PackRaw& raw, cudaStream_t s);
void launch_unpack_landmarks(const BatchDev& bd, double* lm_user, unsigned char* rejected_user, cudaStream_t s);

cudaError_t configure_kernels(int nr_cap_max);
void launch_reset(const BatchDev& bd, const LaunchCfg& lc, cudaStream_t s);
int launch_shard_gather(const BatchDev& bd, const LaunchCfg& lc, cudaStream_t s);  // sharded window: attachment of all ground points
int launch_pass(const BatchDev& bd, const LaunchCfg& lc, Counters* cnt, cudaStream_t s);
void launch_count_active(const BatchDev& bd, cudaStream_t s);
void launch_loop_cond(const BatchDev& bd, unsigned long long handle, int* pass, int max_passes, cudaStream_t s);  // WHILE-node condition
void launch_force_linearize(const BatchDev& bd, cudaStream_t s);
void launch_jacobian_only(const BatchDev& bd, cudaStream_t s);
void launch_expand_jl(const BatchDev& bd, double* out, cudaStream_t s);  // fused path: J_l as its consumers form it

}  // namespace kba
