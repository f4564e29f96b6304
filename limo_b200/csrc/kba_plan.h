// kba_plan.h -- the launch plan of a batch: solver path, Schur kernel instance and split, factorisation, packing.  Each choice
// changes the rounding of the result, so it is made here only.  Host-only: tests/test_launch_plan.py compiles it with g++.
#pragma once
#include <algorithm>
#include <cstdlib>

namespace kba {

constexpr int kFusedMaxRows = 184;          // every window within this many reduced rows: the fused path (k_schur_fused)
constexpr int kSixSlotMaxRows = 176;        // k_schur_fused<6>: 11 16-row block rows; <7> has a 12th for up to kFusedMaxRows
constexpr int kTiledMaxRows = 192;          // k_reduced_solve<true>: the reduced system factorised in one CTA's shared memory
constexpr int kPanelMaxRows = 640;          // shared-memory panel copies of stage 0 of k_reduced_solve / k_chol_trail (227 KB per CTA)
constexpr int kTrackMaxRows = 640;          // a track's large-window solver (kba_track_caps.win_rows); limo's windows are far smaller
constexpr int kSyrkMaxSplit = 16;           // most CTAs k_schur_syrk deals a window's 32-landmark chunks to
constexpr int kSplitSolveMaxWindows = 16;   // batches of at most this many windows spread a large factorisation (k_chol_*) ...
constexpr int kSplitSolveMaxCtas = 32;      // ... over at most this many CTAs per window
constexpr int kFusedMaxKf = 32;             // keyframes the fused-path kernels stage in shared memory
constexpr int kPackMaxLandmarks = 32768;    // device packing: 15 index bits, 128 KB of sort keys in shared memory
constexpr int kMaxKf = 128;                 // keyframes per window the kernels stage in shared memory
static_assert((kFusedMaxRows - 1) / 6 <= kFusedMaxKf, "a window has at least 6 reduced rows per keyframe");

// reduced-system rows of n_kf keyframes: 6 per pose, 4 more with plane blocks, and the right-hand side
constexpr int reduced_rows(int n_kf, bool planes) { return (planes ? 10 : 6) * n_kf + 1; }
// rows a window's reduced system is allocated with (a window that sits a solve out: rows = 0)
constexpr int nr_cap_of(int rows) { return std::max(64, (rows + 63) / 64 * 64); }
// k_schur_fused instance for the largest reduced rows of the free keyframes of a batch
constexpr int fused_slots(int free_rows) { return free_rows <= kSixSlotMaxRows ? 6 : 7; }
// largest reduced system kba_batch_create takes: kMaxKf keyframes with plane blocks (1281 rows, allocated as 1344)
constexpr int kMaxReducedRows = nr_cap_of(reduced_rows(kMaxKf, true));
static_assert(nr_cap_of(kPanelMaxRows) == kPanelMaxRows, "the panel bound is a whole number of 64-row blocks");

// what the environment selects, read once per kba_batch_create (a track's solvers keep those of their creation)
struct Knobs {
    int fused = 1;         // KBA_FUSED=0: small windows on global V panels + k_schur_syrk_tma
    int lin_fused = 1;     // KBA_LINEARIZE=0: three-kernel linearisation over a materialised Jacobian instead of k_linearize
    int p_split = 0;       // KBA_P_SPLIT > 0: CTAs a window's Schur sum is split over; 0: by batch size
    int lin_grid = -1;     // KBA_LIN_GRID, KBA_BS_GRID: CTAs per window of k_linearize / k_backsub_v (-1: by batch size,
    int bs_grid = -1;      //   0: one CTA per unit); any value gives bit-identical results
    int solve_split = -1;  // KBA_SOLVE_SPLIT >= 0: CTAs per window of the split factorisation (0: none); -1: by batch size
    int device_pack = 1;   // KBA_DEVICE_PACK=0: sort / CSR / keyframe-major copy on the host
};

inline Knobs read_knobs() {
    auto get = [](const char* name, int dflt) { const char* e = std::getenv(name); return e ? std::atoi(e) : dflt; };
    Knobs k;
    k.fused = get("KBA_FUSED", 1) != 0;
    k.lin_fused = get("KBA_LINEARIZE", 1) != 0;
    k.p_split = std::max(0, get("KBA_P_SPLIT", 0));
    k.lin_grid = std::max(-1, get("KBA_LIN_GRID", -1));
    k.bs_grid = std::max(-1, get("KBA_BS_GRID", -1));
    k.solve_split = get("KBA_SOLVE_SPLIT", -1);
    k.device_pack = get("KBA_DEVICE_PACK", 1) != 0;
    return k;
}

// TrackFused is planned like a batch; TrackLarge packs on the device and sizes sred for every split a solve re-plans to;
// HostPack (kba_eval) keeps the host-side observation permutation
enum class Purpose : int { Batch, TrackFused, TrackLarge, HostPack };

// rows: reduced rows the window is sized for (reduced_rows on all its keyframes, or a track's own; 0: idle); free_rows: those
// of its free keyframes; 32-landmark chunks (k_schur_syrk), 8-landmark groups (k_schur_fused), landmarks
struct WinShape { int rows = 0, free_rows = 0, n_chunks = 0, n_groups = 0, n_lm = 0; };

// plain data, ints only: the solve graph's cache key holds it byte for byte
struct Plan {
    int nr_cap_max = 64;  // largest nr_cap_of(rows) of the batch
    int small_syrk = 0;   // every window within kFusedMaxRows rows: one CTA per split owns a window's whole reduced system
    int fused = 0;        // ... and KBA_FUSED: k_schur_fused, no J_l, no global V panels
    int fused_slots = 6;  // k_schur_fused<6> or <7>
    int p_split = 1;      // CTAs a window's Schur sum is split over (partial sums folded in a fixed order)
    int p_split_cap = 1;  // the largest p_split sred has room for
    int solve_tiled = 0;  // k_reduced_solve<true>, else the row-major factorisation
    int solve_split = 0;  // > 0: the row-major factorisation spread over this many CTAs per window (k_chol_*)
    int solve_banded = 0; // nr_cap_max > kPanelMaxRows: k_sred_reduce forms A, k_chol_trail_band updates, no panel copy anywhere
    int device_pack = 0;  // packing kernels (kba_pack.cu) instead of the host
};

// CTAs per window k_schur_syrk deals a window's chunks to: enough for the batch's 64-row block pairs to fill the GPU
inline int syrk_split(int nr_cap_max, int n_windows, int sm_count) {
    const int nb = nr_cap_max / 64, pairs = nb * (nb + 1) / 2;
    return std::min(kSyrkMaxSplit, (6 * sm_count + n_windows * pairs - 1) / (n_windows * pairs));
}

// the factorisation: tiled in one CTA when it fits, else row-major, spread over the GPU when the batch has few windows (a single
// SM's FP64 rate bounds the one-CTA factorisation of a large system).  Above kPanelMaxRows the one-CTA factorisation (stage 0)
// has no room for its panel copy: such a batch is always split, over at least one CTA per window, whatever its size.
inline void plan_solve(Plan& p, int n_windows, int sm_count, const Knobs& k) {
    p.solve_tiled = p.nr_cap_max <= kTiledMaxRows;
    p.solve_banded = p.nr_cap_max > kPanelMaxRows;
    const int spread = std::max(1, std::min(kSplitSolveMaxCtas, sm_count / n_windows));
    const int split = (n_windows <= kSplitSolveMaxWindows || p.solve_banded) ? spread : 0;
    p.solve_split = p.solve_tiled ? 0 : (k.solve_split >= 0 ? k.solve_split : split);
    if (p.solve_banded) p.solve_split = std::max(1, p.solve_split);
}

// The plan of a batch of n windows.  The path is decided on the rows of all keyframes, the Schur kernel instance on the free
// ones; one window beyond kFusedMaxRows rows puts the whole batch on the large-window path.
inline Plan make_plan(const WinShape* w, int n, int sm_count, const Knobs& k, Purpose purpose) {
    Plan p;
    int max_rows = 0, max_free = 0, max_chunks = 1, max_groups = 1, max_lm = 0;
    for (int i = 0; i < n; ++i) {
        max_rows = std::max(max_rows, w[i].rows);
        max_free = std::max(max_free, w[i].free_rows);
        max_chunks = std::max(max_chunks, w[i].n_chunks);
        max_groups = std::max(max_groups, w[i].n_groups);
        max_lm = std::max(max_lm, w[i].n_lm);
        p.nr_cap_max = std::max(p.nr_cap_max, nr_cap_of(w[i].rows));
    }
    p.small_syrk = max_rows <= kFusedMaxRows;
    p.fused = p.small_syrk && k.fused;
    p.fused_slots = fused_slots(max_free);
    // Small windows: one CTA per SM, each owning all tiles of its share.  A CTA of k_schur_fused takes at least 8 landmark groups
    // (schur_split, kba_schur_fused.cuh), so a window's partition does not depend on how many CTAs the batch was given.
    int split = p.small_syrk ? (sm_count + n - 1) / n : syrk_split(p.nr_cap_max, n, sm_count);
    if (k.p_split > 0) split = k.p_split;
    p.p_split = std::max(1, std::min(split, p.fused ? max_groups : max_chunks));
    if (purpose == Purpose::TrackLarge) {  // a solve re-plans on windows of more than kFusedMaxRows rows: kTiledMaxRows at the least
        const int most = k.p_split > 0 ? k.p_split : syrk_split(kTiledMaxRows, n, sm_count);
        p.p_split = std::max(p.p_split, std::max(1, std::min(most, max_chunks)));
    }
    p.p_split_cap = p.p_split;
    plan_solve(p, n, sm_count, k);
    p.device_pack = (p.fused || purpose == Purpose::TrackLarge) && purpose != Purpose::HostPack && max_lm <= kPackMaxLandmarks &&
                    k.device_pack;
    return p;
}

// A track solve on the large-window path: the reduced-system size, the Schur split and the factorisation follow the solved
// windows (w[i].rows, 0 for a window that sits the solve out) instead of the capacity windows, within the split sred was sized for,
// so that the solve rounds as kba_solve_window on the same windows does.
inline void replan_large(Plan& p, const WinShape* w, int n, int sm_count, const Knobs& k) {
    int max_chunks = 1;
    p.nr_cap_max = 64;
    for (int i = 0; i < n; ++i) {
        p.nr_cap_max = std::max(p.nr_cap_max, nr_cap_of(w[i].rows));
        max_chunks = std::max(max_chunks, w[i].n_chunks);
    }
    const int split = k.p_split > 0 ? k.p_split : syrk_split(p.nr_cap_max, n, sm_count);
    p.p_split = std::max(1, std::min(std::min(split, max_chunks), p.p_split_cap));
    plan_solve(p, n, sm_count, k);
}

}  // namespace kba
