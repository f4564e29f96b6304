// kba_schur_fused.cuh -- Schur complement of a small window (<= kFusedMaxRows reduced rows) in ONE warp-specialised kernel:
//
//   k_obs_v2 (kba_prep.cuh, one thread per observation, full occupancy) has written V_i = (J_p^T J_l) L^-T compactly:
//   18 doubles per observation (3 columns x 6 rows), no padding.
//   producers (4 warps, each assembling whole groups on its own: four panels under construction at any time):
//                          per group of 8 landmarks the panel (24 columns x the group's reduced-system rows, column-major,
//                          zeros included) is assembled in shared memory by ASYNCHRONOUS copies.  V is stored
//                          landmark-column-major, and a track without gaps sits on consecutive rows, so a landmark's panel
//                          column is ONE bulk copy (cp.async.bulk, 48 B per observation, complete_tx on the stage's "full"
//                          mbarrier): 24 bulk copies + the z rows per group, nobody waits for data and the ring runs five
//                          groups ahead.  A stage is not zeroed whole: per stage and panel column a small table keeps the
//                          rows that the group last assembled there may have left non-zero (its run and z row; every row of
//                          its panel on the per-observation and synchronous paths), and the column's lane zeroes those rows
//                          minus the ones its own bulk copy overwrites.  Alternatives tried and dropped: all 32 lanes
//                          zeroing row-parallel around the runs (one shuffle per column for the run bounds, which queue
//                          behind the consumers' shared-memory loads: slower than zeroing everything), zero segments as
//                          bulk copies too (no stores by the SM at all, but a warp issues its bulk copies one lane after
//                          the other), 16-byte cp.async per lane instead of bulk copies.  Landmarks whose rows are not one
//                          run fall back to nine 16-byte cp.async per observation; windows with ground-plane rows or several cameras per keyframe (rows
//                          that ADD onto others) take a synchronous variant of the same loop.
//   consumers (12 warps) : Sred += V V^T on the FP64 tensor cores (mma.sync m16n8k8 / m16n8k4: on sm_90 they issue at twice
//                          the FLOP rate of m8n8k4, scripts/dmma_rate.cu).  The whole lower triangle lives in the consumers'
//                          registers as 16x16 blocks, each two 16x8 halves (four shared-memory loads per k-step of both
//                          halves, two for a diagonal block); only the blocks inside the group's 16-row-aligned range are
//                          multiplied, and a half whose 8 columns lie outside the group's exact 8-row tile range is skipped.
//   ring                 : 6 panel stages with full / empty mbarriers, so warps drift up to five groups apart and the
//                          per-group imbalance of the static block -> warp map (scripts/syrk_map_search.py) averages out.
//
// Replaces k_obs_v + k_gp_panel + k_schur_syrk_tma of round 1 (zero-padded panels written and re-read every pass; now 144 B
// per observation).  Forming V inside the producer warps was tried too: with only four warps the ~250 dependent instructions
// per observation are latency-bound next to the tensor work.  Included by kba_kernels.cu after the mbarrier helpers and
// gp_row().
#pragma once

namespace kba {

constexpr int kLG = 8;                           // landmarks per group
constexpr int kGC = 3 * kLG;                     // panel columns per group
constexpr int kFStages = 6;                     // 6 x 37.6 KB: the async copies of up to five groups are in flight
constexpr int kFMaxRs = (kFusedMaxRows + 11) / 16 * 16 + 4;  // row stride == 4 mod 16: 196
constexpr int kFStageDoubles = kGC * kFMaxRs;
constexpr int kFObs = 128;                       // observations staged per group = producer lanes
constexpr int kFConsumerWarps = 12;

// 16x16 block (16 bi + bj: block row bi, block column bj <= bi of the 12-row block triangle; 0xff: none) owned by each
// consumer warp: slot 0 is the warp's block of row 11 (only systems of more than kSixSlotMaxRows rows have one), slots 1..6 blocks of
// rows <= 10.
__constant__ unsigned char kSyrkMap12[12][7] = {
    {0xb6, 0x31, 0x61, 0x75, 0x80, 0x93, 0xaa}, {0xb1, 0x40, 0x42, 0x54, 0x84, 0x98, 0xff}, {0xb7, 0x10, 0x43, 0x52, 0x86, 0x95, 0xff},
    {0xbb, 0x32, 0x60, 0x65, 0x83, 0x99, 0xff}, {0xb9, 0x20, 0x53, 0x76, 0x94, 0xa2, 0xff}, {0xb3, 0x30, 0x62, 0x85, 0xa3, 0xa7, 0xff},
    {0xb0, 0x41, 0x66, 0x74, 0x82, 0xa9, 0xff}, {0xb8, 0x33, 0x55, 0x72, 0x81, 0x97, 0xa0}, {0xb2, 0x00, 0x44, 0x51, 0x73, 0x88, 0x96},
    {0xba, 0x11, 0x63, 0x71, 0x87, 0x90, 0xa5}, {0xb5, 0x22, 0x64, 0x70, 0x91, 0xa1, 0xa8}, {0xb4, 0x21, 0x50, 0x77, 0x92, 0xa4, 0xa6}};

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void cp_async_elem(double* dst, const double* src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_elem(float* dst, const float* src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async16(double* dst, const double* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async8(double* dst, const double* src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
// the mbarrier gets one arrival from this thread once all its earlier cp.async have landed (.noinc: the arrival is part of
// the barrier's expected count)
__device__ __forceinline__ void cp_async_arrive(uint64_t* bar) {
    asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void producer_sync() { asm volatile("bar.sync 1, 128;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void reg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void reg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

// stages, then 24 mbarrier slots, then the dirty-row table (one word per stage and panel column)
constexpr size_t schur_fused_smem() {
    return (size_t)kFStages * kFStageDoubles * sizeof(double) + 24 * sizeof(uint64_t) + kFStages * kGC * sizeof(unsigned);
}
// dirty-row table entry, in double2 rows of a panel column: rows [a, b) and row z (kNoRow: none) may be non-zero
constexpr unsigned kNoRow = 0xff;
__device__ __forceinline__ unsigned dirty_rows(int a, int b, unsigned z) { return (unsigned)a | (unsigned)b << 8 | z << 16; }

// KBA_PROF build: cycles per role (lane 0 of every warp, summed over CTAs into BatchDev::prof) --
//   consumers: [0] waiting for a full panel, [1] multiplying;  producers: [4] waiting for an empty stage, [5] zero fill +
//   copy wait + barrier, [6] scatter + rows + hand-over, [7] (unused)
#ifdef KBA_PROF
#define KBA_PROF_DECL long long pt_ = clock64(), pacc_[3] = {0, 0, 0}
#define KBA_PROF_T0 pt_ = clock64()
#define KBA_PROF_ACC(i) do { const long long n_ = clock64(); pacc_[i] += n_ - pt_; pt_ = n_; } while (0)
#define KBA_PROF_FLUSH(base) do { if (lane == 0 && bd.prof) for (int i_ = 0; i_ < 3; ++i_) atomicAdd(bd.prof + (base) + i_, (unsigned long long)pacc_[i_]); } while (0)
#else
#define KBA_PROF_DECL
#define KBA_PROF_T0
#define KBA_PROF_ACC(i)
#define KBA_PROF_FLUSH(base)
#endif

// Landmark groups per CTA and CTAs that own groups, for a window with n_groups groups in a batch launched with p_split CTAs per
// window.  At least 8 groups per CTA: every CTA writes a whole partial triangle (up to 295 KB) that k_sred_reduce folds again --
// one window alone spread over every SM would leave one partial per SM to fold in every pass.  Because of the floor the partition of a small
// window is the same whether it is solved alone, in a batch or inside the capacity-sized batch of a persistent window
// (kba_track_*), which keeps those paths bit-identical.
__device__ __forceinline__ void schur_split(int n_groups, int p_split, int& per, int& used) {
    per = max(8, (n_groups + p_split - 1) / p_split);
    used = max(1, min(p_split, (n_groups + per - 1) / per));
}

// D += A B on Hopper's 16x8 FP64 shapes (PTX ISA, mma.m16n8k4 / m16n8k8 .f64 fragments): a0 / a1 = rows fr / fr + 8 of A
// in column fc, a2 / a3 the same in column fc + 4; b0 / b1 = rows fc / fc + 4 of B in column fr; c[0..1] = D[fr][2 fc + 0..1],
// c[2..3] = D[fr + 8][2 fc + 0..1].  Both issue at twice the FLOP rate of m8n8k4 on sm_90 (scripts/dmma_rate.cu).
__device__ __forceinline__ void dmma16k4(double (&c)[4], double a0, double a1, double b0) {
    asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};\n"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                 : "d"(a0), "d"(a1), "d"(b0));
}
__device__ __forceinline__ void dmma16k8(double (&c)[4], double a0, double a1, double a2, double a3, double b0, double b1) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                 : "d"(a0), "d"(a1), "d"(a2), "d"(a3), "d"(b0), "d"(b1));
}

// One 16x16 accumulator block += (16 rows at pa) (16 rows at pb)^T over the 24 columns of a group panel (lane offset included,
// column stride kFMaxRs).  c[h] is the 16x8 half of columns pb + 8 h; kL / kR multiply the left / right half.  kRhs: pa is
// the 8-row right-hand-side tile, which lands in the upper (odd == false) or lower 8 rows of the block; the other 8 rows
// get exact zero products.  kK8: three m16n8k8 per half instead of six m16n8k4 (same loads, half the dependent MMAs of an
// accumulator); the seven-slot kernel keeps m16n8k4, its 112 accumulator registers leave no room for the wider fragments.
template <bool kL, bool kR, bool kRhs, bool kK8>
__device__ __forceinline__ void syrk_block(double (&c)[2][4], const double* pa, const double* pb, bool odd) {
    if (kK8 && !kRhs) {
#pragma unroll
        for (int kk = 0; kk < kGC; kk += 8) {
            const double* qa = pa + kk * kFMaxRs;
            const double* qb = pb + kk * kFMaxRs;
            const double a0 = qa[0], a1 = qa[8], a2 = qa[4 * kFMaxRs], a3 = qa[4 * kFMaxRs + 8];
            if (kL) dmma16k8(c[0], a0, a1, a2, a3, qb[0], qb[4 * kFMaxRs]);
            if (kR) dmma16k8(c[1], a0, a1, a2, a3, qb[8], qb[4 * kFMaxRs + 8]);
        }
    } else {
#pragma unroll
        for (int kk = 0; kk < kGC; kk += 4) {
            double a0, a1;
            if (kRhs) {
                const double a = pa[kk * kFMaxRs];
                a0 = odd ? 0.0 : a;
                a1 = odd ? a : 0.0;
            } else {
                a0 = pa[kk * kFMaxRs];
                a1 = pa[kk * kFMaxRs + 8];
            }
            if (kL) dmma16k4(c[0], a0, a1, pb[kk * kFMaxRs]);
            if (kR) dmma16k4(c[1], a0, a1, pb[kk * kFMaxRs + 8]);
        }
    }
}

// the halves of a block that meet the group's exact rows: both, left only or right only
template <bool kRhs, bool kK8>
__device__ __forceinline__ void syrk_halves(double (&c)[2][4], const double* pa, const double* pb, bool odd, bool lo, bool hi) {
    if (lo && hi) syrk_block<true, true, kRhs, kK8>(c, pa, pb, odd);
    else if (lo) syrk_block<true, false, kRhs, kK8>(c, pa, pb, odd);
    else if (hi) syrk_block<false, true, kRhs, kK8>(c, pa, pb, odd);
}

template <int kSlots>
__global__ void __launch_bounds__(512, 1) k_schur_fused(BatchDev bd) {
    const int w = blockIdx.y;
    const WinState& st = bd.state[w];
    if (st.phase != PH_ITERATE || st.solve_failed) return;
    const WinDesc& wd = bd.desc[w];
    if (wd.landmarks_fixed) return;
    extern __shared__ __align__(128) unsigned char fsm[];
    double* stage = reinterpret_cast<double*>(fsm);
    uint64_t* full = reinterpret_cast<uint64_t*>(fsm + (size_t)kFStages * kFStageDoubles * sizeof(double));
    uint64_t* empty = full + kFStages;
    unsigned* dirty = reinterpret_cast<unsigned*>(full + 24);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int n_f = st.n_f, nt = (n_f + 8) >> 3, trhs = n_f >> 3;
    int per, used;
    schur_split(wd.n_groups, (int)gridDim.x, per, used);
    if ((int)blockIdx.x >= used) return;  // k_sred_reduce folds the first `used` partials only
    const int g0 = blockIdx.x * per, g1 = min(wd.n_groups, g0 + per);
    const int* grs = bd.grp_rs + wd.grp_off;
    const int* gt0 = bd.grp_t0 + wd.grp_off;
    const int* gt1 = bd.grp_t1 + wd.grp_off;
    const int* gtl = bd.grp_tiles + wd.grp_off;
    if (tid == 0) {
        for (int i = 0; i < kFStages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], kFConsumerWarps); }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // the barriers are armed by bulk copies (async proxy) too
    }
    // shared memory starts undefined: the first group of every stage zeroes whole columns
    for (int i = tid; i < kFStages * kGC; i += blockDim.x) dirty[i] = dirty_rows(0, kFMaxRs / 2, kNoRow);
    __syncthreads();
    auto next_group = [&](int g) { while (g < g1 && grs[g] == 0) ++g; return g; };

    if (warp >= kFConsumerWarps) {
        // =============================== producers ===============================
        reg_dec<56>();  // 4 x 56 + 12 x 152 = 16 x 128: the consumers' 16x8 accumulators need 152 without spills

        // Each producer warp assembles WHOLE groups on its own (group sequence number gi -> warp gi % 4), so four panels are
        // being built at any time and no CTA-level barrier is needed.  Lane roles inside a warp: lanes 0..23 own one panel
        // column each (landmark lane / 3 of the group, column lane % 3) and fetch it with ONE bulk copy when the landmark's
        // rows form a run (BatchDev::lm_run); lanes 24..31 own the z row of landmark lane - 24.
        // A one-deep register pipeline keeps the next group's meta data in flight (no load result is consumed in the
        // iteration that issues it): P1 = this warp's next group, P0 = the group being assembled.
        const int pw = warp - kFConsumerWarps;
        const int* lm_ptr = bd.lm_ptr + wd.lm_off + w;
        const size_t base = (size_t)wd.obs_off, TG = (size_t)bd.tot_gp;
        const bool sync_path = wd.n_gp > 0 || wd.max_rank > 0;  // rows that ADD onto others cannot be async copies
        const int cj = lane / 3, cc = lane - 3 * cj;  // column lanes
        const int zj = lane - 24;                      // z lanes
        int g1_ = -1, rs1 = 0, t01 = 0, t11 = 0, act1 = 0, p01 = 0, p11 = 0;
        int4 run1 = make_int4(0, 0, 0, 0);
        KBA_PROF_DECL;
        // (gi, g) enumerates the non-empty groups of this CTA in order; the warp takes every 4th
        auto load_meta = [&](int g) {  // P1 loads for group g
            g1_ = g; act1 = 0; run1 = make_int4(0, 0, 0, 0); p01 = p11 = 0;
            if (g >= g1) return;
            rs1 = grs[g]; t01 = gt0[g]; t11 = gt1[g];
            if (lane < 24) {
                const int j = g * kLG + cj;
                if (j < wd.n_lm) { run1 = bd.lm_run[wd.lm_off + j]; p01 = lm_ptr[j]; p11 = lm_ptr[j + 1]; }
            } else {
                const int j = g * kLG + zj;
                if (j < wd.n_lm) { act1 = bd.lm_active[wd.lm_off + j]; p01 = lm_ptr[j]; p11 = lm_ptr[j + 1]; }
            }
        };
        auto nth_group = [&](int g, int n) {  // the n-th non-empty group at or after g (n >= 0), g1 if none
            g = next_group(g);
            for (; n > 0 && g < g1; --n) g = next_group(g + 1);
            return g;
        };
        int g = nth_group(g0, pw), gi = pw;
        load_meta(g);
        while (g < g1) {
            // ---- shift: P1 -> P0, issue the loads of this warp's next group
            const int rs = rs1, t0 = t01, t1 = t11, act0 = act1, p00 = p01, p10 = p11;
            const int4 run0 = run1;
            const int gnext = nth_group(g + 1, 3);
            load_meta(gnext);
            // ---- P0
            const int slot = gi % kFStages;
            KBA_PROF_T0;
            if (gi >= kFStages) mbar_wait(&empty[slot], ((gi / kFStages) - 1) & 1);
            KBA_PROF_ACC(0);
            double* sb = stage + (size_t)slot * kFStageDoubles;
            // does every landmark of the group have its rows in one run that starts on an even panel row?
            const bool no_run = lane < 24 && (run0.y < 0 || (run0.y > 0 && ((run0.z - 8 * t0) & 1)));
            const bool bulk = __ballot_sync(0xffffffffu, no_run) == 0u && !sync_path;
            if (lane < kGC) {
                // The column lane zeroes what the stage's previous group may have left in its column (double2 rows) except
                // the rows [s, e) its own bulk copy overwrites, and records what this group may leave: the run and the z
                // row on the bulk path, every row of the panel (rs rows, a multiple of 8) otherwise.  Each lane stores
                // on its own, so the stores issue back to back.  The table word was written before the previous group's
                // "full" arrival and is read after this stage's "empty" wait, the same hand-over as the panel itself.
                unsigned* dl = dirty + slot * kGC + lane;
                const unsigned d = *dl;
                int s = 0, e = 0;
                if (bulk && run0.y > 0) { s = (run0.z - 8 * t0) >> 1; e = s + 3 * run0.y; }
                const int zl = (trhs >= t0 && trhs < t1) ? n_f - 8 * t0 : 8 * (t1 - t0) + (n_f - 8 * trhs);  // z row rl below
                *dl = bulk ? dirty_rows(s, e, (unsigned)(zl >> 1)) : dirty_rows(0, rs >> 1, kNoRow);
                const int a = d & 0xff, b = (d >> 8) & 0xff, z = d >> 16;
                const bool zero_z = z != (int)kNoRow && (z < a || z >= b) && (z < s || z >= e);
                const int m1 = min(b, s), m2 = max(a, e);
                double2* col = reinterpret_cast<double2*>(sb + (size_t)lane * kFMaxRs);
                if (zero_z) col[z] = make_double2(0.0, 0.0);
                for (int r2 = a; r2 < m1; ++r2) col[r2] = make_double2(0.0, 0.0);
                for (int r2 = m2; r2 < b; ++r2) col[r2] = make_double2(0.0, 0.0);
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // the zeros (generic proxy) before the bulk copies (async proxy)
            __syncwarp();
            KBA_PROF_ACC(1);
            const int j0 = g * kLG, j1 = min(wd.n_lm, j0 + kLG);
            const int ob = lm_ptr[j0], oe = lm_ptr[j1];
            const int rl = (trhs >= t0 && trhs < t1) ? n_f - 8 * t0 : 8 * (t1 - t0) + (n_f - 8 * trhs);  // t0, t1: block aligned
            if (bulk) {
                if (lane < 24 && run0.y > 0) {  // one bulk copy: the landmark's column, 6 rows per observation of the run
                    const uint32_t bytes = (uint32_t)(48 * run0.y);
                    asm volatile("mbarrier.expect_tx.relaxed.cta.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(&full[slot])), "r"(bytes) : "memory");
                    tma_load_1d(sb + (size_t)(3 * cj + cc) * kFMaxRs + (run0.z - 8 * t0),
                                bd.vobs + vobs_index(base, p00, p10, p00 + run0.x, cc), bytes, &full[slot]);
                }
            } else {  // per observation: nine 16-byte (or eighteen 8-byte) async copies
                for (int o = ob + lane; o < oe; o += 32) {
                    const size_t oo = base + o;
                    const int row = bd.obs_row[oo];
                    if (row < 0 || bd.obs_rank[oo] != 0) continue;
                    const int lm = bd.obs_lm[oo], q0 = lm_ptr[lm], q1 = lm_ptr[lm + 1];
                    double* dst = sb + (size_t)(3 * (lm - j0)) * kFMaxRs + (row - 8 * t0);
#pragma unroll
                    for (int c = 0; c < 3; ++c) {
                        const double* src = bd.vobs + vobs_index(base, q0, q1, o, c);
                        if (((row - 8 * t0) & 1) == 0) {
#pragma unroll
                            for (int h = 0; h < 3; ++h) cp_async16(dst + c * kFMaxRs + 2 * h, src + 2 * h);
                        } else {
#pragma unroll
                            for (int r = 0; r < 6; ++r) cp_async8(dst + c * kFMaxRs + r, src + r);
                        }
                    }
                }
            }
            if (lane >= 24 && act0 && p10 > p00) {  // right-hand-side row z_j
                const double* zz = bd.lm_z + 3 * (size_t)(wd.lm_off + j0 + zj);
                double* col = sb + (size_t)(3 * zj) * kFMaxRs + rl;
                cp_async8(col, zz); cp_async8(col + kFMaxRs, zz + 1); cp_async8(col + 2 * kFMaxRs, zz + 2);
            }
            if (!sync_path) {
                // every lane: "count my outstanding cp.async into this phase" (increments the pending count now, decrements on
                // completion); then ONE arrival per warp -- the phase completes when the copies and the bulk bytes have landed
                asm volatile("cp.async.mbarrier.arrive.shared::cta.b64 [%0];" ::"r"(smem_u32(&full[slot])) : "memory");
                __syncwarp();
                if (lane == 0) mbar_arrive(&full[slot]);
            } else {
                cp_async_commit();
                cp_async_wait<0>();
                __syncwarp();
                for (int round = 1; round <= wd.max_rank; ++round) {  // further cameras of a rig: add onto the same rows
                    for (int o = ob + lane; o < oe; o += 32) {
                        const size_t oo = base + o;
                        const int row = bd.obs_row[oo];
                        if (row < 0 || bd.obs_rank[oo] != round) continue;
                        const int lm = bd.obs_lm[oo], q0 = lm_ptr[lm], q1 = lm_ptr[lm + 1];
                        double* dst = sb + (size_t)(3 * (lm - j0)) * kFMaxRs + (row - 8 * t0);
                        for (int c = 0; c < 3; ++c) {
                            const double* src = bd.vobs + vobs_index(base, q0, q1, o, c);
                            for (int r = 0; r < 6; ++r) dst[c * kFMaxRs + r] += src[r];
                        }
                    }
                    __syncwarp();
                }
                if (wd.n_gp > 0) {  // ground-plane rows: 8 landmarks x 10 rows, added onto the pose rows
                    for (int it = lane; it < 80; it += 32) {
                        const int jj = it / 10, r = it - 10 * jj, j = j0 + jj;
                        const int L = wd.lm_off + j;
                        if (j >= wd.n_lm || !bd.lm_active[L] || lm_ptr[j + 1] <= lm_ptr[j]) continue;
                        const int gl = bd.gp_of_lm[L];
                        if (gl < 0) continue;
                        const size_t G = (size_t)wd.gp_off + gl;
                        const int row = gp_row(bd, wd, bd.gp_kf[G], r);
                        if (row < 0) continue;
                        double* q = sb + (size_t)(3 * jj) * kFMaxRs + (row - 8 * t0);
                        q[0] += bd.vgp[(3 * r + 0) * TG + G];
                        q[kFMaxRs] += bd.vgp[(3 * r + 1) * TG + G];
                        q[2 * kFMaxRs] += bd.vgp[(3 * r + 2) * TG + G];
                    }
                }
                __syncwarp();  // the warp's panel writes are ordered before lane 0's releasing arrival
                if (lane == 0) mbar_arrive(&full[slot]);
            }
            KBA_PROF_ACC(2);
            g = gnext; gi += 4;
        }
        cp_async_commit();
        cp_async_wait<0>();
        KBA_PROF_FLUSH(4);
        return;
    }

    // =============================== consumers ===============================
    reg_inc<152>();
    const int fr = lane >> 2, fc = lane & 3;
    const int nb2 = (nt + 1) >> 1, brhs = trhs >> 1;
    double acc[kSlots][2][4];  // [slot][column half][rows fr: 0..1, rows fr + 8: 2..3]
    const unsigned char* my_b = kSyrkMap12[warp] + (7 - kSlots);  // read in the group loop: the registers go to the accumulators
#pragma unroll
    for (int s = 0; s < kSlots; ++s)
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[s][0][q] = acc[s][1][q] = 0.0;
    {
        // Group ranges are aligned to 16-row blocks (k_solve_begin), so a block inside the range has both its row tiles, and
        // the only partial row block is the one holding the right-hand-side tile when it lies outside the range.  On the
        // column side a block is two 16x8 products, and a half whose 8 rows lie outside the group's exact tile range
        // [e0, e1) is zero in the panel and skipped.  Straight-line variants, no predicate inside a tensor-core loop; the
        // column stride is the constant kFMaxRs, so every fragment load of a block is base + immediate.  A diagonal block
        // passes the same pointer twice, so its B fragments are its A fragments (two loads per k-step instead of four).
        int gi = 0;
        int g = next_group(g0), tiles = 0;
        if (g < g1) tiles = gtl[g];
        KBA_PROF_DECL;
        for (; g < g1; ++gi) {
            const int gn = next_group(g + 1);  // the next group's range is requested before this group's panel is awaited
            const int tiles_n = gn < g1 ? gtl[gn] : 0;
            const int slot = gi % kFStages;
            KBA_PROF_T0;
            mbar_wait(&full[slot], (gi / kFStages) & 1);
            KBA_PROF_ACC(0);
            const int b0 = (tiles & 255) >> 1, b1 = ((tiles >> 8) & 255) >> 1;  // block range [b0, b1) of the group
            const int e0 = (tiles >> 16) & 255, e1 = tiles >> 24;                // exact tile range [e0, e1)
            const bool rhs_in = brhs >= b0 && brhs < b1;
            const int rhs_row = 16 * (b1 - b0);  // panel row of the rhs tile when it lies outside the range
            const double* sb = stage + (size_t)slot * kFStageDoubles + (size_t)fc * kFMaxRs + fr;
#pragma unroll
            for (int s = 0; s < kSlots; ++s) {
                const int b = my_b[s], bi = b >> 4, bj = b & 15;
                if (bj < b0 || bj >= b1) continue;
                const bool lo = 2 * bj >= e0, hi = 2 * bj + 1 < e1;  // column halves inside the exact range
                const double* pb = sb + 16 * (bj - b0);
                if (bi == bj) syrk_halves<false, kSlots == 6>(acc[s], pb, pb, false, lo, hi);
                else if (bi >= b0 && bi < b1) syrk_halves<false, kSlots == 6>(acc[s], sb + 16 * (bi - b0), pb, false, lo, hi);
                else if (bi == brhs && !rhs_in) syrk_halves<true, false>(acc[s], sb + rhs_row, pb, trhs & 1, lo, hi);
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[slot]);
            KBA_PROF_ACC(1);
            g = gn; tiles = tiles_n;
        }
        KBA_PROF_FLUSH(0);
    }
    double* out = bd.sred + wd.s_off * (size_t)bd.p_split + (size_t)blockIdx.x * wd.nr_cap * wd.nr_cap;
#pragma unroll
    for (int s = 0; s < kSlots; ++s) {
        const int b = my_b[s], bi = b >> 4, bj = b & 15;
        if (bi >= nb2) continue;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int i = 2 * bi + (q >> 1), j = 2 * bj + (q & 1);
            if (i >= nt || j > i) continue;
            double* o = out + (size_t)(8 * i + fr) * wd.nr_cap + 8 * j + 2 * fc;
            o[0] = acc[s][q & 1][2 * (q >> 1)];
            o[1] = acc[s][q & 1][2 * (q >> 1) + 1];
        }
    }
}

}  // namespace kba
