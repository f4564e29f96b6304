// kba_controller.cuh -- the decisions of the window solver, shared by the batch kernels (k_lm_update, k_trim_select in
// kba_kernels.cu) and the one-CTA motion-only kernel (k_adjust_pose in kba_motion.cu):
//   - the LM controller: ceres 1.13 TrustRegionMinimizer + LevenbergMarquardtStrategy as restated in SURVEY.md A.6, and the
//     solveTrimmed outer loop (reference robust_solving.cpp:140-248);
//   - the quantile trimming of one residual group by exact rank (reference robust_solving.cpp:67-125, trimmer_quantile.hpp:40-63).
// Neither touches BatchDev: the callers reduce their own partial sums and pass the scalars.
#pragma once
#include <cfloat>

#include "kba_device.cuh"

namespace kba {

// one iteration record into a window's log (kIterLogCap entries)
__device__ inline void log_iter(IterRecord* log, WinState& st, double cost, double cost_change, double gmax, double step_norm,
                                double rel, double radius, int valid, int successful) {
    if (st.log_n >= kIterLogCap) return;
    IterRecord& e = log[st.log_n++];
    e.cost = cost; e.cost_change = cost_change; e.gradient_max_norm = gmax; e.step_norm = step_norm;
    e.relative_decrease = rel; e.radius = radius; e.iteration = st.iteration; e.solve_index = st.solve_index;
    e.valid = valid; e.successful = successful;
}

// end of one inner solve: the final solve ends the window, a trimming-round solve that did not decrease the cost is retried
// once with three times the iterations (robust_solving.cpp:172-181), otherwise the next trimming step follows
__device__ inline void solve_end(WinState& st, int termination) {
    SolveSummary& s = st.solves[st.solve_index];
    s.termination = termination;
    s.num_iterations = st.iteration;
    st.n_solves = st.solve_index + 1;
    if (st.is_final) { st.phase = PH_DONE; return; }
    if (s.initial_cost - s.final_cost <= 0.0 && !st.retried) {
        st.retried = 1;
        st.phase = PH_SOLVE_BEGIN;
        return;
    }
    st.phase = PH_TRIM;
}

// One controller step of a window in PH_ITERATE, after the pass has (re-)linearised if st.need_linearize, solved for the step
// (st.f_* = pose-side scalars, st.solve_failed) and evaluated the candidate (st.eval_failed = the candidate failed to evaluate).
//   e_model, e_step, e_xn, e_g: the landmark side's model decrease, squared step, squared state norm and gradient max-norm;
//   may_time: max_solver_time applies (not in a sharded solve: the ranks' clocks differ);
//   carry_cost: the accepted candidate's cost is the next x's cost (the linearisation evaluates the cost at iteration zero only);
//   cand_cost(): the candidate's total cost, observations and regularisers -- called only when the step is valid.
template <typename CandCost>
__device__ inline void lm_step(WinState& st, IterRecord* log, const SolveParams& sp, bool may_time, bool carry_cost, double e_model,
                               double e_step, double e_xn, double e_g, CandCost cand_cost) {
    SolveSummary& sum = st.solves[st.solve_index];
    if (st.solve_failed == 2) {  // evaluation failed at iteration zero
        sum.initial_cost = sum.final_cost = -1.0;
        st.solve_failed = 0; st.eval_failed = 0;
        solve_end(st, 2);
        return;
    }
    const int cand_eval_failed = st.eval_failed;  // set by the candidate cost pass of THIS pass (|z| < 0.01)
    st.eval_failed = 0;
    const bool step_ok = !st.solve_failed;
    if (st.need_linearize) {  // a fresh linearisation was evaluated in this pass
        if (step_ok || st.iter0) {
            st.gmax = fmax(st.f_gmax, e_g);
            st.x_norm = sqrt(st.f_xnorm_sq + e_xn);
        }
        if (st.iter0) {
            sum.initial_cost = sum.final_cost = st.x_cost;
            log_iter(log, st, st.x_cost, 0, st.gmax, 0, 0, st.radius, 0, 0);
        } else {
            if (st.x_cost < sum.final_cost) sum.final_cost = st.x_cost;
            // complete the record of the successful iteration that led here
            if (st.log_n > 0) {
                IterRecord& e = log[st.log_n - 1];
                e.cost = st.x_cost; e.gradient_max_norm = st.gmax;
            }
        }
    }
    // ---- loop head of the next iteration (FinalizeIterationAndCheckIfMinimizerCanContinue) ----
    if (st.iteration >= st.max_iter) { st.solve_failed = 0; solve_end(st, 1); return; }
    // max_solver_time_in_seconds of THIS inner solve (robust_solving.cpp:233-238 sets it per ceres::Solve): NO_CONVERGENCE, the
    // accepted iterate stands and solveTrimmed goes on to its next solve
    if (sp.max_solver_time > 0 && may_time &&
        (double)(global_timer_ns() - st.t_solve_start) * 1e-9 >= sp.max_solver_time) { st.solve_failed = 0; solve_end(st, 1); return; }
    if (st.last_successful && st.gmax <= sp.gradient_tolerance) { st.solve_failed = 0; solve_end(st, 0); return; }
    if (st.radius <= sp.min_radius) { st.solve_failed = 0; solve_end(st, 0); return; }
    st.iteration++;
    st.last_successful = 0;
    // ---- step validity ----
    const double model_change = 0.5 * (st.f_model + e_model);
    const bool valid = step_ok && isfinite(model_change) && model_change > 0.0;
    if (!valid) {
        st.solve_failed = 0;
        if (++st.num_invalid >= sp.max_consecutive_invalid_steps) { solve_end(st, 2); return; }
        st.radius /= st.decrease_factor; st.decrease_factor *= 2.0;
        st.need_linearize = 0; st.iter0 = 0;
        log_iter(log, st, st.x_cost, 0, st.gmax, 0, 0, st.radius, 0, 0);
        return;
    }
    st.num_invalid = 0;
    // ---- candidate cost ----
    double cand = cand_cost();
    if (cand_eval_failed) cand = DBL_MAX;  // "Step failed to evaluate": infinite cost -> rejected
    const double step_norm = sqrt(st.f_step_sq + e_step);
    if (step_norm <= sp.parameter_tolerance * (st.x_norm + sp.parameter_tolerance)) {
        log_iter(log, st, st.x_cost, 0, st.gmax, step_norm, 0, st.radius, 1, 0);
        solve_end(st, 0);
        return;
    }
    const double cost_change = st.x_cost - cand;
    if (fabs(cost_change) <= sp.function_tolerance * st.x_cost) {
        log_iter(log, st, st.x_cost, cost_change, st.gmax, step_norm, 0, st.radius, 1, 0);
        solve_end(st, 0);
        return;
    }
    const double rel = cost_change / model_change;
    if (rel > sp.min_relative_decrease) {
        st.cur = 1 - st.cur;
        st.need_linearize = 1; st.iter0 = 0; st.last_successful = 1;
        if (carry_cost) st.x_cost = cand;  // the accepted candidate is the next x: its cost is known (ceres: x_cost = candidate_cost)
        sum.num_successful_steps++;
        const double t = 2.0 * rel - 1.0;
        st.radius = fmin(sp.max_radius, st.radius / fmax(1.0 / 3.0, 1.0 - t * t * t));
        st.decrease_factor = 2.0;
        log_iter(log, st, cand, cost_change, st.gmax, step_norm, rel, st.radius, 1, 1);
    } else {
        st.radius /= st.decrease_factor; st.decrease_factor *= 2.0;
        st.need_linearize = 0; st.iter0 = 0;
        log_iter(log, st, cand, cost_change, st.gmax, step_norm, rel, st.radius, 1, 0);
    }
}

// end of a trimming step: the next inner solve begins (the last one is the final refinement)
__device__ inline void trim_advance(WinState& st) {
    st.round++;
    st.retried = 0;
    st.solve_index++;
    st.is_final = (st.round >= st.rounds_total) || (st.solve_index >= 7);
    st.phase = PH_SOLVE_BEGIN;
}

// shared memory of trim_select_group
struct TrimSmem {
    int n;
    unsigned hist[256];
    unsigned long long prefix;
    int k;
};

// Quantile rejection of ONE residual group by exact rank (ties broken by the caller's landmark index), block-cooperative (any
// block size that is a multiple of 32): every thread of the block calls it with the same arguments.  val(j) is item j's
// value (< 0: the item has no residual of this group), oid(j) its tie-break index; rejected items get rej[j] = 1, the others
// are left as they are.  The value of rank `num` (the smallest rejected one) is found with an 8-pass MSB-first radix select
// over the IEEE bit patterns (non-negative doubles order like unsigned integers); only exact ties with it need the O(n)
// index count.
template <typename Val, typename Oid>
__device__ inline void trim_select_group(TrimSmem& sm, int n_items, double quant, int min_residual_groups, Val val, Oid oid,
                                         uint8_t* rej) {
    if (threadIdx.x == 0) sm.n = 0;
    __syncthreads();
    int cnt = 0;
    for (int j = threadIdx.x; j < n_items; j += blockDim.x) cnt += (val(j) >= 0.0);
    if (cnt) atomicAdd(&sm.n, cnt);
    __syncthreads();
    const int N = sm.n;
    __syncthreads();
    if (N == 0 || N < min_residual_groups) return;
    const int num = (int)((double)N * quant);
    if (num >= N) return;
    if (threadIdx.x == 0) { sm.prefix = 0ull; sm.k = num; }
    unsigned long long mask = 0ull;
    constexpr unsigned long long kInvalid = ~0ull;  // not a non-negative double
    auto load_key = [&](int j) -> unsigned long long {
        const double vj = (j < n_items) ? val(j) : -1.0;
        return (vj >= 0.0) ? ((unsigned long long)__double_as_longlong(vj) & 0x7fffffffffffffffull) : kInvalid;
    };
    // up to 8 keys per thread stay in registers over the 8 passes (a 512-thread block: windows of <= 4096 landmarks, every key)
    unsigned long long kreg[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) kreg[q] = load_key(threadIdx.x + q * (int)blockDim.x);
    const int n_reg = 8 * (int)blockDim.x;
    for (int shift = 56; shift >= 0; shift -= 8) {
        for (int i = threadIdx.x; i < 256; i += blockDim.x) sm.hist[i] = 0u;
        __syncthreads();
        const unsigned long long prefix = sm.prefix;
        auto count = [&](unsigned long long key) {  // every lane of the warp calls this (warp vote inside)
            const bool in = key != kInvalid && (key & mask) == prefix;
            // the leading bytes are nearly constant (exponent): aggregate equal bins inside the warp first
            const unsigned bin = in ? (unsigned)((key >> shift) & 255ull) : 256u;
            const unsigned peers = __match_any_sync(0xffffffffu, bin);
            if (in && (threadIdx.x & 31) == (unsigned)(__ffs(peers) - 1)) atomicAdd(&sm.hist[bin], (unsigned)__popc(peers));
        };
#pragma unroll
        for (int q = 0; q < 8; ++q) count(kreg[q]);
        for (int j0 = n_reg; j0 < n_items; j0 += 4 * blockDim.x) {  // larger windows: 4 independent loads per round
            unsigned long long k4[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) k4[q] = load_key(j0 + q * (int)blockDim.x + threadIdx.x);
#pragma unroll
            for (int q = 0; q < 4; ++q) count(k4[q]);
        }
        __syncthreads();
        if (threadIdx.x < 32) {  // warp 0 finds the bin holding rank sm.k: 8 bins per lane, shuffle prefix sum
            const int lane = threadIdx.x;
            unsigned h[8], tot = 0;
#pragma unroll
            for (int q = 0; q < 8; ++q) { h[q] = sm.hist[8 * lane + q]; tot += h[q]; }
            unsigned incl = tot;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const unsigned up = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += up;
            }
            const unsigned k = (unsigned)sm.k, excl = incl - tot;
            const bool mine = k >= excl && k < incl;  // exactly one lane (k < total count)
            if (mine) {
                unsigned rem = k - excl;
                int q = 0;
                for (; q < 7; ++q) { if (rem < h[q]) break; rem -= h[q]; }
                sm.k = (int)rem;
                sm.prefix = prefix | ((unsigned long long)(8 * lane + q) << shift);
            }
        }
        mask |= 255ull << shift;
        __syncthreads();
    }
    const unsigned long long pivot = sm.prefix;  // bit pattern of the value with rank `num`
    const int tie_keep = sm.k;                   // ties with fewer than tie_keep smaller-index ties stay
    // how many values equal the pivot?  Normally one (the pivot itself): then the O(n) index count below -- one thread walking
    // every value -- is not needed
    __syncthreads();
    if (threadIdx.x == 0) sm.n = 0;
    __syncthreads();
    {
        int ties = 0;
        for (int j = threadIdx.x; j < n_items; j += blockDim.x) {
            const double vj = val(j);
            if (vj >= 0.0) ties += (((unsigned long long)__double_as_longlong(vj) & 0x7fffffffffffffffull) == pivot);
        }
        if (ties) atomicAdd(&sm.n, ties);
    }
    __syncthreads();
    const int n_ties = sm.n;
    for (int j = threadIdx.x; j < n_items; j += blockDim.x) {
        const double vj = val(j);
        if (!(vj >= 0.0)) continue;
        const unsigned long long key = (unsigned long long)__double_as_longlong(vj) & 0x7fffffffffffffffull;
        if (key < pivot) continue;
        bool reject = key > pivot;
        if (!reject) {
            const int oj = oid(j);
            int before = 0;
            for (int k = 0; k < (n_ties > 1 ? n_items : 0); ++k) {
                const double vk = val(k);
                if (!(vk >= 0.0)) continue;
                const unsigned long long kk = (unsigned long long)__double_as_longlong(vk) & 0x7fffffffffffffffull;
                before += (kk == pivot && oid(k) < oj);
            }
            reject = before >= tie_keep;
        }
        if (reject) rej[j] = 1;
    }
    __syncthreads();
}

}  // namespace kba
