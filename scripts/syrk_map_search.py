#!/usr/bin/env python
"""Offline search of the static block -> warp map of k_schur_fused (limo_b200/csrc/kba_schur_fused.cuh).

The kernel keeps the lower triangle of the reduced system as 16x16 accumulator blocks in the registers of 12 consumer
warps (3 per SM sub-partition), so ownership is static.  A landmark group (8 landmarks) only touches the blocks inside
its keyframe row range plus the right-hand-side row; the FP64 tensor pipe is per sub-partition, so what a stage costs
is the MMA count of its busiest sub-partition.  A block is two 16x8 halves (mma.m16n8k4, 6 k-steps per group): a block
costs its halves whose 8 columns meet the group's exact 8-row tile range, when its rows lie in the group's 16-row-aligned
block range or hold the right-hand-side tile outside it.  The ring lets warps drift a few stages, so the long-run totals count
too.  Objective: sum over groups of the busiest sub-partition + the long-run maximum, on config-2 windows (29 free
keyframes) and on 30-free-keyframe windows (184 rows).

  python scripts/syrk_map_search.py  -> prints the table for kSyrkMap12
"""
import random
import sys

import numpy as np

sys.path.insert(0, ".")
from limo_b200 import synth  # noqa: E402

NW, NSLOT, NB = 12, 7, 12
BLOCKS = [(bi, bj) for bi in range(NB) for bj in range(bi + 1)]  # linear id bi(bi+1)/2+bj


def groups_of(win, fixed_first):
    """(t0, t1, trhs, nt) per 8-landmark group of a window, landmarks sorted by (first, last) keyframe"""
    ptr, kf = win.lm_obs_ptr, win.obs_kf
    first = np.array([kf[ptr[j]] if ptr[j + 1] > ptr[j] else win.n_kf for j in range(win.n_lm)])
    last = np.array([kf[ptr[j + 1] - 1] if ptr[j + 1] > ptr[j] else win.n_kf for j in range(win.n_lm)])
    order = np.lexsort((last, first))
    n_free = win.n_kf - (1 if fixed_first else 0)
    n_f = 6 * n_free
    off = lambda k: 6 * (k - 1) if fixed_first else 6 * k
    out = []
    for g0 in range(0, win.n_lm, 8):
        js = order[g0:g0 + 8]
        ks = [k for j in js for k in (first[j], last[j]) if k < win.n_kf]
        ks = [k for k in ks if not (fixed_first and k == 0)] or []
        if not ks:
            continue
        k0, k1 = min(ks), max(ks)
        r0, r1 = off(k0), off(k1) + 6
        out.append((r0 // 8, (r1 + 7) // 8, n_f >> 3, (n_f + 1 + 7) >> 3))
    return out


def block_cost(bi, bj, t0, t1, trhs):
    """m16n8k4 MMAs of one 16x16 block for a group with exact tile range [t0, t1) (6 k-steps of 4 columns)"""
    b0, b1 = t0 // 2, (t1 + 1) // 2                   # 16-row-aligned block range
    rhs_in = b0 <= trhs // 2 < b1
    e1 = max(t1, trhs + 1) if rhs_in else t1           # the rhs tile is part of the exact range when inside the blocks
    if not b0 <= bj < b1 or not (b0 <= bi < b1 or (bi == trhs // 2 and not rhs_in)):
        return 0
    return 6 * (int(2 * bj >= t0) + int(2 * bj + 1 < e1))


def build_costs(groups):
    C = np.zeros((len(groups), len(BLOCKS)), dtype=np.int32)
    for gi, (t0, t1, trhs, nt) in enumerate(groups):
        nb2 = (nt + 1) // 2
        for b, (bi, bj) in enumerate(BLOCKS):
            if bi < nb2:
                C[gi, b] = block_cost(bi, bj, t0, t1, trhs)
    return C


def score(owner, C):
    W = np.zeros((C.shape[0], NW), dtype=np.int64)
    for w in range(NW):
        W[:, w] = C[:, owner == w].sum(axis=1)
    S = W[:, 0:4] + W[:, 4:8] + W[:, 8:12]      # sub-partition = warp % 4
    per_stage = S.max(axis=1).sum()
    longrun = S.sum(axis=0).max() * 1.0
    ideal = C.sum() / 4.0
    warp_stage = W.max(axis=1).sum() * 4.0 / 3.0  # a warp alone can use its sub-partition
    return 0.6 * per_stage / ideal + 0.3 * longrun / ideal + 0.1 * warp_stage / (C.sum() / 3.0 / 4.0 * 4.0 / 3.0 * 3.0), per_stage / ideal, longrun / ideal


def main():
    rng = random.Random(1)
    groups = []
    for seed in (1, 2, 3):
        groups += groups_of(synth.make_window(2, seed=seed), True)
    g30 = []
    for seed in (4,):
        g30 += groups_of(synth.make_window(2, seed=seed), False)
    C = np.concatenate([build_costs(groups), build_costs(g30)[::3]])
    print("groups", C.shape[0], "mean MMA per group", C.sum() / C.shape[0])
    # start: rows dealt cyclically with a skew; every warp gets exactly one block of row 11 and at most one of row 10
    owner = np.zeros(len(BLOCKS), dtype=np.int64)
    cnt = [0] * NW
    for b, (bi, bj) in enumerate(BLOCKS):
        if bi == 11:
            owner[b] = bj
        else:  # least loaded warp, ties broken by a skewed cyclic order
            w = min(range(NW), key=lambda w: (cnt[w], (w - 5 * bi - bj) % NW))
            owner[b] = w
            cnt[w] += 1
    cap = lambda ow: np.bincount(ow, minlength=NW).max() <= NSLOT
    row11 = [b for b, (bi, bj) in enumerate(BLOCKS) if bi == 11]
    low = [b for b, (bi, bj) in enumerate(BLOCKS) if bi <= 10]

    def ok(ow):
        if not cap(ow):
            return False
        if len(set(ow[row11])) != 12:
            return False
        return np.bincount(ow[low], minlength=NW).max() <= NSLOT - 1  # rows <= 10 fit 6 slots
    assert ok(owner), np.bincount(owner)
    best, pb, lb = score(owner, C)
    for it in range(30000):
        a, b = rng.sample(range(len(BLOCKS)), 2)
        if owner[a] == owner[b]:
            continue
        ow = owner.copy()
        ow[a], ow[b] = ow[b], ow[a]
        if not ok(ow):
            continue
        s, p, l = score(ow, C)
        if s < best:
            owner, best, pb, lb = ow, s, p, l
            if it % 50 == 0:
                print(it, "score %.4f per-stage %.4f long-run %.4f" % (best, pb, lb), flush=True)
    print("final: per-stage busiest-subpartition / ideal = %.4f, long-run = %.4f" % (pb, lb))
    # slot 0 = the warp's row-11 block, slots 1..6 = blocks of rows <= 10 (0xff padded), as 16 bi + bj
    code = lambda b: "0x%02x" % (16 * BLOCKS[b][0] + BLOCKS[b][1])
    print("__constant__ unsigned char kSyrkMap12[12][7] = {")
    for w in range(NW):
        r11 = [code(b) for b in row11 if owner[b] == w]
        rest = [code(b) for b in low if owner[b] == w]
        row = r11 + rest + ["0xff"] * (NSLOT - 1 - len(rest))
        print("    {%s}," % ", ".join(row))
    print("};")


if __name__ == "__main__":
    main()
