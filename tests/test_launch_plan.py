"""The launch plan of a batch (limo_b200/csrc/kba_plan.h) on the CPU: which solver path, Schur kernel instance, Schur split,
factorisation and packing a window shape selects.

A small driver compiled against the header alone answers queries on stdin.  Every expected value below was read from the rules
as kba_batch_create, kba_batch_upload and the track solve stated them before they moved into the header (132 SMs, as on an
H100 SXM), so a change to any rule fails here before it changes the rounding of a solve.
"""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SM = 132

DRIVER = r"""
#include <cstdio>
#include <cstring>
#include <vector>
#include "kba_plan.h"
using namespace kba;

static void print(const Plan& p) {
    printf("%d %d %d %d %d %d %d %d %d\n", p.nr_cap_max, p.small_syrk, p.fused, p.fused_slots, p.p_split, p.p_split_cap,
           p.solve_tiled, p.solve_split, p.device_pack);
}
static std::vector<WinShape> shapes(int n) {
    std::vector<WinShape> w(n);
    for (auto& s : w)
        if (scanf("%d %d %d %d %d", &s.rows, &s.free_rows, &s.n_chunks, &s.n_groups, &s.n_lm) != 5) s = WinShape{};
    return w;
}
int main() {
    char op[16];
    while (scanf("%15s", op) == 1) {
        if (!strcmp(op, "knobs")) {
            const Knobs k = read_knobs();
            printf("%d %d %d %d %d %d %d\n", k.fused, k.lin_fused, k.p_split, k.lin_grid, k.bs_grid, k.solve_split, k.device_pack);
        } else if (!strcmp(op, "plan") || !strcmp(op, "replan")) {
            int purpose = 0, n = 0, sm = 0;
            Knobs k;
            if (scanf("%d %d %d %d %d %d %d", &purpose, &n, &sm, &k.fused, &k.p_split, &k.solve_split, &k.device_pack) != 7) return 1;
            const std::vector<WinShape> w = shapes(n);
            Plan p = make_plan(w.data(), n, sm, k, (Purpose)purpose);
            if (!strcmp(op, "replan")) {
                const std::vector<WinShape> solved = shapes(n);
                replan_large(p, solved.data(), n, sm, k);
            }
            print(p);
        } else if (!strcmp(op, "rows")) {
            int n_kf = 0, planes = 0;
            if (scanf("%d %d", &n_kf, &planes) != 2) return 1;
            printf("%d\n", reduced_rows(n_kf, planes != 0));
        } else if (!strcmp(op, "slots")) {
            int free_rows = 0;
            if (scanf("%d", &free_rows) != 1) return 1;
            printf("%d\n", fused_slots(free_rows));
        } else {
            return 1;
        }
    }
    return 0;
}
"""

FIELDS = ("nr_cap_max", "small_syrk", "fused", "fused_slots", "p_split", "p_split_cap", "solve_tiled", "solve_split", "device_pack")
PURPOSE = {"batch": 0, "track_fused": 1, "track_large": 2, "host_pack": 3}
KNOBS = ("KBA_FUSED", "KBA_LINEARIZE", "KBA_P_SPLIT", "KBA_LIN_GRID", "KBA_BS_GRID", "KBA_SOLVE_SPLIT", "KBA_DEVICE_PACK")


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    d = tmp_path_factory.mktemp("plan")
    (d / "plan.cpp").write_text(DRIVER)
    exe = d / "plan"
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-Wall", "-Werror", "-I", os.path.join(ROOT, "limo_b200", "csrc"),
                           str(d / "plan.cpp"), "-o", str(exe)])

    def run(text, env=None):
        e = {k: v for k, v in os.environ.items() if k not in KNOBS}
        e.update(env or {})
        return subprocess.run([str(exe)], input=text, capture_output=True, text=True, env=e, check=True).stdout.split("\n")
    return run


def win(n_kf, n_lm=3000, fixed=1, planes=False, rows=None, free_rows=None):
    """(rows, free rows, 32-landmark chunks, 8-landmark groups, landmarks) of a window as kba_batch_create sizes it: 6 rows per
    keyframe, 10 with plane blocks, plus one -- over all keyframes for the path (or a track's own rows), over the free ones for
    the Schur kernel instance"""
    per = 10 if planes else 6
    return (per * n_kf + 1 if rows is None else rows, per * (n_kf - fixed) + 1 if free_rows is None else free_rows,
            -(-n_lm // 32), -(-n_lm // 8), n_lm)


def _query(op, windows, purpose, fused, p_split, device_pack, solve_split=-1, solved=None):
    head = "%s %d %d %d %d %d %d %d" % (op, PURPOSE[purpose], len(windows), SM, fused, p_split, solve_split, device_pack)
    return " ".join([head] + ["%d %d %d %d %d" % w for w in windows + (solved or [])])


CONFIG2 = win(30)                            # synth config 2: 30 keyframes, keyframe 0 fixed, 3000 landmarks
CONFIG3 = win(30, planes=True)               # the same with ground-plane blocks: 301 rows
LARGE_TRACK = win(30, n_lm=2000, planes=True, rows=301)   # capacity window of a win_rows = 301 track's large solver

# name -> (windows, purpose, KBA_FUSED, KBA_P_SPLIT, KBA_DEVICE_PACK, the plan fields that are asserted)
CASES = {
    # the path: every window within 184 rows over all its keyframes
    "config2_batch1": ([CONFIG2], "batch", 1, 0, 1, dict(nr_cap_max=192, small_syrk=1, fused=1, fused_slots=6, p_split=132,
                                                          solve_tiled=1, solve_split=0, device_pack=1)),
    "config2_batch264": ([CONFIG2] * 264, "batch", 1, 0, 1, dict(fused=1, fused_slots=6, p_split=1, solve_tiled=1)),
    "config2_p_split6": ([CONFIG2], "batch", 1, 6, 1, dict(fused=1, p_split=6)),
    "kf31_181_free_rows": ([win(31, n_lm=700)], "batch", 1, 0, 1, dict(nr_cap_max=192, small_syrk=0, fused=0, p_split=16,
                                                                        solve_tiled=1, solve_split=0, device_pack=0)),
    "kf30_none_fixed": ([win(30, n_lm=700, fixed=0)], "batch", 1, 0, 1, dict(fused=1, fused_slots=7, p_split=88)),
    "mixed_batch": ([CONFIG2, win(31, n_lm=700)], "batch", 1, 0, 1, dict(small_syrk=0, fused=0, nr_cap_max=192, p_split=16)),
    "rows_of_184": ([win(30, rows=184)], "track_fused", 1, 0, 1, dict(nr_cap_max=192, small_syrk=1, fused=1, device_pack=1)),
    "rows_of_185": ([win(30, rows=185)], "track_fused", 1, 0, 1, dict(nr_cap_max=192, small_syrk=0, fused=0, p_split=16,
                                                                       solve_tiled=1, device_pack=0)),
    # the Schur kernel instance: the largest free rows of the batch
    "free_rows_176": ([win(30, free_rows=176)], "batch", 1, 0, 1, dict(fused=1, fused_slots=6)),
    "free_rows_177": ([win(30, free_rows=177)], "batch", 1, 0, 1, dict(fused=1, fused_slots=7)),
    "free_rows_177_in_batch": ([CONFIG2, win(30, free_rows=177)], "batch", 1, 0, 1, dict(fused=1, fused_slots=7, p_split=66)),
    # the factorisation: tiled up to 192 rows, split over the GPU for at most 16 large windows
    "rows_of_192": ([win(30, rows=192)], "batch", 1, 0, 1, dict(nr_cap_max=192, solve_tiled=1, solve_split=0)),
    "rows_of_193": ([win(30, rows=193)], "batch", 1, 0, 1, dict(nr_cap_max=256, solve_tiled=0, solve_split=32)),
    "config5_kf40": ([win(40)], "batch", 1, 0, 1, dict(nr_cap_max=256, fused=0, p_split=16, solve_tiled=0, solve_split=32)),
    "config3_batch1": ([CONFIG3], "batch", 1, 0, 1, dict(nr_cap_max=320, small_syrk=0, fused=0, p_split=16, solve_tiled=0,
                                                          solve_split=32, device_pack=0)),
    "config3_batch264": ([CONFIG3] * 264, "batch", 1, 0, 1, dict(p_split=1, solve_tiled=0, solve_split=0)),
    "config3_p_split6": ([CONFIG3], "batch", 1, 6, 1, dict(p_split=6, solve_split=32)),
    "config3_16_windows": ([CONFIG3] * 16, "batch", 1, 0, 1, dict(p_split=4, solve_split=8)),
    "config3_17_windows": ([CONFIG3] * 17, "batch", 1, 0, 1, dict(p_split=4, solve_split=0)),
    # packing, by purpose and knobs
    "config2_fused0": ([CONFIG2], "batch", 0, 0, 1, dict(small_syrk=1, fused=0, p_split=94, solve_tiled=1, device_pack=0)),
    "config2_device_pack0": ([CONFIG2], "batch", 1, 0, 0, dict(fused=1, device_pack=0)),
    "config2_host_pack": ([CONFIG2], "host_pack", 1, 0, 1, dict(fused=1, p_split=132, device_pack=0)),
    "config2_track_fused": ([CONFIG2], "track_fused", 1, 0, 1, dict(fused=1, device_pack=1)),
    "config2_track_fused_fused0": ([CONFIG2], "track_fused", 0, 0, 1, dict(fused=0, device_pack=0)),
    "over_32768_landmarks": ([win(30, n_lm=32769)], "batch", 1, 0, 1, dict(fused=1, device_pack=0)),
    # a track's large-window solver: device packing, sred room for the split of a 192-row solve
    "track_large_1": ([LARGE_TRACK], "track_large", 1, 0, 1, dict(nr_cap_max=320, fused=0, p_split=16, p_split_cap=16,
                                                                  device_pack=1)),
    "track_large_4": ([LARGE_TRACK] * 4, "track_large", 1, 0, 1, dict(p_split=16, p_split_cap=16, solve_split=32)),
    "track_large_40": ([LARGE_TRACK] * 40, "track_large", 1, 0, 1, dict(p_split=4, p_split_cap=4, solve_split=0)),
    "track_large_p_split6": ([LARGE_TRACK] * 4, "track_large", 1, 6, 1, dict(p_split=6, p_split_cap=6)),
    "track_large_fused0": ([LARGE_TRACK], "track_large", 0, 0, 1, dict(fused=0, device_pack=1)),
    "track_large_device_pack0": ([LARGE_TRACK], "track_large", 1, 0, 0, dict(device_pack=0)),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_plan(driver, name):
    windows, purpose, fused, p_split, device_pack, want = CASES[name]
    got = dict(zip(FIELDS, map(int, driver(_query("plan", windows, purpose, fused, p_split, device_pack))[0].split())))
    assert {k: got[k] for k in want} == want


# the large-window path of a track solve: nr_cap, split and factorisation follow the solved windows (0 rows: the window sits
# the solve out), within the split the solver was created with
REPLAN = {
    "ground_kf19": ([LARGE_TRACK], [win(19, n_lm=1100, planes=True)], 0,
                    dict(nr_cap_max=192, p_split=16, p_split_cap=16, solve_tiled=1, solve_split=0, fused=0, device_pack=1)),
    "ground_kf30": ([LARGE_TRACK], [LARGE_TRACK], 0, dict(nr_cap_max=320, p_split=16, solve_tiled=0, solve_split=32)),
    "plane_free_kf40": ([win(40, n_lm=3000, rows=301)], [win(40, n_lm=3000)], 0,
                        dict(nr_cap_max=256, p_split=16, solve_tiled=0, solve_split=32)),
    "group_with_idle": ([LARGE_TRACK] * 4, [LARGE_TRACK] * 3 + [(0, 0, 0, 0, 0)], 0,
                        dict(nr_cap_max=320, p_split=14, p_split_cap=16, solve_split=32)),
    "group_of_40": ([LARGE_TRACK] * 40, [win(19, n_lm=1100, planes=True)] * 40, 0,
                    dict(nr_cap_max=192, p_split=4, p_split_cap=4, solve_tiled=1, solve_split=0)),
    "p_split6": ([LARGE_TRACK], [win(19, n_lm=1100, planes=True)], 6, dict(p_split=6, p_split_cap=6, solve_tiled=1)),
}


@pytest.mark.parametrize("name", sorted(REPLAN))
def test_track_large_replan(driver, name):
    created, solved, p_split, want = REPLAN[name]
    got = dict(zip(FIELDS, map(int, driver(_query("replan", created, "track_large", 1, p_split, 1, solved=solved))[0].split())))
    assert {k: got[k] for k in want} == want


def test_rows_and_slots(driver):
    """reduced rows on each side of the fused path and of the six-slot kernel; a track request whose candidates count plane
    rows takes the seven-slot kernel at 18 free keyframes, a plane-free window the six-slot one"""
    want = {"rows 30 0": 181, "rows 31 0": 187, "rows 18 1": 181, "rows 19 1": 191, "rows 106 0": 637, "rows 63 1": 631,
            "slots 176": 6, "slots 177": 7, "slots 0": 6}
    out = driver("\n".join(want) + "\n")
    assert dict(zip(want, map(int, out))) == want
    candidates, plane_free = driver("rows 18 1\nrows 18 0\n")[:2]
    assert driver("slots %s\nslots %s\n" % (candidates, plane_free))[:2] == ["7", "6"]


def test_knobs_are_read_from_the_environment(driver):
    assert driver("knobs\n")[0] == "1 1 0 -1 -1 -1 1"
    env = dict(KBA_FUSED="0", KBA_LINEARIZE="0", KBA_P_SPLIT="6", KBA_LIN_GRID="0", KBA_BS_GRID="5", KBA_SOLVE_SPLIT="3",
               KBA_DEVICE_PACK="0")
    assert driver("knobs\n", env)[0] == "0 0 6 0 5 3 0"
    # a non-positive split is the automatic one, grids below -1 are -1
    assert driver("knobs\n", dict(KBA_P_SPLIT="-3", KBA_LIN_GRID="-7", KBA_FUSED="2"))[0] == "1 1 0 -1 -1 -1 1"
