"""CPU check of the static block -> warp map of k_schur_fused (kSyrkMap12 in limo_b200/csrc/kba_schur_fused.cuh).

The consumer warps keep the lower block triangle of the reduced system in registers, so a block that two warps own is
summed twice and a block that no warp owns stays zero; neither would show until a GPU solve went wrong.  The six-slot
kernel reads slots 1..6 of every warp (block rows <= 10, systems of up to 176 rows), the seven-slot kernel all seven
(block row 11 as well)."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NWARPS, NSLOTS, NONE = 12, 7, 0xff


def _map():
    src = open(os.path.join(ROOT, "limo_b200", "csrc", "kba_schur_fused.cuh")).read()
    m = re.search(r"kSyrkMap12\[(\d+)\]\[(\d+)\]\s*=\s*\{(.*?)\};", src, re.S)
    assert m, "kSyrkMap12 not found"
    assert (int(m.group(1)), int(m.group(2))) == (NWARPS, NSLOTS)
    rows = re.findall(r"\{([^{}]*)\}", m.group(3))
    table = [[int(v, 0) for v in r.split(",")] for r in rows]
    assert len(table) == NWARPS and all(len(r) == NSLOTS for r in table)
    return table


def _owners(table, first_slot, n_rows):
    owners = {}
    for w, row in enumerate(table):
        for code in row[first_slot:]:
            if code == NONE:
                continue
            bi, bj = code >> 4, code & 15
            assert bj <= bi < n_rows, "warp %d: block (%d, %d) outside the triangle of %d block rows" % (w, bi, bj, n_rows)
            owners.setdefault((bi, bj), []).append(w)
    return owners


def test_row11_slot_holds_row11_blocks():
    for w, row in enumerate(_map()):
        assert row[0] >> 4 == 11, "warp %d: slot 0 is not a block of row 11" % w
        assert all(c == NONE or c >> 4 <= 10 for c in row[1:]), "warp %d: a block of row 11 outside slot 0" % w


def test_six_slot_kernel_owns_rows_up_to_10_once():
    owners = _owners(_map(), 1, 11)
    want = {(bi, bj) for bi in range(11) for bj in range(bi + 1)}
    assert set(owners) == want
    assert all(len(ws) == 1 for ws in owners.values()), {b: ws for b, ws in owners.items() if len(ws) > 1}


def test_seven_slot_kernel_owns_every_block_once():
    owners = _owners(_map(), 0, 12)
    want = {(bi, bj) for bi in range(12) for bj in range(bi + 1)}
    assert set(owners) == want
    assert all(len(ws) == 1 for ws in owners.values()), {b: ws for b, ws in owners.items() if len(ws) > 1}
