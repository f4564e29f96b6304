"""The keyframe solve's C ABI without a GPU: the library exports its three entry points, the ctypes mirror has the header's layout
field by field, and null arguments are refused before any device work."""
import ctypes as C
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ["kba_track_keyframe_solve", "kba_track_group_keyframe_solve", "kba_track_group_keyframe_solve_opts"]


def _build():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "limo_b200", "csrc"), "-s", "all"])


def test_library_exports_the_keyframe_solve():
    _build()
    from limo_b200 import capi
    L = capi.lib()
    for name in NEW:
        assert hasattr(L, name), name
        assert name in capi.SYMBOLS, name


def test_keyframe_solve_layout_matches_header(tmp_path):
    """sizeof and offsetof of every field of the new structs as the C compiler sees them == the ctypes mirror's"""
    from limo_b200 import capi_types as T
    structs = {"kba_label_class": T.KbaLabelClass, "kba_tracklet": T.KbaTracklet, "kba_kfsolve_request": T.KbaKfsolveRequest,
               "kba_kfsolve_out": T.KbaKfsolveOut}
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "kba_b200.h"', 'int main(){']
    want = []
    for cname, py in structs.items():
        lines.append('printf("%%zu\\n", sizeof(%s));' % cname)
        want.append(C.sizeof(py))
        for f, _t in py._fields_:
            lines.append('printf("%%zu\\n", offsetof(%s, %s));' % (cname, f))
            want.append(getattr(py, f).offset)
    lines += ['printf("%d %d %d\\n", KBA_LABEL_OUTLIER, KBA_LABEL_SHRUBBERY, KBA_LABEL_GROUND);', 'return 0;}']
    prog = tmp_path / "layout.c"
    prog.write_text("\n".join(lines) + "\n")
    exe = tmp_path / "layout"
    subprocess.check_call([os.environ.get("CC", "cc"), "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)])
    out = subprocess.check_output([str(exe)]).decode().split("\n")
    assert [int(x) for x in out[:len(want)]] == want
    assert out[len(want)].split() == [str(T.LABEL_OUTLIER), str(T.LABEL_SHRUBBERY), str(T.LABEL_GROUND)]


def test_keyframe_solve_null_arguments_need_no_device():
    _build()
    from limo_b200 import capi
    L = capi.lib()
    q, o, r = capi.KbaKfsolveRequest(), capi.KbaKfsolveOut(), capi.KbaResult()
    opt = capi.KbaOptions()
    assert L.kba_track_keyframe_solve(None, C.byref(q), C.byref(opt), C.byref(o), C.byref(r)) == 1
    assert L.kba_track_group_keyframe_solve(None, C.byref(q), C.byref(opt), C.byref(o), C.byref(r)) == 1
    assert L.kba_track_group_keyframe_solve_opts(None, C.byref(q), C.byref(opt), C.byref(o), C.byref(r)) == 1
    assert b"null argument" in L.kba_last_error()
