"""The frame step's C ABI without a GPU: the library exports its three entry points, the ctypes mirror has the header's layout
field by field, and null arguments are refused before any device work."""
import ctypes as C
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ["kba_track_frame_step", "kba_track_group_frame_step", "kba_track_group_frame_step_opts"]


def _build():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "limo_b200", "csrc"), "-s", "all"])


def test_library_exports_the_frame_step():
    _build()
    from limo_b200 import capi
    L = capi.lib()
    for name in NEW:
        assert hasattr(L, name), name
        assert name in capi.SYMBOLS, name


def test_frame_step_layout_matches_header(tmp_path):
    """sizeof and offsetof of every field of the new structs as the C compiler sees them == the ctypes mirror's"""
    from limo_b200 import capi_types as T
    structs = {"kba_frame_step_request": T.KbaFrameStepRequest, "kba_frame_step_out": T.KbaFrameStepOut}
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "kba_b200.h"', 'int main(){']
    want = []
    for cname, py in structs.items():
        lines.append('printf("%%zu\\n", sizeof(%s));' % cname)
        want.append(C.sizeof(py))
        for f, _t in py._fields_:
            lines.append('printf("%%zu\\n", offsetof(%s, %s));' % (cname, f))
            want.append(getattr(py, f).offset)
    lines += ['return 0;}']
    prog = tmp_path / "layout.c"
    prog.write_text("\n".join(lines) + "\n")
    exe = tmp_path / "layout"
    subprocess.check_call([os.environ.get("CC", "cc"), "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)])
    out = subprocess.check_output([str(exe)]).decode().split()
    assert [int(x) for x in out] == want


def test_frame_step_null_arguments_need_no_device():
    _build()
    from limo_b200 import capi
    L = capi.lib()
    q, o, r = capi.KbaFrameStepRequest(), capi.KbaFrameStepOut(), capi.KbaResult()
    opt = capi.KbaOptions()
    assert L.kba_track_frame_step(None, C.byref(q), C.byref(opt), C.byref(o), C.byref(r)) == 1
    assert L.kba_track_group_frame_step(None, C.byref(q), C.byref(opt), C.byref(o), C.byref(r)) == 1
    assert L.kba_track_group_frame_step_opts(None, C.byref(q), C.byref(opt), C.byref(o), C.byref(r)) == 1
    assert b"null argument" in L.kba_last_error()
