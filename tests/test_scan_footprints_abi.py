"""CPU-side checks of the footprint stage's C-ABI: the header declares rpl_scan_filter_footprint_batch_dev and
rpl_capsule_stream_set_scan_footprints, the library exports them and refuses null arguments without a device,
rpl_scan_footprint as a C compiler lays it out is the ctypes binding's struct, and the binding's helper builds
footprints the definition accepts or refuses as the library does."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from oracle import scan_footprint_oracle as FP
from test_scan_footprints_oracle import BAD, GOOD, make

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "rpl_b200.h")
FIELDS = ("x", "y", "n_vertices", "invert", "pose_x", "pose_y", "pose_yaw")
OFFSETS = [0, 256, 512, 528, 532, 536, 540]


@pytest.fixture(scope="module")
def capi():
    from rplidar_ros2_driver_b200 import capi

    return capi


def _header():
    return re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)


def test_header_declares_the_calls(capi):
    src = _header()
    assert re.search(r"rpl_result\s+rpl_scan_filter_footprint_batch_dev\s*\(\s*rpl_ctx\s*\*\s*\w+\s*,\s*"
                     r"const\s+rpl_scan_filter_settings\s*\*\s*\w+\s*,\s*const\s+rpl_scan_footprint\s*\*\s*\w+\s*,"
                     r"\s*float\s*\*\s*\w+\s*,\s*const\s+float\s*\*\s*\w+\s*,\s*const\s+uint32_t\s*\*\s*\w+\s*,"
                     r"\s*const\s+float\s*\*\s*\w+\s*,\s*uint32_t\s+\w+\s*,\s*uint32_t\s+\w+\s*,\s*void\s*\*\s*\w+\s*\)\s*;",
                     src)
    assert re.search(r"rpl_result\s+rpl_capsule_stream_set_scan_footprints\s*\(\s*rpl_capsule_stream\s*\*\s*\w+\s*,\s*"
                     r"const\s+rpl_scan_footprint\s*\*\s*\w+\s*,\s*const\s+uint8_t\s*\*\s*\w+\s*\)\s*;", src)
    for name in ("rpl_scan_filter_footprint_batch_dev", "rpl_capsule_stream_set_scan_footprints"):
        assert name in capi.EXPORTS


def test_library_exports_the_calls_and_refuses_null_arguments(capi):
    L = capi.lib()
    bad = capi.RESULT_INVALID_DATA
    assert L.rpl_capsule_stream_set_scan_footprints(None, None, None) == bad
    fp = capi.scan_footprint()
    assert L.rpl_capsule_stream_set_scan_footprints(None, ctypes.cast(ctypes.pointer(fp), ctypes.c_void_p), None) == bad
    s = capi.scan_filter_settings()
    assert L.rpl_scan_filter_footprint_batch_dev(None, ctypes.byref(s), ctypes.byref(fp), None, None, None, None, 0, 1,
                                                 None) == bad


def test_ctypes_struct_layout(capi):
    S = capi.ScanFootprint
    assert ctypes.sizeof(S) == 544
    assert [getattr(S, f).offset for f in FIELDS] == OFFSETS
    box = [(-0.2, -0.1), (0.3, -0.1), (0.3, 0.1), (-0.2, 0.1)]
    f = capi.scan_footprint([box, [], box[:3]], invert=[0, 0, 1], pose=(0.1, -0.2, 0.5))
    assert list(f.n_vertices) == [4, 0, 3, 0] and list(f.invert) == [0, 0, 1, 0]
    assert [f.x[0][k] for k in range(4)] == [ctypes.c_float(v).value for v, _ in box]
    assert [f.y[2][k] for k in range(3)] == [ctypes.c_float(v).value for _, v in box[:3]]
    assert (f.pose_x, f.pose_y, f.pose_yaw) == tuple(ctypes.c_float(v).value for v in (0.1, -0.2, 0.5))
    # the helper and the definition hold the same footprint
    o = FP.footprint([box, [], box[:3]], invert=[0, 0, 1], pose=(0.1, -0.2, 0.5))
    assert [(u.tobytes(), v.tobytes(), i) for u, v, i in FP.scan_frame(f)] == \
           [(u.tobytes(), v.tobytes(), i) for u, v, i in FP.scan_frame(o)]
    assert np.array(f.x, np.float32).tobytes() == o.x.tobytes()


@pytest.mark.skipif(shutil.which("cc") is None, reason="no C compiler")
def test_c_layout_is_the_ctypes_layout(tmp_path):
    prog = tmp_path / "layout.c"
    offs = ", ".join(f"offsetof(rpl_scan_footprint, {f})" for f in FIELDS)
    fmt = " ".join(["%zu"] * (len(FIELDS) + 1))
    prog.write_text(
        '#include <stddef.h>\n#include <stdio.h>\n#include "rpl_b200.h"\n'
        "int main(void) {\n"
        f'  printf("{fmt}\\n", sizeof(rpl_scan_footprint), {offs});\n'
        "  return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.run(["cc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)], check=True)
    out = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert out == [544] + OFFSETS


@pytest.mark.parametrize("kw,ok", [(k, False) for k in BAD] + [(k, True) for k in GOOD])
def test_footprint_validation(capi, kw, ok):
    assert FP.footprint_ok(make(capi.scan_footprint, kw)) == ok
    assert FP.footprint_ok(make(FP.footprint, kw)) == ok
