"""CPU-side checks of the C-ABI of the re-gridded LaserScans: the header declares rpl_rescan_batch_dev,
rpl_capsule_stream_set_rescans and rpl_capsule_stream_rescan_msgs[_dev], the library exports them and refuses null
arguments without a device, and rpl_rescan_settings as a C compiler lays it out is the ctypes binding's struct."""
import ctypes
import math
import os
import re
import shutil
import subprocess

import pytest

from oracle import rescan_oracle as RQ

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "rpl_b200.h")
NAMES = ("rpl_rescan_batch_dev", "rpl_capsule_stream_set_rescans", "rpl_capsule_stream_rescan_msgs",
         "rpl_capsule_stream_rescan_msgs_dev")
FIELDS = ("angle_min", "angle_max", "angle_increment", "range_min", "range_max", "min_height", "max_height",
          "inf_epsilon", "scan_time", "use_inf", "enabled", "pad")
OFFSETS = (0, 4, 8, 12, 16, 20, 24, 28, 32, 36, 37, 38)


@pytest.fixture(scope="module")
def capi():
    from rplidar_ros2_driver_b200 import capi

    return capi


def _header():
    return re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)


def test_header_declares_the_calls(capi):
    src = _header()
    P = r"\s*\*\s*\w+\s*"
    assert re.search(r"rpl_result\s+rpl_rescan_batch_dev\s*\(\s*rpl_ctx" + P + r",\s*const\s+rpl_rescan_settings" + P +
                     r",\s*const\s+rpl_scan_cloud_params" + P + r",\s*const\s+rpl_scan_cloud_transform" + P +
                     r",\s*const\s+float" + P + r",\s*const\s+float" + P + r",\s*const\s+uint32_t" + P +
                     r",\s*const\s+float" + P + r",\s*float\s+\w+\s*,\s*float\s+\w+\s*,\s*uint32_t\s+\w+\s*,"
                     r"\s*uint32_t\s+\w+\s*,\s*float" + P + r",\s*void" + P + r"\)\s*;", src)
    assert re.search(r"rpl_result\s+rpl_capsule_stream_set_rescans\s*\(\s*rpl_capsule_stream" + P +
                     r",\s*const\s+rpl_rescan_settings" + P + r",\s*const\s+uint8_t" + P + r"\)\s*;", src)
    for dev in (False, True):
        name = "rpl_capsule_stream_rescan_msgs" + ("_dev" if dev else "")
        tail = r",\s*void" + P if dev else ""
        assert re.search(r"rpl_result\s+" + name + r"\s*\(\s*rpl_capsule_stream" + P + r",\s*const\s+rpl_scan_params" +
                         P + r",\s*const\s+rpl_scan_cloud_params" + P + r",\s*int64_t\s+\w+\s*,\s*uint8_t" + P +
                         r",\s*uint64_t\s+\w+\s*,\s*uint64_t" + P + r",\s*uint32_t" + P + r",\s*uint64_t" + P + tail +
                         r"\)\s*;", src), name
    for name in NAMES:
        assert name in capi.EXPORTS


def test_library_refuses_null_arguments(capi):
    L = capi.lib()
    bad = capi.RESULT_INVALID_DATA
    s, p = capi.rescan_settings(), capi.scan_cloud_params()
    assert L.rpl_rescan_batch_dev(None, ctypes.byref(s), ctypes.byref(p), None, None, None, None, None, 0.15, 40.0, 0,
                                  1, None, None) == bad
    assert L.rpl_capsule_stream_set_rescans(None, None, None) == bad
    assert L.rpl_capsule_stream_rescan_msgs(None, None, None, 0, None, 0, None, None, None) == bad
    assert L.rpl_capsule_stream_rescan_msgs_dev(None, None, None, 0, None, 0, None, None, None, None) == bad


def test_ctypes_struct_and_defaults(capi):
    S = capi.RescanSettings
    assert ctypes.sizeof(S) == 40
    assert tuple(getattr(S, f).offset for f in FIELDS) == OFFSETS
    d = capi.rescan_settings()
    o = RQ.settings()
    for f in FIELDS[:9]:
        assert getattr(d, f) == getattr(o, f), f
    assert d.use_inf == 1 and d.enabled == 1 and d.inf_epsilon == 1.0
    assert d.angle_min == pytest.approx(-math.pi) and d.angle_increment == pytest.approx(math.pi / 180)
    assert capi.rescan_ranges_size(d) == RQ.ranges_size(o) == 360
    assert capi.rescan_settings(enabled=False).enabled == 0


@pytest.mark.skipif(shutil.which("cc") is None, reason="no C compiler")
def test_c_layout_is_the_ctypes_layout(tmp_path):
    prog = tmp_path / "layout.c"
    offs = ", ".join("offsetof(rpl_rescan_settings, %s)" % f for f in FIELDS)
    prog.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "rpl_b200.h"\n'
                    "int main(void) {\n"
                    '  size_t v[] = {sizeof(rpl_rescan_settings), %s};\n'
                    '  for (size_t i = 0; i < sizeof(v) / sizeof(v[0]); ++i) printf("%%zu ", v[i]);\n'
                    "  return 0;\n}\n" % offs)
    exe = tmp_path / "layout"
    subprocess.run(["cc", "-std=c11", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()
    assert [int(v) for v in out] == [40, *OFFSETS]
