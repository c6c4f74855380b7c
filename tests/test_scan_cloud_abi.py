"""CPU-side checks of the scan projection's C-ABI: the header declares rpl_scan_cloud_batch_dev and
rpl_capsule_stream_scan_cloud_msgs[_dev] and the channel macros, the library exports the calls and refuses null arguments
without a device, and rpl_scan_cloud_params as a C compiler lays it out is the ctypes binding's struct."""
import ctypes
import math
import os
import re
import shutil
import subprocess

import pytest

from oracle import scan_cloud_oracle as SC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "rpl_b200.h")
MACROS = {"RPL_SCAN_CLOUD_INTENSITY": SC.INTENSITY, "RPL_SCAN_CLOUD_INDEX": SC.INDEX,
          "RPL_SCAN_CLOUD_DISTANCE": SC.DISTANCE, "RPL_SCAN_CLOUD_TIMESTAMP": SC.TIMESTAMP}


@pytest.fixture(scope="module")
def capi():
    from rplidar_ros2_driver_b200 import capi

    return capi


def _header():
    return re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)


def test_header_declares_the_calls_and_macros(capi):
    src = _header()
    P = r"\s*\*\s*\w+\s*"
    assert re.search(r"rpl_result\s+rpl_scan_cloud_batch_dev\s*\(\s*rpl_ctx" + P + r",\s*const\s+rpl_scan_cloud_params"
                     + P + r",\s*const\s+float" + P + r",\s*const\s+float" + P + r",\s*const\s+uint32_t" + P +
                     r",\s*const\s+float" + P + r",\s*const\s+float" + P + r",\s*float\s+\w+\s*,\s*float\s+\w+\s*,"
                     r"\s*uint32_t\s+\w+\s*,\s*uint32_t\s+\w+\s*,\s*void" + P + r",\s*uint32_t" + P + r",\s*void" + P +
                     r"\)\s*;", src)
    tail = (r",\s*const\s+rpl_scan_params" + P + r",\s*const\s+rpl_scan_cloud_params" + P + r",\s*int64_t\s+\w+\s*,"
            r"\s*uint8_t" + P + r",\s*uint64_t\s+\w+\s*,\s*uint64_t" + P + r",\s*uint32_t" + P + r",\s*uint64_t" + P)
    assert re.search(r"rpl_result\s+rpl_capsule_stream_scan_cloud_msgs_dev\s*\(\s*rpl_capsule_stream" + P + tail +
                     r",\s*void" + P + r"\)\s*;", src)
    assert re.search(r"rpl_result\s+rpl_capsule_stream_scan_cloud_msgs\s*\(\s*rpl_capsule_stream" + P + tail +
                     r"\)\s*;", src)
    for name, v in MACROS.items():
        m = re.search(rf"#define\s+{name}\s+(0x[0-9a-fA-F]+)u?\b", src)
        assert m and int(m.group(1), 16) == v, name
        assert getattr(capi, name[4:]) == v
    for name in ("rpl_scan_cloud_batch_dev", "rpl_capsule_stream_scan_cloud_msgs",
                 "rpl_capsule_stream_scan_cloud_msgs_dev"):
        assert name in capi.EXPORTS


def test_library_refuses_null_arguments(capi):
    L = capi.lib()
    bad = capi.RESULT_INVALID_DATA
    p = capi.scan_cloud_params()
    assert L.rpl_scan_cloud_batch_dev(None, ctypes.byref(p), None, None, None, None, None, 0.15, 40.0, 0, 1, None, None,
                                      None) == bad
    assert L.rpl_capsule_stream_scan_cloud_msgs(None, None, ctypes.byref(p), 0, None, 0, None, None, None) == bad
    assert L.rpl_capsule_stream_scan_cloud_msgs_dev(None, None, ctypes.byref(p), 0, None, 0, None, None, None,
                                                    None) == bad


def test_ctypes_struct_and_helper(capi):
    S = capi.ScanCloudParams
    assert ctypes.sizeof(S) == 8 and S.channels.offset == 0 and S.range_cutoff.offset == 4
    d = capi.scan_cloud_params()
    assert (d.channels, d.range_cutoff) == (SC.DEFAULT, -1.0) == (SC.params().channels, SC.params().range_cutoff)
    for ch in range(16):
        assert capi.scan_cloud_point_step(ch) == SC.point_step(ch)
    assert SC.params_ok(capi.scan_cloud_params(0x0F, math.inf))
    assert not SC.params_ok(capi.scan_cloud_params(0x10)) and not SC.params_ok(capi.scan_cloud_params(0, math.nan))


@pytest.mark.skipif(shutil.which("cc") is None, reason="no C compiler")
def test_c_layout_is_the_ctypes_layout(tmp_path):
    prog = tmp_path / "layout.c"
    prog.write_text(
        '#include <stddef.h>\n#include <stdio.h>\n#include "rpl_b200.h"\n'
        "int main(void) {\n"
        '  printf("%zu %zu %zu %u %u %u %u\\n", sizeof(rpl_scan_cloud_params), offsetof(rpl_scan_cloud_params, '
        "channels), offsetof(rpl_scan_cloud_params, range_cutoff), RPL_SCAN_CLOUD_INTENSITY, RPL_SCAN_CLOUD_INDEX, "
        "RPL_SCAN_CLOUD_DISTANCE, RPL_SCAN_CLOUD_TIMESTAMP);\n"
        "  return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.run(["cc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)], check=True)
    out = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert out == [8, 0, 4, 1, 2, 4, 8]
