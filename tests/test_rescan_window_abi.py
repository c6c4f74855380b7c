"""CPU-side checks of the C-ABI of the windows over the re-gridded LaserScans: the header declares
rpl_rescan_window_batch_dev, rpl_capsule_stream_set_rescan_windows and rpl_capsule_stream_push_rescan_msgs[_dev], the
library exports them and refuses null and out-of-range arguments without a device, and rpl_rescan_window as a C compiler
lays it out is the ctypes binding's struct."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest

from oracle import rescan_window_oracle as RW

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "rpl_b200.h")
NAMES = ("rpl_rescan_window_batch_dev", "rpl_capsule_stream_set_rescan_windows", "rpl_capsule_stream_push_rescan_msgs",
         "rpl_capsule_stream_push_rescan_msgs_dev")


@pytest.fixture(scope="module")
def capi():
    from rplidar_ros2_driver_b200 import capi

    return capi


def _header():
    return re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)


def test_header_declares_the_calls(capi):
    src = _header()
    P = r"\s*\*\s*\w+\s*"
    assert re.search(r"rpl_result\s+rpl_rescan_window_batch_dev\s*\(\s*rpl_ctx" + P + r",\s*const\s+rpl_rescan_window" +
                     P + r",\s*const\s+float" + P + r",\s*uint32_t\s+\w+\s*,\s*uint32_t\s+\w+\s*,\s*float" + P +
                     r",\s*void" + P + r"\)\s*;", src)
    assert re.search(r"rpl_result\s+rpl_capsule_stream_set_rescan_windows\s*\(\s*rpl_capsule_stream" + P +
                     r",\s*const\s+rpl_rescan_window" + P + r",\s*const\s+uint8_t" + P + r"\)\s*;", src)
    for dev in (False, True):
        name = "rpl_capsule_stream_push_rescan_msgs" + ("_dev" if dev else "")
        tail = r",\s*void" + P if dev else ""
        assert re.search(r"rpl_result\s+" + name + r"\s*\(\s*rpl_capsule_stream" + P + r",\s*const\s+rpl_push_input" +
                         P + r",\s*const\s+rpl_scan_params" + P + r",\s*const\s+rpl_scan_cloud_params" + P +
                         r",\s*int64_t\s+\w+\s*,\s*const\s+rpl_msgs_out" + P + r",\s*const\s+rpl_msgs_out" + P +
                         r",\s*uint32_t" + P + tail + r"\)\s*;", src), name
    assert re.search(r"#define\s+RPL_RESCAN_WINDOW_MEDIAN\s+0u", src)
    assert re.search(r"#define\s+RPL_RESCAN_WINDOW_MEAN\s+1u", src)
    for name in NAMES:
        assert name in capi.EXPORTS


def test_constants(capi):
    assert (capi.RESCAN_WINDOW_MEDIAN, capi.RESCAN_WINDOW_MEAN) == (RW.MEDIAN, RW.MEAN) == (0, 1)
    assert capi.RESCAN_WINDOW_MAX == RW.MAX_OBSERVATIONS == 16


def test_library_refuses_null_arguments(capi):
    L = capi.lib()
    bad = capi.RESULT_INVALID_DATA
    w = capi.rescan_window(5)
    assert L.rpl_rescan_window_batch_dev(None, ctypes.byref(w), None, 1, 1, None, None) == bad
    assert L.rpl_capsule_stream_set_rescan_windows(None, None, None) == bad
    assert L.rpl_capsule_stream_push_rescan_msgs(None, None, None, None, 0, None, None, None) == bad
    assert L.rpl_capsule_stream_push_rescan_msgs_dev(None, None, None, None, 0, None, None, None, None) == bad


def test_limits_match_the_restatement(capi):
    for obs in range(0, 19):
        for stat in (0, 1, 2, 0xFFFFFFFF):
            assert RW.window_ok(obs, stat) == (1 <= obs <= 16 and stat in (0, 1)), (obs, stat)


def test_ctypes_struct_and_helper(capi):
    S = capi.RescanWindow
    assert ctypes.sizeof(S) == 8
    assert (S.observations.offset, S.statistic.offset) == (0, 4)
    d = capi.rescan_window()
    assert (d.observations, d.statistic) == (1, capi.RESCAN_WINDOW_MEDIAN)
    m = capi.rescan_window(16, "mean")
    assert (m.observations, m.statistic) == (16, capi.RESCAN_WINDOW_MEAN)
    import rplidar_ros2_driver_b200 as R

    assert R.RescanWindow is S and R.rescan_window is capi.rescan_window


@pytest.mark.skipif(shutil.which("cc") is None, reason="no C compiler")
def test_c_layout_is_the_ctypes_layout(tmp_path):
    prog = tmp_path / "layout.c"
    prog.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "rpl_b200.h"\n'
                    "int main(void) {\n"
                    "  size_t v[] = {sizeof(rpl_rescan_window), offsetof(rpl_rescan_window, observations),\n"
                    "                offsetof(rpl_rescan_window, statistic), RPL_RESCAN_WINDOW_MEDIAN,\n"
                    "                RPL_RESCAN_WINDOW_MEAN};\n"
                    '  for (size_t i = 0; i < sizeof(v) / sizeof(v[0]); ++i) printf("%zu ", v[i]);\n'
                    "  return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.run(["cc", "-std=c11", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()
    assert [int(v) for v in out] == [8, 0, 4, 0, 1]
