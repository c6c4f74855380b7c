"""CPU-side checks of the C-ABI of the merged scans: the header declares rpl_rescan_merge_batch_dev,
rpl_capsule_stream_set_rescan_merges and rpl_capsule_stream_push_rescan_merge_msgs[_dev] and RPL_RESCAN_MERGE_NONE, the
library exports them and refuses null arguments without a device, and a C compiler takes the calls with the argument
types the ctypes binding passes."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest

from oracle import rescan_merge_oracle as RM

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "rpl_b200.h")
NAMES = ("rpl_rescan_merge_batch_dev", "rpl_capsule_stream_set_rescan_merges",
         "rpl_capsule_stream_push_rescan_merge_msgs", "rpl_capsule_stream_push_rescan_merge_msgs_dev")


@pytest.fixture(scope="module")
def capi():
    from rplidar_ros2_driver_b200 import capi

    return capi


def _header():
    return re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)


def test_header_declares_the_calls(capi):
    src = _header()
    P = r"\s*\*\s*\w+\s*"
    assert re.search(r"rpl_result\s+rpl_rescan_merge_batch_dev\s*\(\s*rpl_ctx" + P + r",\s*const\s+rpl_rescan_settings" +
                     P + r",\s*const\s+float" + P + r",\s*const\s+uint32_t" + P +
                     r",\s*uint32_t\s+\w+\s*,\s*uint32_t\s+\w+\s*,\s*float" + P + r",\s*void" + P + r"\)\s*;", src)
    assert re.search(r"rpl_result\s+rpl_capsule_stream_set_rescan_merges\s*\(\s*rpl_capsule_stream" + P +
                     r",\s*const\s+uint32_t" + P + r",\s*const\s+uint32_t" + P + r",\s*uint32_t\s+\w+\s*\)\s*;", src)
    for dev in (False, True):
        name = "rpl_capsule_stream_push_rescan_merge_msgs" + ("_dev" if dev else "")
        tail = r",\s*void" + P if dev else ""
        assert re.search(r"rpl_result\s+" + name + r"\s*\(\s*rpl_capsule_stream" + P + r",\s*const\s+rpl_push_input" +
                         P + r",\s*const\s+rpl_scan_params" + P + r",\s*const\s+rpl_scan_cloud_params" + P +
                         r",\s*int64_t\s+\w+\s*" + r",\s*const\s+rpl_msgs_out" + P + r",\s*const\s+rpl_msgs_out" +
                         P + r",\s*const\s+rpl_msgs_out" + P + r",\s*uint32_t" + P + tail + r"\)\s*;", src), name
    assert re.search(r"#define\s+RPL_RESCAN_MERGE_NONE\s+0xFFFFFFFFu", src)
    for name in NAMES:
        assert name in capi.EXPORTS


def test_constants(capi):
    import rplidar_ros2_driver_b200 as R

    assert capi.RESCAN_MERGE_NONE == RM.NONE == R.RESCAN_MERGE_NONE == 0xFFFFFFFF


def test_library_refuses_null_arguments(capi):
    L = capi.lib()
    bad = capi.RESULT_INVALID_DATA
    s = capi.rescan_settings()
    assert L.rpl_rescan_merge_batch_dev(None, ctypes.byref(s), None, None, 1, 1, None, None) == bad
    assert L.rpl_capsule_stream_set_rescan_merges(None, None, None, 0) == bad
    assert L.rpl_capsule_stream_push_rescan_merge_msgs(None, None, None, None, 0, None, None, None, None) == bad
    assert L.rpl_capsule_stream_push_rescan_merge_msgs_dev(None, None, None, None, 0, None, None, None, None,
                                                           None) == bad


@pytest.mark.skipif(shutil.which("cc") is None, reason="no C compiler")
def test_c_calls_take_the_binding_arguments(tmp_path):
    """the prototypes assign to function pointers of the argument lists the binding passes, and the constant is the
    32-bit all-ones value"""
    prog = tmp_path / "probe.c"
    prog.write_text(
        '#include <stdio.h>\n#include "rpl_b200.h"\n'
        "typedef rpl_result (*batch_fn)(rpl_ctx*, const rpl_rescan_settings*, const float*, const uint32_t*, uint32_t,\n"
        "                               uint32_t, float*, void*);\n"
        "typedef rpl_result (*set_fn)(rpl_capsule_stream*, const uint32_t*, const uint32_t*, uint32_t);\n"
        "typedef rpl_result (*push_fn)(rpl_capsule_stream*, const rpl_push_input*, const rpl_scan_params*,\n"
        "                              const rpl_scan_cloud_params*, int64_t, const rpl_msgs_out*, const rpl_msgs_out*,\n"
        "                              const rpl_msgs_out*, uint32_t*);\n"
        "typedef rpl_result (*push_dev_fn)(rpl_capsule_stream*, const rpl_push_input*, const rpl_scan_params*,\n"
        "                                  const rpl_scan_cloud_params*, int64_t, const rpl_msgs_out*,\n"
        "                                  const rpl_msgs_out*, const rpl_msgs_out*, uint32_t*, void*);\n"
        "int main(void) {\n"
        "  batch_fn b = rpl_rescan_merge_batch_dev;\n  set_fn s = rpl_capsule_stream_set_rescan_merges;\n"
        "  push_fn p = rpl_capsule_stream_push_rescan_merge_msgs;\n"
        "  push_dev_fn d = rpl_capsule_stream_push_rescan_merge_msgs_dev;\n"
        '  printf("%u %zu %d", (unsigned)RPL_RESCAN_MERGE_NONE, sizeof(RPL_RESCAN_MERGE_NONE),\n'
        "         b != 0 && s != 0 && p != 0 && d != 0);\n  return 0;\n}\n")
    obj = tmp_path / "probe.o"
    subprocess.run(["cc", "-std=c11", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), "-c", str(prog), "-o",
                    str(obj)], check=True)
    exe = tmp_path / "probe"
    lib = os.path.join(ROOT, "rplidar_ros2_driver_b200")
    r = subprocess.run(["cc", str(obj), "-L", lib, "-lrplidar_b200", "-Wl,-rpath," + lib, "-o", str(exe)])
    if r.returncode != 0 or not os.path.exists(os.path.join(lib, "librplidar_b200.so")):
        pytest.skip("the library is not built here")
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()
    assert out == ["4294967295", "4", "1"]
