"""CPU-side checks of the per-stream lidar settings' C-ABI: the header declares the calls and flags, and
rpl_lidar_settings as a C compiler lays it out is the ctypes binding's struct (20 bytes)."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "rpl_b200.h")


@pytest.fixture(scope="module")
def capi():
    from rplidar_ros2_driver_b200 import capi

    return capi


def _header():
    return re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)


def test_header_declares_the_call_and_flags(capi):
    src = _header()
    assert re.search(r"rpl_result\s+rpl_capsule_stream_set_lidars\s*\(\s*rpl_capsule_stream\s*\*\s*\w+\s*,\s*"
                     r"const\s+rpl_lidar_settings\s*\*\s*\w+\s*,\s*const\s+uint8_t\s*\*\s*\w+\s*\)\s*;", src)
    flags = dict(re.findall(r"#define\s+(RPL_\w+)\s+(\d+)u", src))
    assert int(flags["RPL_FLAG_PER_STREAM"]) == capi.FLAG_PER_STREAM == 8
    assert int(flags["RPL_CLOUD_PER_STREAM"]) == capi.CLOUD_PER_STREAM == 2
    # the new bits overlap none of the existing ones
    assert capi.FLAG_PER_STREAM & (capi.FLAG_FORCE_GENERAL | capi.FLAG_NO_TMA | capi.FLAG_NO_SMALL) == 0
    assert capi.CLOUD_PER_STREAM & capi.CLOUD_NO_FUSED == 0


def test_ctypes_struct_layout(capi):
    L = capi.LidarSettings
    assert ctypes.sizeof(L) == 20
    assert [getattr(L, f).offset for f in ("is_new_protocol", "scan_processing", "inverted", "pad", "timing")] == \
        [0, 1, 2, 3, 4]
    s = capi.lidar_settings(1, 0, 1, capi.Timing(63, 256000, 17, 1))
    raw = bytes(s)
    assert raw[:4] == bytes([1, 0, 1, 0])
    assert [int.from_bytes(raw[4 + 4 * i: 8 + 4 * i], "little") for i in range(4)] == [63, 256000, 17, 1]


@pytest.mark.skipif(shutil.which("cc") is None, reason="no C compiler")
def test_c_layout_is_the_ctypes_layout(capi, tmp_path):
    prog = tmp_path / "layout.c"
    prog.write_text(
        '#include <stddef.h>\n#include <stdio.h>\n#include "rpl_b200.h"\n'
        "int main(void) {\n"
        '  printf("%zu %zu %zu %zu %zu %zu\\n", sizeof(rpl_lidar_settings), offsetof(rpl_lidar_settings, is_new_protocol),\n'
        "         offsetof(rpl_lidar_settings, scan_processing), offsetof(rpl_lidar_settings, inverted),\n"
        "         offsetof(rpl_lidar_settings, pad), offsetof(rpl_lidar_settings, timing));\n"
        "  return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.run(["cc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()
    L = capi.LidarSettings
    assert [int(v) for v in out] == [ctypes.sizeof(L)] + [getattr(L, f).offset for f in
                                                          ("is_new_protocol", "scan_processing", "inverted", "pad",
                                                           "timing")]
