"""CPU-side checks of the C-ABI of projected clouds in a target frame: the header declares
rpl_capsule_stream_set_scan_cloud_transforms and rpl_scan_cloud_transform_batch_dev and the two bits, the library
exports the calls and refuses null arguments without a device, and rpl_scan_cloud_transform as a C compiler lays it out
is the ctypes binding's struct."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest

import scan_cloud_transform_oracle as SCT

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "rpl_b200.h")
MACROS = {"RPL_SCAN_CLOUD_VIEWPOINT": SCT.VIEWPOINT,
          "RPL_SCAN_CLOUD_PER_STREAM_TRANSFORMS": SCT.PER_STREAM_TRANSFORMS}


@pytest.fixture(scope="module")
def capi():
    from rplidar_ros2_driver_b200 import capi

    return capi


def _header():
    return re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)


def test_header_declares_the_calls_and_macros(capi):
    src = _header()
    P = r"\s*\*\s*\w+\s*"
    assert re.search(r"rpl_result\s+rpl_capsule_stream_set_scan_cloud_transforms\s*\(\s*rpl_capsule_stream" + P +
                     r",\s*const\s+rpl_scan_cloud_transform" + P + r",\s*const\s+char\s*\*\s*const\s*\*\s*\w+\s*,"
                     r"\s*const\s+uint8_t" + P + r"\)\s*;", src)
    assert re.search(r"rpl_result\s+rpl_scan_cloud_transform_batch_dev\s*\(\s*rpl_ctx" + P +
                     r",\s*const\s+rpl_scan_cloud_params" + P + r",\s*const\s+rpl_scan_cloud_transform" + P +
                     r",\s*const\s+float" + P + r",\s*const\s+float" + P + r",\s*const\s+uint32_t" + P +
                     r",\s*const\s+float" + P + r",\s*const\s+float" + P + r",\s*float\s+\w+\s*,\s*float\s+\w+\s*,"
                     r"\s*uint32_t\s+\w+\s*,\s*uint32_t\s+\w+\s*,\s*void" + P + r",\s*uint32_t" + P + r",\s*void" + P +
                     r"\)\s*;", src)
    for name, v in MACROS.items():
        m = re.search(rf"#define\s+{name}\s+(0x[0-9a-fA-F]+)u?\b", src)
        assert m and int(m.group(1), 16) == v, name
        assert getattr(capi, name[4:]) == v
    for name in ("rpl_capsule_stream_set_scan_cloud_transforms", "rpl_scan_cloud_transform_batch_dev"):
        assert name in capi.EXPORTS


def test_library_refuses_null_arguments(capi):
    L = capi.lib()
    bad = capi.RESULT_INVALID_DATA
    p = capi.scan_cloud_params()
    t = capi.scan_cloud_transform()
    assert L.rpl_scan_cloud_transform_batch_dev(None, ctypes.byref(p), ctypes.byref(t), None, None, None, None, None,
                                                0.15, 40.0, 0, 1, None, None, None) == bad
    assert L.rpl_capsule_stream_set_scan_cloud_transforms(None, None, None, None) == bad


def test_ctypes_struct_and_helpers(capi):
    S = capi.ScanCloudTransform
    assert ctypes.sizeof(S) == 64
    assert (S.translation.offset, S.rotation.offset, S.enabled.offset) == (0, 24, 56)
    d = capi.scan_cloud_transform()
    assert list(d.translation) == [0.0, 0.0, 0.0] and list(d.rotation) == [0.0, 0.0, 0.0, 1.0] and d.enabled == 1
    assert capi.scan_cloud_transform(enabled=False).enabled == 0
    for ch in range(32):
        assert capi.scan_cloud_point_step(ch) == SCT.point_step(ch)


@pytest.mark.skipif(shutil.which("cc") is None, reason="no C compiler")
def test_c_layout_is_the_ctypes_layout(tmp_path):
    prog = tmp_path / "layout.c"
    prog.write_text(
        '#include <stddef.h>\n#include <stdio.h>\n#include "rpl_b200.h"\n'
        "int main(void) {\n"
        '  printf("%zu %zu %zu %zu %zu %u %u\\n", sizeof(rpl_scan_cloud_transform),\n'
        "         offsetof(rpl_scan_cloud_transform, translation), offsetof(rpl_scan_cloud_transform, rotation),\n"
        "         offsetof(rpl_scan_cloud_transform, enabled), offsetof(rpl_scan_cloud_transform, pad),\n"
        "         RPL_SCAN_CLOUD_VIEWPOINT, RPL_SCAN_CLOUD_PER_STREAM_TRANSFORMS);\n"
        "  return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.run(["cc", "-std=c11", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()
    assert [int(v) for v in out] == [64, 0, 24, 56, 57, SCT.VIEWPOINT, SCT.PER_STREAM_TRANSFORMS]
