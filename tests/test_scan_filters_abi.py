"""CPU-side checks of the LaserScan filters' C-ABI: the header declares rpl_scan_filter_batch_dev,
rpl_capsule_stream_set_scan_filters and RPL_FLAG_PER_STREAM_FILTERS, rpl_scan_filter_settings as a C compiler lays it
out is the ctypes binding's struct, and the binding's helper builds entries the definition accepts or refuses as the
library does."""
import ctypes
import math
import os
import re
import shutil
import subprocess

import pytest

from oracle import scan_filter_oracle as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "rpl_b200.h")
FIELDS = ("mask_lo", "mask_hi", "range_lo", "range_hi", "intensity_min", "speckle_max_diff", "shadow_angle",
          "speckle_window", "speckle_min_neighbours", "shadow_window", "enabled", "pad")
OFFSETS = [0, 16, 32, 36, 40, 44, 48, 52, 56, 60, 64, 65]


@pytest.fixture(scope="module")
def capi():
    from rplidar_ros2_driver_b200 import capi

    return capi


def _header():
    return re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)


def test_header_declares_the_calls_and_flag(capi):
    src = _header()
    assert re.search(r"rpl_result\s+rpl_scan_filter_batch_dev\s*\(\s*rpl_ctx\s*\*\s*\w+\s*,\s*"
                     r"const\s+rpl_scan_filter_settings\s*\*\s*\w+\s*,\s*float\s*\*\s*\w+\s*,\s*const\s+float\s*\*\s*\w+\s*,"
                     r"\s*const\s+uint32_t\s*\*\s*\w+\s*,\s*const\s+float\s*\*\s*\w+\s*,\s*uint32_t\s+\w+\s*,\s*uint32_t\s+\w+\s*,"
                     r"\s*void\s*\*\s*\w+\s*\)\s*;", src)
    assert re.search(r"rpl_result\s+rpl_capsule_stream_set_scan_filters\s*\(\s*rpl_capsule_stream\s*\*\s*\w+\s*,\s*"
                     r"const\s+rpl_scan_filter_settings\s*\*\s*\w+\s*,\s*const\s+uint8_t\s*\*\s*\w+\s*\)\s*;", src)
    flags = {k: int(v) for k, v in re.findall(r"#define\s+(RPL_FLAG_\w+)\s+(\d+)u", src)}
    assert flags["RPL_FLAG_PER_STREAM_FILTERS"] == capi.FLAG_PER_STREAM_FILTERS == 16
    others = [v for k, v in flags.items() if k != "RPL_FLAG_PER_STREAM_FILTERS"]
    assert len(others) == 4 and all(v & 16 == 0 for v in others)
    for name in ("rpl_scan_filter_batch_dev", "rpl_capsule_stream_set_scan_filters"):
        assert name in capi.EXPORTS


def test_ctypes_struct_layout(capi):
    S = capi.ScanFilterSettings
    assert ctypes.sizeof(S) == 68
    assert [getattr(S, f).offset for f in FIELDS] == OFFSETS
    s = capi.scan_filter_settings(mask=[(0.1, 0.2)], range_lo=0.15, speckle_window=3, speckle_min_neighbours=2,
                                  speckle_max_diff=0.05, shadow_window=8, shadow_angle=0.2, enabled=False)
    assert list(s.mask_lo) == [ctypes.c_float(0.1).value, math.inf, math.inf, math.inf]
    assert list(s.mask_hi) == [ctypes.c_float(0.2).value, -math.inf, -math.inf, -math.inf]
    assert s.range_hi == math.inf and s.intensity_min == -math.inf and s.enabled == 0
    assert bytes(s)[65:] == bytes(3)


@pytest.mark.skipif(shutil.which("cc") is None, reason="no C compiler")
def test_c_layout_is_the_ctypes_layout(capi, tmp_path):
    prog = tmp_path / "layout.c"
    offs = ", ".join(f"offsetof(rpl_scan_filter_settings, {f})" for f in FIELDS)
    fmt = " ".join(["%zu"] * (len(FIELDS) + 1))
    prog.write_text(
        '#include <stddef.h>\n#include <stdio.h>\n#include "rpl_b200.h"\n'
        "int main(void) {\n"
        f'  printf("{fmt}\\n", sizeof(rpl_scan_filter_settings), {offs});\n'
        "  return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.run(["cc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)], check=True)
    out = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert out == [68] + OFFSETS


# entries the library refuses with RPL_RESULT_INVALID_DATA (tests/test_gpu_scan_filters.py plays them against it)
BAD = [
    dict(speckle_window=17),
    dict(shadow_window=17, shadow_angle=0.5),
    dict(speckle_window=2, speckle_min_neighbours=5),
    dict(shadow_window=1, shadow_angle=0.0),
    dict(shadow_window=1, shadow_angle=math.pi / 2),
    dict(range_lo=2.0, range_hi=1.0),
    dict(range_hi=math.nan),
    dict(intensity_min=math.nan),
    dict(speckle_max_diff=math.nan),
    dict(shadow_angle=math.nan),
    dict(mask=[(0.0, math.nan)]),
]
GOOD = [
    dict(),
    dict(speckle_window=16, speckle_min_neighbours=32, shadow_window=16, shadow_angle=1.5707),
    dict(range_lo=3.0, range_hi=3.0, shadow_angle=7.0),  # the angle is only checked when the stage is on
    dict(mask=[(1.0, 0.0)] * 4, intensity_min=math.inf),
]


@pytest.mark.parametrize("kw,ok", [(k, False) for k in BAD] + [(k, True) for k in GOOD])
def test_settings_validation(capi, kw, ok):
    assert F.settings_ok(capi.scan_filter_settings(**kw)) == ok
    assert F.settings_ok(F.settings(**kw)) == ok
