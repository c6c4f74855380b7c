"""CPU-side checks of the session counters' C-ABI: the header declares rpl_capsule_stream_counters and
rpl_stream_counters, whose 14 uint64 fields (112 bytes, in the documented order) are the ctypes binding's dtype."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "rpl_b200.h")
ORDER = ["bytes_in", "frames", "skipped_bytes", "bad_frames", "checksum_errors", "encoder_resets", "scan_resets",
         "discarded_capsules", "nodes", "nodes_unopened", "nodes_overwritten", "scans_rewound", "scans_published",
         "scans_unreturned"]


@pytest.fixture(scope="module")
def capi():
    from rplidar_ros2_driver_b200 import capi

    return capi


def _header():
    return re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)


def test_header_declares_the_call_and_the_struct():
    src = _header()
    assert re.search(r"rpl_result\s+rpl_capsule_stream_counters\s*\(\s*rpl_capsule_stream\s*\*\s*\w+\s*,\s*"
                     r"rpl_stream_counters\s*\*\s*\w+\s*,\s*const\s+uint8_t\s*\*\s*\w+\s*\)\s*;", src)
    body = re.search(r"typedef\s+struct\s+rpl_stream_counters\s*\{(.*?)\}\s*rpl_stream_counters\s*;", src, re.S).group(1)
    assert re.findall(r"uint64_t\s+(\w+)\s*;", body) == ORDER
    assert int(re.search(r"#define\s+RPL_ABI_VERSION\s+(\d+)u", src).group(1)) == 1


def test_numpy_dtype_is_the_struct(capi):
    dt = capi.STREAM_COUNTERS_DTYPE
    assert dt.itemsize == 112 and list(dt.names) == ORDER == list(capi.STREAM_COUNTER_FIELDS)
    assert [dt.fields[f][1] for f in ORDER] == [8 * i for i in range(14)]
    assert all(dt.fields[f][0] == np.dtype("<u8") for f in ORDER)


@pytest.mark.skipif(shutil.which("cc") is None, reason="no C compiler")
def test_c_layout_is_the_numpy_layout(capi, tmp_path):
    prog = tmp_path / "layout.c"
    offs = ", ".join(f"offsetof(rpl_stream_counters, {f})" for f in ORDER)
    prog.write_text(
        '#include <stddef.h>\n#include <stdio.h>\n#include "rpl_b200.h"\n'
        "int main(void) {\n"
        f'  size_t o[] = {{sizeof(rpl_stream_counters), {offs}}};\n'
        '  for (int i = 0; i < 15; ++i) printf("%zu ", o[i]);\n'
        "  return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.run(["cc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert got == [112] + [capi.STREAM_COUNTERS_DTYPE.fields[f][1] for f in ORDER]
