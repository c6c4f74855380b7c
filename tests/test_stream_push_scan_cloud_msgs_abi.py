"""CPU-side checks of rpl_capsule_stream_push_scan_cloud_msgs[_dev]: the header declares both calls and rpl_msgs_out,
a C compiler lays rpl_msgs_out out as the ctypes binding's MsgsOut, the binding's prototypes are the header's, the
library refuses null arguments without a device, and a numpy model of the two packings: the clouds' offsets carried
from chunk to chunk equal the one-pass packing, and skip the slots whose LaserScan message was not written."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from test_stream_push_msgs_abi import packing

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "rpl_b200.h")
NAMES = ("rpl_capsule_stream_push_scan_cloud_msgs", "rpl_capsule_stream_push_scan_cloud_msgs_dev")


@pytest.fixture(scope="module")
def capi():
    from rplidar_ros2_driver_b200 import capi

    return capi


def _header():
    return re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)


def test_header_declares_both_calls_and_the_struct(capi):
    src = _header()
    P = r"\s*\*\s*\w+\s*"
    assert re.search(r"typedef\s+struct\s+rpl_msgs_out\s*\{\s*uint8_t" + P + r";\s*uint64_t\s+capacity\s*;\s*uint64_t"
                     + P + r";\s*uint32_t" + P + r";\s*uint64_t" + P + r";\s*\}\s*rpl_msgs_out\s*;", src)
    common = (r"\(\s*rpl_capsule_stream" + P + r",\s*const\s+rpl_push_input" + P + r",\s*const\s+rpl_scan_params" + P +
              r",\s*const\s+rpl_scan_cloud_params" + P + r",\s*int64_t\s+\w+\s*,\s*const\s+rpl_msgs_out" + P +
              r",\s*const\s+rpl_msgs_out" + P + r",\s*uint32_t" + P)
    assert re.search(r"rpl_result\s+rpl_capsule_stream_push_scan_cloud_msgs\s*" + common + r"\)\s*;", src)
    assert re.search(r"rpl_result\s+rpl_capsule_stream_push_scan_cloud_msgs_dev\s*" + common + r",\s*void" + P +
                     r"\)\s*;", src)
    for name in NAMES:
        assert name in capi.EXPORTS


def test_ctypes_prototypes(capi):
    L = capi.lib()
    vp = ctypes.c_void_p
    base = [vp, ctypes.POINTER(capi.PushInput), ctypes.POINTER(capi.ScanParams), ctypes.POINTER(capi.ScanCloudParams),
            ctypes.c_int64, ctypes.POINTER(capi.MsgsOut), ctypes.POINTER(capi.MsgsOut), vp]
    assert L.rpl_capsule_stream_push_scan_cloud_msgs.argtypes == base
    assert L.rpl_capsule_stream_push_scan_cloud_msgs_dev.argtypes == base + [vp]
    for name in NAMES:
        assert getattr(L, name).restype == ctypes.c_uint32


def test_library_refuses_null_arguments(capi):
    L = capi.lib()
    bad = capi.RESULT_INVALID_DATA
    p, cp = capi.scan_params(), capi.scan_cloud_params()
    o = capi.MsgsOut()
    assert L.rpl_capsule_stream_push_scan_cloud_msgs(None, None, ctypes.byref(p), ctypes.byref(cp), 0, ctypes.byref(o),
                                                     ctypes.byref(o), None) == bad
    assert L.rpl_capsule_stream_push_scan_cloud_msgs_dev(None, None, ctypes.byref(p), ctypes.byref(cp), 0,
                                                         ctypes.byref(o), ctypes.byref(o), None, None) == bad


def test_msgs_out_layout(capi):
    S = capi.MsgsOut
    assert ctypes.sizeof(S) == 40
    assert [S.msgs.offset, S.capacity.offset, S.msg_offsets.offset, S.msg_sizes.offset, S.total_bytes.offset] == \
        [0, 8, 16, 24, 32]


@pytest.mark.skipif(shutil.which("cc") is None, reason="no C compiler")
def test_c_layout_is_the_ctypes_layout(tmp_path):
    prog = tmp_path / "layout.c"
    prog.write_text(
        '#include <stddef.h>\n#include <stdio.h>\n#include "rpl_b200.h"\n'
        "int main(void) {\n"
        '  printf("%zu %zu %zu %zu %zu %zu\\n", sizeof(rpl_msgs_out), offsetof(rpl_msgs_out, msgs), '
        "offsetof(rpl_msgs_out, capacity), offsetof(rpl_msgs_out, msg_offsets), offsetof(rpl_msgs_out, msg_sizes), "
        "offsetof(rpl_msgs_out, total_bytes));\n"
        "  return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.run(["cc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)], check=True)
    out = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert out == [40, 0, 8, 16, 24, 32]


# ---- the packings ------------------------------------------------------------------------------------------------
def cloud_size(hdr_bytes, tail_bytes, point_step, kept):
    return hdr_bytes + tail_bytes + point_step * kept + 1


def one_pass(sizes, capacity):
    """scan_cloud_msgs' packing of exact sizes (0: no message): offsets, the total (end of the last message), and the
    per-message rule of the push forms (written iff offset + size <= capacity)"""
    r = (sizes + 15) // 16 * 16
    offs = np.concatenate([[0], np.cumsum(r)[:-1]]).astype(np.uint64)
    nz = np.flatnonzero(sizes)
    total = int(offs[nz[-1]] + sizes[nz[-1]]) if len(nz) else 0
    return offs, total, (sizes > 0) & (offs + sizes <= capacity)


def carried(sizes, chunk_slots, capacity):
    """push_msg_dir_kernel<kScanCloud> chunk by chunk: the running offset and the end of the last message pass through
    the carry pair"""
    carry, last = 0, 0
    offs = np.zeros(len(sizes), np.uint64)
    written = np.zeros(len(sizes), bool)
    for c0 in range(0, len(sizes), chunk_slots):
        for i in range(c0, min(c0 + chunk_slots, len(sizes))):
            offs[i] = carry
            if sizes[i]:
                written[i] = carry + sizes[i] <= capacity
                last = carry + int(sizes[i])
            carry += (int(sizes[i]) + 15) // 16 * 16
    return offs, last, written


def model(rng, n, ms, frame_lens, point_step, tail_bytes, scan_capacity):
    """one push: the LaserScan packing under scan_capacity, then the clouds' sizes of the written scans"""
    counts = rng.integers(0, 5000, n * ms)
    sps = rng.integers(0, ms + 2, n)
    _, _, _, written = packing(frame_lens, counts, sps, ms, scan_capacity)
    beams = np.where(written, counts, 0)  # a written scan's beam count (here: its node count)
    kept = np.array([rng.integers(0, b + 1) if b else 0 for b in beams])
    hdr = np.array([4 + ((12 + frame_lens[i // ms] + 1 + 3) & ~3) for i in range(n * ms)])
    sizes = np.where(written & (beams > 0), cloud_size(hdr, tail_bytes, point_step, kept), 0).astype(np.uint64)
    return written, sizes


@pytest.mark.parametrize("seed", range(6))
def test_carried_cloud_packing_is_the_one_pass_packing(seed):
    rng = np.random.default_rng(seed)
    n, ms = 23, 3
    frame_lens = [int(x) for x in rng.integers(0, 256, n)]
    _, sizes = model(rng, n, ms, frame_lens, 12 + 4 * (seed % 5), 100 + 4 * seed, 1 << 40)
    offs, total, _ = one_pass(sizes, 1 << 40)
    for chunk_streams in (1, 3, 4, 7, n):
        c_offs, c_total, _ = carried(sizes, chunk_streams * ms, 1 << 40)
        assert c_offs.tolist() == offs.tolist() and c_total == total
    for cap in (0, total - 1, total, int(offs[len(offs) // 2]) + 5):
        _, _, w1 = one_pass(sizes, cap)
        _, _, w2 = carried(sizes, 3 * ms, cap)
        assert w1.tolist() == w2.tolist()
        idx = np.flatnonzero(sizes)
        assert not any(w1[idx[k + 1]] and not w1[idx[k]] for k in range(len(idx) - 1))  # a prefix


def test_unwritten_scans_take_no_cloud_room():
    rng = np.random.default_rng(7)
    n, ms = 9, 3
    frame_lens = [3] * n
    counts = rng.integers(100, 5000, n * ms)
    sps = np.full(n, ms)
    _, s_offs, s_total, _ = packing(frame_lens, counts, sps, ms, 1 << 40)
    cap = int(s_offs[n * ms // 2]) + 8  # inside the middle scan's message: it and every scan after it do not fit
    _, _, _, written = packing(frame_lens, counts, sps, ms, cap)
    assert written[: n * ms // 2].all() and not written[n * ms // 2:].any()
    kept = counts // 2
    sizes = np.where(written, cloud_size(20, 132, 20, kept), 0).astype(np.uint64)
    offs, total, _ = one_pass(sizes, 1 << 40)
    # the clouds past the cut have size 0 and the same offset, the end of the last written cloud's room
    tail = offs[n * ms // 2:]
    assert (tail == tail[0]).all() and total == int(offs[n * ms // 2 - 1] + sizes[n * ms // 2 - 1])
