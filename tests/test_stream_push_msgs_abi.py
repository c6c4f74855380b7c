"""CPU-side checks of the messages-from-the-push C-ABI (rpl_capsule_stream_push_laserscan_msgs[_dev]): the header declares
both calls and rpl_push_input, the ctypes struct is the C compiler's layout, and a numpy model of the packing rule
(bound, offsets, capacity) agrees with worked examples.  tests/test_gpu_stream_push_msgs.py holds the device to it."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "rpl_b200.h")


@pytest.fixture(scope="module")
def capi():
    from rplidar_ros2_driver_b200 import capi

    return capi


def _header():
    return re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)


def laserscan_cdr_size(frame_id_len, beams):
    """rpl_laserscan_cdr_size: encapsulation, stamp, frame_id string padded to 4, 7 floats, two float sequences"""
    return 4 + ((12 + frame_id_len + 1 + 3) & ~3) + 28 + 4 + 4 * beams + 4 + 4 * beams


def packing(frame_lens, node_counts, scans_per_stream, max_scans, capacity):
    """(bounds, offsets, total, written): slot i = s * max_scans + k is bounded by its message at the scan's node count,
    rounded up to 16, when k < min(scans_per_stream[s], max_scans), else by 0; offsets are the exclusive scan of the
    bounds; message i is written iff offsets[i] + bounds[i] <= capacity (and it has a bound)"""
    n = len(scans_per_stream)
    bounds = np.zeros(n * max_scans, np.uint64)
    for i in range(n * max_scans):
        s, k = divmod(i, max_scans)
        if k < min(int(scans_per_stream[s]), max_scans):
            bounds[i] = (laserscan_cdr_size(frame_lens[s], int(node_counts[i])) + 15) // 16 * 16
    offsets = np.concatenate([[0], np.cumsum(bounds)[:-1]]).astype(np.uint64)
    total = int(bounds.sum())
    written = (bounds > 0) & (offsets + bounds <= capacity)
    return bounds, offsets, total, written


def test_header_declares_both_calls_and_the_descriptor(capi):
    src = _header()
    assert re.search(r"typedef\s+struct\s+rpl_push_input\s*\{\s*const\s+uint8_t\s*\*\s*data\s*;\s*const\s+uint32_t\s*\*\s*"
                     r"counts\s*;\s*const\s+uint64_t\s*\*\s*rx_us\s*;\s*const\s+rpl_timing\s*\*\s*timing\s*;\s*uint32_t\s+"
                     r"sample_duration_us\s*;\s*uint32_t\s+chunk_bytes\s*;\s*\}\s*rpl_push_input\s*;", src)
    common = (r"\(\s*rpl_capsule_stream\s*\*\s*\w+\s*,\s*const\s+rpl_push_input\s*\*\s*\w+\s*,\s*const\s+rpl_scan_params"
              r"\s*\*\s*\w+\s*,\s*int64_t\s+\w+\s*,\s*uint8_t\s*\*\s*\w+\s*,\s*uint64_t\s+\w+\s*,\s*uint64_t\s*\*\s*\w+\s*,"
              r"\s*uint32_t\s*\*\s*\w+\s*,\s*uint64_t\s*\*\s*\w+\s*,\s*uint32_t\s*\*\s*\w+")
    assert re.search(r"rpl_result\s+rpl_capsule_stream_push_laserscan_msgs\s*" + common + r"\s*\)\s*;", src)
    assert re.search(r"rpl_result\s+rpl_capsule_stream_push_laserscan_msgs_dev\s*" + common +
                     r"\s*,\s*void\s*\*\s*\w+\s*\)\s*;", src)
    assert "rpl_capsule_stream_push_laserscan_msgs" in capi.EXPORTS
    assert "rpl_capsule_stream_push_laserscan_msgs_dev" in capi.EXPORTS


def test_ctypes_struct_layout(capi):
    P = capi.PushInput
    assert ctypes.sizeof(P) == 40
    assert [getattr(P, f).offset for f in ("data", "counts", "rx_us", "timing", "sample_duration_us", "chunk_bytes")] == \
        [0, 8, 16, 24, 32, 36]


@pytest.mark.skipif(shutil.which("cc") is None, reason="no C compiler")
def test_c_layout_is_the_ctypes_layout(capi, tmp_path):
    fields = ("data", "counts", "rx_us", "timing", "sample_duration_us", "chunk_bytes")
    prog = tmp_path / "layout.c"
    prog.write_text(
        '#include <stddef.h>\n#include <stdio.h>\n#include "rpl_b200.h"\n'
        "int main(void) {\n"
        '  printf("%zu' + " %zu" * len(fields) + '\\n", sizeof(rpl_push_input)' +
        "".join(f", offsetof(rpl_push_input, {f})" for f in fields) + ");\n"
        "  return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.run(["cc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()
    P = capi.PushInput
    assert [int(v) for v in out] == [ctypes.sizeof(P)] + [getattr(P, f).offset for f in fields]


def test_cdr_size_model_is_the_library_rule(capi):
    # header bytes for frame_id lengths 0, 1, 3, 4, 255: 20, 20, 20, 24, 272 -- every padding of the string
    assert [laserscan_cdr_size(L, 0) - 36 for L in (0, 1, 3, 4, 255)] == [20, 20, 20, 24, 272]
    L = capi.lib()
    for fl in (0, 1, 2, 3, 4, 5, 11, 254, 255):
        for n in (0, 1, 360, 4097, 8192):
            assert L.rpl_laserscan_cdr_size(fl, n) == laserscan_cdr_size(fl, n)
    assert laserscan_cdr_size(11, 360) == 24 + 4 + 28 + 4 + 1440 + 4 + 1440  # "laser_frame", an A1 revolution


def test_packing_worked_example():
    # two streams, max_scans 3: stream 0 ("ab") published 2 scans of 10 and 3 nodes, stream 1 ("") published 4 -- more
    # than its slots -- of 1, 2, 5 (the fourth dropped)
    node_counts = np.array([10, 3, 0, 1, 2, 5], np.uint32)
    b, o, total, w = packing([2, 0], node_counts, [2, 4], 3, capacity=10 ** 9)
    # "ab": header 20; 10 beams: 20 + 32 + 80 + 4 = 136 -> 144; 3 beams: 80 -> 80; "": 20 + 32 + 8n + 4
    assert b.tolist() == [144, 80, 0, 64, 80, 96]
    assert o.tolist() == [0, 144, 224, 224, 288, 368]
    assert total == 464 and w.tolist() == [True, True, False, True, True, True]


@pytest.mark.parametrize("capacity,written", [
    (0, [False] * 6),
    (100, [False] * 6),                           # ends inside the first message
    (300, [True, True, False, True, False, False]),  # ends inside the message of slot 4 (288..368)
    (368, [True, True, False, True, True, False]),   # exactly at a message's end
    (464, [True, True, False, True, True, True]),    # exactly the total
])
def test_packing_capacity(capacity, written):
    _, o, total, w = packing([2, 0], np.array([10, 3, 0, 1, 2, 5], np.uint32), [2, 4], 3, capacity)
    assert w.tolist() == written
    assert o.tolist() == [0, 144, 224, 224, 288, 368] and total == 464  # offsets and total do not depend on capacity


def test_packing_aligns_every_message_and_leaves_unused_slots_empty():
    rng = np.random.default_rng(7)
    n, ms = 9, 4
    lens = rng.integers(0, 256, n)
    sps = rng.integers(0, 7, n)
    counts = rng.integers(1, 8193, n * ms).astype(np.uint32)
    b, o, total, _ = packing(lens, counts, sps, ms, 0)
    assert (o % 16 == 0).all() and (b % 16 == 0).all() and total == int(b.sum())
    used = np.array([k < min(sps[s], ms) for s in range(n) for k in range(ms)])
    assert (b[~used] == 0).all() and (b[used] >= np.array([laserscan_cdr_size(lens[i // ms], counts[i])
                                                          for i in np.flatnonzero(used)])).all()
