"""CPU-side checks of the PointCloud2-messages-from-the-push C-ABI (rpl_capsule_stream_push_cloud_msgs[_dev]): the header
declares both calls as the ctypes prototypes take them, and a numpy model of the exact packing -- carried from chunk to
chunk as the push's directories carry it -- equals the packing of rpl_capsule_stream_cloud_msgs over every slot at once,
with the per-message capacity rule writing a prefix.  tests/test_gpu_stream_push_cloud_msgs.py holds the device to it."""
import ctypes
import re

import numpy as np
import pytest

from test_stream_push_msgs_abi import _header


@pytest.fixture(scope="module")
def capi():
    from rplidar_ros2_driver_b200 import capi

    return capi


def pointcloud2_cdr_size(frame_id_len, points):
    """rpl_pointcloud2_cdr_size: encapsulation, stamp, frame_id padded to 4, the 116-byte tail, 16 B a point, is_dense"""
    return 4 + ((12 + frame_id_len + 1 + 3) & ~3) + 116 + 16 * points + 1


def cloud_msgs_packing(frame_lens, point_counts, scans_per_stream, max_scans):
    """(sizes, offsets, total) of rpl_capsule_stream_cloud_msgs over every slot at once: a published slot's message at
    its cloud's point count (empty clouds included), none for an unused slot; offsets the exclusive scan of the sizes
    rounded up to 16; the total the end of the last message"""
    n = len(scans_per_stream)
    sizes = np.zeros(n * max_scans, np.uint64)
    for i in range(n * max_scans):
        s, k = divmod(i, max_scans)
        if k < min(int(scans_per_stream[s]), max_scans):
            sizes[i] = pointcloud2_cdr_size(frame_lens[s], int(point_counts[i]))
    rounded = (sizes + 15) // 16 * 16
    offsets = np.concatenate([[0], np.cumsum(rounded)[:-1]]).astype(np.uint64)
    used = np.flatnonzero(sizes)
    total = int(offsets[used[-1]] + sizes[used[-1]]) if len(used) else 0
    return sizes, offsets, total


def push_packing(frame_lens, point_counts, scans_per_stream, max_scans, chunk, capacity):
    """the push's directories, one per chunk of `chunk` streams, each continuing from the carry the one before it left
    (the running offset and the end of the last message): (offsets, written sizes, total, extents)"""
    n = len(scans_per_stream)
    offsets = np.zeros(n * max_scans, np.uint64)
    written = np.zeros(n * max_scans, np.uint64)
    carry, last_end, extents = 0, 0, []
    for s0 in range(0, n, chunk):
        first, fit_end = carry, carry
        for i in range(s0 * max_scans, min(n, s0 + chunk) * max_scans):
            s, k = divmod(i, max_scans)
            size = pointcloud2_cdr_size(frame_lens[s], int(point_counts[i])) if k < min(int(scans_per_stream[s]),
                                                                                         max_scans) else 0
            offsets[i] = carry
            if size and carry + size <= capacity:
                written[i] = size
                fit_end = max(fit_end, carry + size)
            if size:
                last_end = carry + size
            carry += (size + 15) // 16 * 16
        extents.append((first, fit_end, last_end))
    return offsets, written, last_end, extents


def test_header_declares_both_calls(capi):
    src = _header()
    common = (r"\(\s*rpl_capsule_stream\s*\*\s*\w+\s*,\s*const\s+rpl_push_input\s*\*\s*\w+\s*,\s*const\s+rpl_cloud_params"
              r"\s*\*\s*\w+\s*,\s*int64_t\s+\w+\s*,\s*uint8_t\s*\*\s*\w+\s*,\s*uint64_t\s+\w+\s*,\s*uint64_t\s*\*\s*\w+\s*,"
              r"\s*uint32_t\s*\*\s*\w+\s*,\s*uint64_t\s*\*\s*\w+\s*,\s*uint32_t\s*\*\s*\w+")
    assert re.search(r"rpl_result\s+rpl_capsule_stream_push_cloud_msgs\s*" + common + r"\s*\)\s*;", src)
    assert re.search(r"rpl_result\s+rpl_capsule_stream_push_cloud_msgs_dev\s*" + common +
                     r"\s*,\s*void\s*\*\s*\w+\s*\)\s*;", src)
    assert "rpl_capsule_stream_push_cloud_msgs" in capi.EXPORTS
    assert "rpl_capsule_stream_push_cloud_msgs_dev" in capi.EXPORTS


def test_ctypes_prototypes_match_the_header(capi):
    L = capi.lib()
    P = ctypes.POINTER
    for name, extra in (("rpl_capsule_stream_push_cloud_msgs", []),
                        ("rpl_capsule_stream_push_cloud_msgs_dev", [ctypes.c_void_p])):
        fn = getattr(L, name)
        assert fn.restype == ctypes.c_uint32
        assert list(fn.argtypes) == [ctypes.c_void_p, P(capi.PushInput), P(capi.CloudParams), ctypes.c_int64,
                                     ctypes.c_void_p, ctypes.c_uint64, ctypes.c_void_p, ctypes.c_void_p,
                                     ctypes.c_void_p, ctypes.c_void_p] + extra


def test_cdr_size_model_is_the_library_rule(capi):
    L = capi.lib()
    for fl in (0, 1, 2, 3, 4, 5, 11, 254, 255):
        for n in (0, 1, 360, 4097, 8192):
            assert L.rpl_pointcloud2_cdr_size(fl, n) == pointcloud2_cdr_size(fl, n)


def test_packing_worked_example():
    # two streams, max_scans 3: stream 0 ("ab") published 2 clouds of 10 and 0 points, stream 1 ("") published 4 --
    # more than its slots -- of 1, 2, 5 points (the fourth dropped)
    points = np.array([10, 0, 7, 1, 2, 5], np.uint32)  # slot 2 is unused: its count is not read
    sizes, offs, total = cloud_msgs_packing([2, 0], points, [2, 4], 3)
    # header 20 for both; 20 + 116 + 16 n + 1: 297 -> 304, 137 -> 144, 153 -> 160, 169 -> 176, 217
    assert sizes.tolist() == [297, 137, 0, 153, 169, 217]
    assert offs.tolist() == [0, 304, 448, 448, 608, 784]
    assert total == 784 + 217


@pytest.mark.parametrize("chunk", [1, 2, 3, 5, 7, 11, 64])
def test_carried_packing_is_the_one_pass_packing(chunk):
    """uneven chunks (the last one short), unused slots, streams without a scan, and chunks that end in unused slots:
    the carried offsets and total are those of cloud_msgs over every slot"""
    rng = np.random.default_rng(chunk)
    n, ms = 23, 4
    lens = rng.integers(0, 256, n)
    sps = rng.integers(0, 7, n)
    sps[[3, 4, 5, 21, 22]] = 0  # a chunk may publish nothing, and the push may end without a message
    points = rng.integers(0, 8193, n * ms).astype(np.uint32)
    sizes, offs, total = cloud_msgs_packing(lens, points, sps, ms)
    o, w, t, extents = push_packing(lens, points, sps, ms, chunk, capacity=1 << 62)
    assert o.tolist() == offs.tolist() and t == total and w.tolist() == sizes.tolist()
    assert (o % 16 == 0).all()
    # each chunk's extent: the stretch its messages fill, back to back from chunk to chunk
    assert extents[0][0] == 0
    for (a0, a1, _), (b0, _, _) in zip(extents, extents[1:]):
        assert a0 <= a1 <= b0
    assert extents[-1][2] == total


@pytest.mark.parametrize("chunk", [2, 5])
def test_capacity_writes_a_prefix(chunk):
    rng = np.random.default_rng(40 + chunk)
    n, ms = 13, 3
    lens = rng.integers(0, 40, n)
    sps = rng.integers(0, 5, n)
    points = rng.integers(0, 3000, n * ms).astype(np.uint32)
    sizes, offs, total = cloud_msgs_packing(lens, points, sps, ms)
    used = np.flatnonzero(sizes)
    cuts = [0, total - 1, total, total + 100] + [int(offs[i] + sizes[i]) - 1 for i in used[::3]] + \
        [int(offs[i] + sizes[i]) for i in used[1::3]]
    for cap in cuts:
        o, w, t, extents = push_packing(lens, points, sps, ms, chunk, cap)
        assert o.tolist() == offs.tolist() and t == total  # offsets and total do not depend on capacity
        fits = (sizes > 0) & (offs + sizes <= cap)
        assert w.tolist() == np.where(fits, sizes, 0).tolist()
        # a prefix of the messages: no written message behind one that is not
        k = np.flatnonzero(fits[used])
        assert k.tolist() == list(range(len(k)))
        # nothing written at or past min(total, capacity); each chunk's stretch ends where its last fitting message does
        if fits.any():
            last = int(np.flatnonzero(fits)[-1])
            assert offs[last] + sizes[last] <= min(total, cap)
        assert all(e[1] == e[0] or e[1] <= min(total, cap) for e in extents)
