"""CPU-side checks of the per-stream clouds' C-ABI: the header declares rpl_capsule_stream_set_clouds and
RPL_CLOUD_PER_STREAM_CHAIN, rpl_cloud_settings as a C compiler lays it out is the ctypes binding's struct (28 bytes,
the first 24 as rpl_cloud_params), and a model of the message packing with streams that publish no cloud."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "rpl_b200.h")
FIELDS = ("range_min", "range_max", "intensity_min", "voxel_size", "sor_k", "sor_alpha", "enabled", "pad")


@pytest.fixture(scope="module")
def capi():
    from rplidar_ros2_driver_b200 import capi

    return capi


def _header():
    return re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)


def test_header_declares_the_call_and_flag(capi):
    src = _header()
    assert re.search(r"rpl_result\s+rpl_capsule_stream_set_clouds\s*\(\s*rpl_capsule_stream\s*\*\s*\w+\s*,\s*"
                     r"const\s+rpl_cloud_settings\s*\*\s*\w+\s*,\s*const\s+uint8_t\s*\*\s*\w+\s*\)\s*;", src)
    flags = {k: int(v) for k, v in re.findall(r"#define\s+(RPL_CLOUD_\w+)\s+(\d+)u", src)}
    assert flags["RPL_CLOUD_PER_STREAM_CHAIN"] == capi.CLOUD_PER_STREAM_CHAIN == 4
    # one bit, overlapping no other RPL_CLOUD_* bit
    others = [v for k, v in flags.items() if k != "RPL_CLOUD_PER_STREAM_CHAIN"]
    assert others and bin(capi.CLOUD_PER_STREAM_CHAIN).count("1") == 1
    assert all(v & capi.CLOUD_PER_STREAM_CHAIN == 0 for v in others)
    assert capi.CLOUD_PER_STREAM_CHAIN & (capi.CLOUD_NO_FUSED | capi.CLOUD_PER_STREAM) == 0
    assert "rpl_capsule_stream_set_clouds" in capi.EXPORTS


def test_ctypes_struct_layout(capi):
    S, P = capi.CloudSettings, capi.CloudParams
    assert ctypes.sizeof(S) == 28
    assert [getattr(S, f).offset for f in FIELDS] == [0, 4, 8, 12, 16, 20, 24, 25]
    # the chain's six fields sit where rpl_cloud_params has them
    for f in FIELDS[:6]:
        assert getattr(S, f).offset == getattr(P, f).offset
    s = capi.cloud_settings(0.2, 0.0, 3.0, 0.05, 8, 1.5, enabled=False)
    raw = bytes(s)
    assert np.frombuffer(raw[:24], "<f4")[[0, 1, 2, 3, 5]].tolist() == [np.float32(0.2), 0.0, 3.0, np.float32(0.05), 1.5]
    assert int.from_bytes(raw[16:20], "little") == 8 and raw[24:] == bytes(4)


@pytest.mark.skipif(shutil.which("cc") is None, reason="no C compiler")
def test_c_layout_is_the_ctypes_layout(capi, tmp_path):
    prog = tmp_path / "layout.c"
    offs = ", ".join(f"offsetof(rpl_cloud_settings, {f})" for f in FIELDS)
    prog.write_text(
        '#include <stddef.h>\n#include <stdio.h>\n#include "rpl_b200.h"\n'
        "int main(void) {\n"
        f'  printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu\\n", sizeof(rpl_cloud_settings), {offs});\n'
        "  return 0;\n}\n")
    exe = tmp_path / "layout"
    subprocess.run(["cc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)], check=True)
    out = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    S = capi.CloudSettings
    assert out == [ctypes.sizeof(S)] + [getattr(S, f).offset for f in FIELDS]


# ---- the packing of cloud_msgs and push_cloud_msgs with disabled streams (msg_table_kernel, push_msg_dir_kernel) --
def _size(hdr, n):
    return hdr + 116 + 16 * n + 1


def _table(hdr, published, points, enabled, max_scans):
    """msg_table_kernel: every slot's size (0: no message), the exclusive scan of the sizes rounded up to 16, the end
    of the last message"""
    n = len(points)
    s = np.arange(n) // max_scans
    has = published & enabled[s]
    sizes = np.where(has, _size(hdr[s], points), 0).astype(np.int64)
    rounded = (sizes + 15) // 16 * 16
    offs = np.concatenate([[0], np.cumsum(rounded)[:-1]])
    total = int((offs + sizes)[sizes > 0].max()) if (sizes > 0).any() else 0
    return sizes, offs, total


def _directory(hdr, published, points, enabled, max_scans, chunk_streams):
    """push_msg_dir_kernel, chunk by chunk with the carry on the device"""
    n = len(points)
    per = chunk_streams * max_scans
    sizes, offs = np.zeros(n, np.int64), np.zeros(n, np.int64)
    carry, last_end = 0, 0
    for i0 in range(0, n, per):
        sl = slice(i0, min(n, i0 + per))
        sz, of, _ = _table(hdr[i0 // max_scans:], published[sl], points[sl], enabled[i0 // max_scans:], max_scans)
        sizes[sl], offs[sl] = sz, of + carry
        if (sz > 0).any():
            last_end = int((offs[sl] + sz)[sz > 0].max())
        carry += int(((sz + 15) // 16 * 16).sum())
    return sizes, offs, last_end


@pytest.mark.parametrize("seed", range(6))
def test_packing_model_with_disabled_streams(seed):
    rng = np.random.default_rng(seed)
    n_streams, max_scans = int(rng.integers(1, 40)), int(rng.integers(1, 5))
    hdr = rng.integers(1, 70, n_streams) * 4 + 16
    published = rng.random(n_streams * max_scans) < 0.8
    points = rng.integers(0, 4097, n_streams * max_scans) * published
    enabled = rng.random(n_streams) < 0.7
    sizes, offs, total = _table(hdr, published, points, enabled, max_scans)
    # a disabled stream has no message: size 0, and the scan skips it (the next message starts where it would have)
    off_slots = ~enabled[np.arange(n_streams * max_scans) // max_scans]
    assert (sizes[off_slots] == 0).all()
    assert (offs % 16 == 0).all()
    # the same as a session that holds only the enabled streams, packed on their own
    keep = np.flatnonzero(~off_slots)
    s2, o2, t2 = _table(hdr[enabled], published[keep], points[keep], np.ones(int(enabled.sum()), bool), max_scans)
    assert (sizes[keep] == s2).all() and (offs[keep] == o2).all() and total == t2
    # the push's directory, chunk by chunk, gives the same packing
    for chunk in (1, 3, n_streams):
        ds, do, dt = _directory(hdr, published, points, enabled, max_scans, chunk)
        assert (ds == sizes).all() and (do == offs).all() and dt == total
