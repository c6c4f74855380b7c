"""LaserScan filters on the device (rpl_scan_filter_batch_dev, rpl_capsule_stream_set_scan_filters,
RPL_FLAG_PER_STREAM_FILTERS) against their definition, oracle/scan_filter_oracle.py.

The stateless call must be the restatement bit for bit on rows of rpl_scan_batch_dev.  The session cases pair two
sessions fed the same pieces: A makes the call without the flag and the restatement is applied to its outputs on the
host, B makes the flagged call.  Ranges, intensities, beam counts, increments, scans_per_stream, message offsets, sizes
and bytes must be identical, and so must every later call that ignores the flag."""
import ctypes
import math

import numpy as np
import pytest

from oracle import scan_filter_oracle as F
from test_gpu_capsule_stream import _pieces_from_cuts, _random_cuts
from test_gpu_stream_push_msgs import CHUNK, Pair, lidar_settings, make_session, pieces_for, receive_times
from test_normal_stream_pieces import normal_stream
from test_scan_filters_abi import BAD, GOOD
from test_timestamps_vs_ref import TIMINGS

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def R():
    import rplidar_ros2_driver_b200 as R

    return R


def fleet_filters(R, n):
    """every stage alone, the whole chain, and disabled streams"""
    table = [
        R.scan_filter_settings(mask=[(0.0, 0.3), (5.9, 2 * math.pi)], range_lo=0.2, range_hi=8.0, intensity_min=2.0,
                               speckle_window=3, speckle_min_neighbours=2, speckle_max_diff=0.05, shadow_window=8,
                               shadow_angle=math.radians(10)),
        R.scan_filter_settings(enabled=False, speckle_window=2, speckle_min_neighbours=4, speckle_max_diff=0.0),
        R.scan_filter_settings(mask=[(1.0, 2.5)]),
        R.scan_filter_settings(range_lo=1.0, range_hi=5.0),
        R.scan_filter_settings(intensity_min=20.0),
        R.scan_filter_settings(speckle_window=1, speckle_min_neighbours=1, speckle_max_diff=0.02),
        R.scan_filter_settings(shadow_window=16, shadow_angle=math.radians(20)),
    ]
    return [table[s % len(table)] for s in range(n)]


def flagged(R, prm):
    return R.scan_params(prm.is_new_protocol, prm.scan_processing, prm.inverted, prm.apply_ascend,
                         prm.flags | R.FLAG_PER_STREAM_FILTERS)


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def filter_msg(m, e):
    """F applied to one serialised LaserScan: the ranges rewritten in place, everything else as it is"""
    if m is None:
        return None
    L = int(np.frombuffer(m, "<u4", 1, 12)[0])  # frame_id length with its NUL
    hb = 4 + ((12 + L + 3) & ~3)
    inc = np.frombuffer(m, "<f4", 1, hb + 8)[0]
    M = int(np.frombuffer(m, "<u4", 1, hb + 28)[0])
    r = np.frombuffer(m, "<f4", M, hb + 32)
    it = np.frombuffer(m, "<f4", M, hb + 32 + 4 * M + 4)
    return m[:hb + 32] + F.filter_scan(e, r, it, inc).tobytes() + m[hb + 32 + 4 * M:]


def filter_msgs(msgs, table, ms):
    return [filter_msg(m, table[i // ms]) for i, m in enumerate(msgs)]


# ---- the stateless primitive -------------------------------------------------------------------------------------
STAGES = {
    "mask": dict(mask=[(0.0, 0.5), (3.0, 3.1), (6.0, 2 * math.pi), (2.0, 1.0)]),
    "range": dict(range_lo=0.5, range_hi=6.0),
    "intensity": dict(intensity_min=10.0),
    "speckle": dict(speckle_window=4, speckle_min_neighbours=3, speckle_max_diff=0.03),
    "shadow": dict(shadow_window=16, shadow_angle=math.radians(12)),
    "chain": dict(mask=[(0.2, 0.4)], range_lo=0.3, range_hi=7.0, intensity_min=3.0, speckle_window=2,
                  speckle_min_neighbours=1, speckle_max_diff=0.05, shadow_window=5, shadow_angle=math.radians(8)),
}


def _batch_rows(R, O, ctx, mode_a, inv, seed):
    counts = np.array([1, 2, 3, 4, 17, 360, 1000, 3200, 4095, 4096, 4097, 8000, 8191, 8192], np.uint32)
    nodes = O.synth_batch(seed, len(counts), 8192, seed % 5)
    return ctx.scan_batch(nodes.view(R.NODE_DTYPE), counts, R.scan_params(seed % 2, mode_a, inv, 1))


def _filter_dev(R, ctx, s, out):
    import torch

    d = torch.device("cuda", 0)
    n, stride = out["ranges"].shape
    tr = torch.from_numpy(np.ascontiguousarray(out["ranges"])).to(d)
    ti = torch.from_numpy(np.ascontiguousarray(out["intensities"])).to(d)
    tb = torch.from_numpy(out["beam_counts"].view(np.int32)).to(d)
    ta = torch.from_numpy(out["angle_increment"]).to(d)
    ctx.scan_filter_batch_dev(s, tr.data_ptr(), ti.data_ptr(), tb.data_ptr(), ta.data_ptr(), n, stride)
    torch.cuda.synchronize()
    return tr.cpu().numpy(), ti.cpu().numpy()


@pytest.mark.parametrize("mode_a,inv", [(0, 0), (0, 1), (1, 0), (1, 1)])
def test_batch_dev_is_the_restatement(R, oracle, mode_a, inv):
    ctx = R.Context(0, 8192, 16)
    removed = 0
    for k, (name, kw) in enumerate(STAGES.items()):
        out = _batch_rows(R, oracle, ctx, mode_a, inv, 10 * k + 2 * mode_a + inv)
        assert out["beam_counts"].max() > 4096
        s = R.scan_filter_settings(**kw)
        got_r, got_i = _filter_dev(R, ctx, s, out)
        want = F.filter_rows(s, out["ranges"], out["intensities"], out["beam_counts"], out["angle_increment"])
        assert (bits(got_r) == bits(want)).all(), name
        assert (bits(got_i) == bits(out["intensities"])).all()
        removed += int((bits(got_r) != bits(out["ranges"])).sum())
    assert removed > 0
    ctx.close()


@pytest.mark.parametrize("seed", range(4))
def test_batch_dev_random_settings(R, oracle, seed):
    from test_scan_filters_oracle import _random_settings

    rng = np.random.default_rng(seed)
    ctx = R.Context(0, 8192, 16)
    for t in range(3):
        out = _batch_rows(R, oracle, ctx, int(rng.integers(0, 2)), int(rng.integers(0, 2)), 100 + 3 * seed + t)
        e = _random_settings(rng)
        s = R.scan_filter_settings(mask=list(zip(e.mask_lo, e.mask_hi)), range_lo=e.range_lo, range_hi=e.range_hi,
                                   intensity_min=e.intensity_min, speckle_window=e.speckle_window,
                                   speckle_min_neighbours=e.speckle_min_neighbours,
                                   speckle_max_diff=e.speckle_max_diff, shadow_window=e.shadow_window,
                                   shadow_angle=e.shadow_angle)
        got_r, _ = _filter_dev(R, ctx, s, out)
        want = F.filter_rows(s, out["ranges"], out["intensities"], out["beam_counts"], out["angle_increment"])
        assert (bits(got_r) == bits(want)).all()
    ctx.close()


# ---- sessions: rows and the messages of the last push --------------------------------------------------------------
class RowPair:
    """A: the calls without the flag, the restatement on the host; B: the flagged calls."""

    def __init__(self, R, ctx, kind, ans, n, stride, max_nodes, ms, table, lidars=None, types=None):
        self.R, self.kind, self.n, self.stride, self.ms = R, kind, n, stride, ms
        self.A = make_session(R, ctx, kind, ans, n, stride, max_nodes, ms, types)
        self.B = make_session(R, ctx, kind, ans, n, stride, max_nodes, ms, types)
        for x in (self.A, self.B):
            x.set_frames([f"laser_{s}" for s in range(n)])
            if lidars:
                x.set_lidars(lidars)
        self.table = list(table)
        self.B.set_scan_filters(self.table)
        self.timing = R.Timing(*TIMINGS[0])
        self.changed = 0

    def buffers(self, push):
        if self.kind == "framed":
            buf = np.zeros((self.n, self.stride, self.A.capsule_bytes), np.uint8)
        else:
            buf = np.full((self.n, self.stride), 0xEE, np.uint8)
        cnt = np.zeros(self.n, np.uint32)
        for s, p in enumerate(push):
            buf[s, : len(p)] = p
            cnt[s] = len(p)
        return buf, cnt

    def _push_host(self, x, buf, cnt, prm, rx):
        if rx is None:
            return x.push(buf, cnt, prm)
        tm = None if prm.flags & self.R.FLAG_PER_STREAM else self.timing
        if self.kind == "framed":
            return x.push(buf, cnt, prm, rx_us=rx, timing=tm)
        return x.push(buf, cnt, prm, chunk_bytes=CHUNK, chunk_rx_us=rx, timing=tm)

    def _push_dev(self, x, buf, cnt, prm, rx):
        import torch

        d = torch.device("cuda", 0)
        ns, mn = self.n * self.ms, x.max_nodes
        o = {k: torch.full(shape, -1, dtype=dt, device=d) for k, shape, dt in (
            ("ranges", (ns, mn), torch.float32), ("intensities", (ns, mn), torch.float32),
            ("beam_counts", (ns,), torch.int32), ("angle_increment", (ns,), torch.float32),
            ("scans_per_stream", (self.n,), torch.int32), ("scan_begin_ts_us", (ns,), torch.int64))}
        tb = torch.from_numpy(buf).to(d)
        tc = torch.from_numpy(cnt.view(np.int32)).to(d)
        a = [o[k].data_ptr() for k in ("ranges", "intensities", "beam_counts", "angle_increment", "scans_per_stream")]
        if rx is None:
            x.push_dev(tb.data_ptr(), tc.data_ptr(), prm, *a)
        else:
            trx = torch.from_numpy(np.ascontiguousarray(rx).view(np.int64)).to(d)
            tm = None if prm.flags & self.R.FLAG_PER_STREAM else self.timing
            if self.kind == "framed":
                x.push_dev(tb.data_ptr(), tc.data_ptr(), prm, *a, rx_us=trx.data_ptr(), timing=tm,
                           scan_begin_ts_us=o["scan_begin_ts_us"].data_ptr())
            else:
                x.push_dev(tb.data_ptr(), tc.data_ptr(), prm, *a, chunk_bytes=CHUNK, chunk_rx_us=trx.data_ptr(),
                           timing=tm, scan_begin_ts_us=o["scan_begin_ts_us"].data_ptr())
        torch.cuda.synchronize()
        out = {k: v.cpu().numpy() for k, v in o.items()}
        for k in ("beam_counts", "scans_per_stream"):
            out[k] = out[k].view(np.uint32)
        if rx is None:
            del out["scan_begin_ts_us"]
        return out

    def push(self, push, prm, rx=None, dev=False):
        """every output of the scans the push published (a row past its beam count, and a slot the push did not
        publish, hold whatever the staging held)"""
        buf, cnt = self.buffers(push)
        fn = self._push_dev if dev else self._push_host
        a = fn(self.A, buf, cnt, prm, rx)
        b = fn(self.B, buf, cnt, flagged(self.R, prm), rx)
        assert sorted(a) == sorted(b)
        sps = a["scans_per_stream"]
        assert sps.tolist() == b["scans_per_stream"].tolist()
        used = np.flatnonzero(np.arange(self.ms)[None, :] < sps[:, None])  # slot s * ms + j, j < sps[s]
        for k in ("beam_counts", "angle_increment", "scan_begin_ts_us"):
            if k in a:
                assert a[k][used].tobytes() == b[k][used].tobytes(), k
        for i in used:
            M = int(a["beam_counts"][i])
            want = F.filter_scan(self.table[i // self.ms], a["ranges"][i, :M], a["intensities"][i, :M],
                                 a["angle_increment"][i])
            assert (bits(b["ranges"][i, :M]) == bits(want)).all(), i
            assert (bits(b["intensities"][i, :M]) == bits(a["intensities"][i, :M])).all(), i
            self.changed += int((bits(want) != bits(a["ranges"][i, :M])).sum())

    def compare_after(self, prm):
        """the last push's LaserScan messages with the flag, and every call that ignores it"""
        R, A, B = self.R, self.A, self.B
        assert filter_msgs(A.laserscan_msgs(prm, 7), self.table, self.ms) == B.laserscan_msgs(flagged(R, prm), 7)
        assert A.laserscan_msgs(prm, 7) == B.laserscan_msgs(prm, 7)
        cprm = R.cloud_params(is_new_protocol=prm.is_new_protocol)
        assert A.cloud_msgs(cprm, 7) == B.cloud_msgs(cprm, 7)
        assert A.counters().tobytes() == B.counters().tobytes()
        na, sa = A.nodes()
        nb, sb = B.nodes()
        assert [x.tobytes() for x in na] == [x.tobytes() for x in nb] and list(sa) == list(sb)

    def close(self):
        self.A.close()
        self.B.close()


CASES = [("framed", a) for a in (0x82, 0x83, 0x84, 0x85, 0x86)] + \
        [("bytes", a) for a in (0x81, 0x82, 0x83, 0x84, 0x85, 0x86)]


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
@pytest.mark.parametrize("kind,ans", CASES)
def test_session_rows_every_answer_type(R, oracle, kind, ans, dev):
    """stamped and unstamped pushes; the device cases with per-stream lidar settings mixing Mode A / B and inversion"""
    n, ms = 7, 3
    rng = np.random.default_rng(ans * 4 + dev + (kind == "bytes") * 2)
    streams, pieces, stride = pieces_for(oracle, kind, ans, n, 9000 + ans, rng)
    rx = receive_times(kind, rng, streams, pieces, stride)
    ctx = R.Context(0, 4096, n * ms)
    lid = lidar_settings(R, n) if dev else None
    p = RowPair(R, ctx, kind, ans, n, stride, 4096, ms, fleet_filters(R, n), lidars=lid)
    prm = R.scan_params(0, 1, 0, 1, R.FLAG_PER_STREAM) if dev else R.scan_params(int(ans % 2), int(ans > 0x83),
                                                                                int(ans % 3 == 0), 1)
    for t, push in enumerate(pieces):
        p.push(push, prm, rx=rx[t] if t % 2 == 0 else None, dev=dev)
        p.compare_after(prm)
    assert p.changed > 0
    p.close()
    ctx.close()


# ---- sessions: messages from the push -----------------------------------------------------------------------------
class MsgPair(Pair):
    """Pair of test_gpu_stream_push_msgs with B flagged: A's push and laserscan_msgs without the flag, the restatement
    applied to its messages on the host"""

    def __init__(self, R, ctx, kind, ans, n, stride, max_nodes, ms, table, settings=None, types=None):
        super().__init__(R, ctx, kind, ans, n, stride, max_nodes, ms, settings=settings, types=types)
        self.table = list(table)
        self.B.set_scan_filters(self.table)

    def push(self, push, prm, off, rx=None, dev=False, capacity=None, timing=True):
        buf, cnt = self.buffers(push)
        tm = (self.timing if timing else None) if rx is not None else None
        cb = CHUNK if (rx is not None and self.kind != "framed") else None
        if rx is None:
            out = self.A.push(buf, cnt, prm)
        elif self.kind == "framed":
            out = self.A.push(buf, cnt, prm, rx_us=rx, timing=tm)
        else:
            out = self.A.push(buf, cnt, prm, chunk_bytes=CHUNK, chunk_rx_us=rx, timing=tm)
        exp = filter_msgs(self.A.laserscan_msgs(prm, off), self.table, self.ms)
        got = self.push_b(buf, cnt, flagged(self.R, prm), off, rx, tm, cb, dev, capacity)
        assert got["sps"].tolist() == out["scans_per_stream"].tolist()
        self.check(got, exp, capacity)
        return got

    def compare_after(self, prm, cprm, off):
        super().compare_after(prm, cprm, off)
        exp = filter_msgs(self.A.laserscan_msgs(prm, off), self.table, self.ms)
        assert exp == self.B.laserscan_msgs(flagged(self.R, prm), off)


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
@pytest.mark.parametrize("kind,ans", CASES)
def test_push_msgs_every_answer_type(R, oracle, kind, ans, dev):
    n, ms = 7, 3
    rng = np.random.default_rng(ans * 8 + dev + (kind == "bytes") * 2)
    streams, pieces, stride = pieces_for(oracle, kind, ans, n, 9100 + ans, rng)
    rx = receive_times(kind, rng, streams, pieces, stride)
    ctx = R.Context(0, 4096, n * ms)
    p = MsgPair(R, ctx, kind, ans, n, stride, 4096, ms, fleet_filters(R, n),
                settings=lidar_settings(R, n) if dev else None)
    if dev:
        prm = R.scan_params(0, 1, 0, 1, R.FLAG_PER_STREAM)
        cprm = R.cloud_params(flags=R.CLOUD_PER_STREAM)
    else:
        prm = R.scan_params(int(ans % 2), int(ans > 0x83), int(ans % 3 == 0), 1)
        cprm = R.cloud_params(is_new_protocol=int(ans % 2))
    for t, push in enumerate(pieces):
        p.push(push, prm, 11, rx=rx[t] if t % 2 == 0 else None, dev=dev, timing=not dev)
        p.compare_after(prm, cprm, 11)
    assert p.n_msgs > n
    p.close()
    ctx.close()


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
def test_mixed_byte_session_with_a_switch(R, oracle, dev):
    from test_gpu_stream_stamps import _normal_rx, _streams

    O = oracle
    types = [0x81, 0x82, 0x83, 0x84, 0x85, 0x86]
    after = [0x85, 0x86, 0x81, 0x82, 0x83, 0x84]
    n, ms = len(types), 3
    rng = np.random.default_rng(21 + dev)
    before_s = [_streams(O, t, 1, 500 + s)[0].reshape(-1) for s, t in enumerate(types)]
    after_s = [_streams(O, t, 1, 600 + s)[0].reshape(-1) for s, t in enumerate(after)]
    cut = lambda b: _random_cuts(rng, len(b), [1, 83, 85, 4000, 20000])  # noqa: E731
    p1, _ = _pieces_from_cuts(before_s, [cut(b) for b in before_s])
    p2, _ = _pieces_from_cuts(after_s, [cut(b) for b in after_s])
    stride = max(len(x) for push in p1 + p2 for x in push)
    rx1 = _normal_rx(rng, p1, stride, CHUNK)[0]
    ctx = R.Context(0, 4096, n * ms)
    table = fleet_filters(R, n)[::-1]
    p = MsgPair(R, ctx, "bytes", 0, n, stride, 4096, ms, table, types=types)
    rp = RowPair(R, ctx, "bytes", 0, n, stride, 4096, ms, table, types=types)
    prm = R.scan_params(1, 0, 1, 1)
    cprm = R.cloud_params(is_new_protocol=1)
    for t, push in enumerate(p1):
        p.push(push, prm, 5, rx=rx1[t] if t % 2 else None, dev=dev)
        p.compare_after(prm, cprm, 5)
        rp.push(push, prm, rx=rx1[t] if t % 2 else None, dev=dev)
        rp.compare_after(prm)
    for x in (p.A, p.B, rp.A, rp.B):
        x.set_answer_types(after)
    for push in p2:
        p.push(push, prm, 5, dev=dev)
        p.compare_after(prm, cprm, 5)
        rp.push(push, prm, dev=dev)
        rp.compare_after(prm)
    p.close()
    rp.close()
    ctx.close()


@pytest.mark.parametrize("flags", [0, "FLAG_FORCE_GENERAL"])
@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
def test_general_kernel_and_8192_node_holders(R, oracle, dev, flags):
    """max_nodes 8192 with revolutions up to 8192 nodes (0x81), and the ultra feed's duplicate measured keys, which send
    revolutions to the general kernel"""
    n, ms = 4, 3
    streams = [normal_stream(30000, 177 + s, nodes_per_rev=5192 + 1000 * s, noise=50) for s in range(n)]
    rng = np.random.default_rng(15 + dev)
    cuts = [_random_cuts(rng, len(b), [1, 4, 5000, 40000]) for b in streams]
    pieces, _ = _pieces_from_cuts(streams, cuts)
    stride = max(len(x) for push in pieces for x in push)
    ctx = R.Context(0, 8192, n * ms)
    f = getattr(R, flags) if flags else 0
    prm = R.scan_params(0, 0, 1, 1, f)
    table = fleet_filters(R, n)
    p = MsgPair(R, ctx, "bytes", 0x81, n, stride, 8192, ms, table)
    rp = RowPair(R, ctx, "bytes", 0x81, n, stride, 8192, ms, table)
    big = 0
    for push in pieces:
        p.push(push, prm, 0, dev=dev)
        p.compare_after(prm, R.cloud_params(), 0)
        rp.push(push, prm, dev=dev)
        rp.compare_after(prm)
        big = max(big, int(rp.B.nodes(packed=True)["node_counts"].max()))
    assert big >= 8000
    p.close()
    rp.close()
    ctx.close()
    streams, pieces, stride = pieces_for(oracle, "framed", 0x84, 6, 8200, np.random.default_rng(4))
    ctx = R.Context(0, 4096, 18)
    table = fleet_filters(R, 6)
    p = MsgPair(R, ctx, "framed", 0x84, 6, stride, 4096, 3, table)
    rp = RowPair(R, ctx, "framed", 0x84, 6, stride, 4096, 3, table)
    prm = R.scan_params(1, 0, 0, 1, f)
    for push in pieces:
        p.push(push, prm, 0, dev=dev)
        p.compare_after(prm, R.cloud_params(), 0)
        rp.push(push, prm, dev=dev)
        rp.compare_after(prm)
    p.close()
    rp.close()
    ctx.close()


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
def test_several_chunks_per_push(R, oracle, dev):
    """23 streams: device chunks of 7 (the context's max_scans / max_scans) and host chunks of 4 (the 16 MiB input
    rule); chunks without an enabled stream launch no filter"""
    n, ms = 23, 3
    from test_gpu_stream_stamps import _streams

    streams = [c.reshape(-1) for c in _streams(oracle, 0x82, n, 1300)]
    rng = np.random.default_rng(19 + dev)
    cuts = [_random_cuts(rng, len(b), [1, 83, 85, 4000, 20000]) for b in streams]
    pieces, _ = _pieces_from_cuts(streams, cuts)
    stride = (16 << 20) // 5 + 1
    ctx = R.Context(0, 4096, 7 * ms)
    table = fleet_filters(R, n)
    for s in range(7, 14):  # the second device chunk: every stream disabled
        table[s] = R.scan_filter_settings(enabled=False)
    p = MsgPair(R, ctx, "bytes", 0x82, n, stride, 4096, ms, table)
    rp = RowPair(R, ctx, "bytes", 0x82, n, stride, 4096, ms, table)
    prm = R.scan_params(0, 1, 0, 1)
    for push in pieces:
        p.push(push, prm, 42, dev=dev)
        p.compare_after(prm, R.cloud_params(), 42)
        rp.push(push, prm, dev=dev)
        rp.compare_after(prm)
    p.close()
    rp.close()
    ctx.close()


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
def test_push_msgs_capacity(R, oracle, dev):
    """capacity 0, inside the first message, inside a middle message, exactly the total"""
    n, ms = 6, 3
    rng = np.random.default_rng(31 + dev)
    streams, pieces, stride = pieces_for(oracle, "framed", 0x85, n, 5200, rng)
    ctx = R.Context(0, 4096, n * ms)
    table = fleet_filters(R, n)
    p = MsgPair(R, ctx, "framed", 0x85, n, stride, 4096, ms, table)
    probe = MsgPair(R, ctx, "framed", 0x85, n, stride, 4096, ms, table)
    prm = R.scan_params(1, 0, 0, 1)
    for t, push in enumerate(pieces):
        full = probe.push(push, prm, 0)
        offs, total = full["msg_offsets"], full["total_bytes"]
        used = np.flatnonzero(full["msg_sizes"])
        caps = [0, total] if len(used) < 3 else [0, int(offs[used[0]]) + 8, int(offs[used[len(used) // 2]]) + 8, total]
        got = p.push(push, prm, 0, dev=dev, capacity=caps[t % len(caps)])
        assert got["total_bytes"] == total
        p.compare_after(prm, R.cloud_params(), 0)
    probe.close()
    p.close()
    ctx.close()


def test_every_stream_disabled_is_the_unflagged_call(R, oracle):
    n, ms = 5, 3
    rng = np.random.default_rng(41)
    streams, pieces, stride = pieces_for(oracle, "framed", 0x83, n, 5300, rng)
    ctx = R.Context(0, 4096, n * ms)
    off = [R.scan_filter_settings(enabled=False, **kw) for kw in STAGES.values()][:n]
    p = MsgPair(R, ctx, "framed", 0x83, n, stride, 4096, ms, off)
    rp = RowPair(R, ctx, "framed", 0x83, n, stride, 4096, ms, off)
    prm = R.scan_params(1, 1, 1, 1)
    for push in pieces:
        p.push(push, prm, 3)
        p.compare_after(prm, R.cloud_params(), 3)
        rp.push(push, prm)
        rp.compare_after(prm)
    # no filter launch: the flagged push on B makes the launches of the unflagged one on A (same state, same input)
    buf, cnt = rp.buffers(pieces[0])
    before = ctx.launch_count
    a = rp.A.push(buf, cnt, prm)
    plain = ctx.launch_count - before
    before = ctx.launch_count
    b = rp.B.push(buf, cnt, flagged(R, prm))
    assert ctx.launch_count - before == plain
    assert all((np.ascontiguousarray(a[k]).view(np.uint8) == np.ascontiguousarray(b[k]).view(np.uint8)).all() for k in a)
    p.close()
    rp.close()
    ctx.close()


# ---- argument checks ---------------------------------------------------------------------------------------------
def test_argument_checks(R, oracle):
    import torch

    n, ms = 3, 2
    ctx = R.Context(0, 4096, n * ms)
    fr = R.CapsuleStreamSession(ctx, 0x85, n, 8, 4096, ms)
    L = R.lib()
    bad = R.RESULT_INVALID_DATA
    prm = R.scan_params(1, 0, 0, 1)
    fprm = flagged(R, prm)
    caps = np.zeros((n, 8, 84), np.uint8)
    cnt = np.zeros(n, np.uint32)
    # the flag before the first set_scan_filters: every flagged call is refused
    with pytest.raises(R.RplError) as e:
        fr.push(caps, cnt, fprm)
    assert e.value.code == bad
    with pytest.raises(R.RplError) as e:
        fr.push_laserscan_msgs(caps, cnt, fprm)
    assert e.value.code == bad
    fr.push(caps, cnt, prm)
    with pytest.raises(R.RplError) as e:
        fr.laserscan_msgs(fprm)
    assert e.value.code == bad
    # the first call must set every stream; a null table
    arr = (R.ScanFilterSettings * n)(*[R.scan_filter_settings()] * n)
    m = np.array([1, 0, 1], np.uint8)
    fn = L.rpl_capsule_stream_set_scan_filters
    assert fn(fr._h, ctypes.cast(arr, ctypes.c_void_p), ctypes.c_void_p(m.ctypes.data)) == bad
    assert fn(fr._h, None, None) == bad
    # every entry outside the limits is refused, and the table stays as it was
    keep = [R.scan_filter_settings(range_lo=0.5 + s) for s in range(n)]
    fr.set_scan_filters(keep)
    fr.push(caps, cnt, prm)
    ref = fr.laserscan_msgs(fprm)
    for kw in BAD:
        with pytest.raises(R.RplError) as e:
            fr.set_scan_filters([R.scan_filter_settings()] * (n - 1) + [R.scan_filter_settings(**kw)])
        assert e.value.code == bad
        assert fr.laserscan_msgs(fprm) == ref
    for kw in GOOD:
        fr.set_scan_filters([R.scan_filter_settings(**kw)] * n, mask=[0, 1, 0])
    # the stateless call's checks
    d = torch.device("cuda", 0)
    rows = torch.zeros((4, 8192), dtype=torch.float32, device=d)
    beams = torch.ones(4, dtype=torch.int32, device=d)
    inc = torch.ones(4, dtype=torch.float32, device=d)
    s = R.scan_filter_settings(speckle_window=1, speckle_min_neighbours=1)
    ctx.scan_filter_batch_dev(s, rows.data_ptr(), rows.data_ptr(), beams.data_ptr(), inc.data_ptr(), 4, 8192)
    with pytest.raises(R.RplError) as e:
        ctx.scan_filter_batch_dev(s, rows.data_ptr(), rows.data_ptr(), beams.data_ptr(), inc.data_ptr(), 4, 8193)
    assert e.value.code == bad
    for kw in BAD:
        with pytest.raises(R.RplError) as e:
            ctx.scan_filter_batch_dev(R.scan_filter_settings(**kw), rows.data_ptr(), rows.data_ptr(),
                                      beams.data_ptr(), inc.data_ptr(), 4, 8192)
        assert e.value.code == bad
    for k in range(4):
        a = [rows.data_ptr(), rows.data_ptr(), beams.data_ptr(), inc.data_ptr()]
        a[k] = None
        with pytest.raises(R.RplError):
            ctx.scan_filter_batch_dev(s, *a, 4, 8192)
    torch.cuda.synchronize()
    assert (rows[:, 1:] == 0).all() and torch.isnan(rows[:, 0]).all()  # M = 1: no neighbour, removed
    # a flagged device push needs angle_increment
    tcap = torch.zeros((n, 8, 84), dtype=torch.uint8, device=d)
    tcnt = torch.zeros(n, dtype=torch.int32, device=d)
    o = torch.zeros((n * ms, 4096), dtype=torch.float32, device=d)
    b = torch.zeros(n * ms, dtype=torch.int32, device=d)
    sp = torch.zeros(n, dtype=torch.int32, device=d)
    with pytest.raises(R.RplError) as e:
        fr.push_dev(tcap.data_ptr(), tcnt.data_ptr(), fprm, o.data_ptr(), o.data_ptr(), b.data_ptr(), None,
                    sp.data_ptr())
    assert e.value.code == bad
    fr.push_dev(tcap.data_ptr(), tcnt.data_ptr(), prm, o.data_ptr(), o.data_ptr(), b.data_ptr(), None, sp.data_ptr())
    torch.cuda.synchronize()
    fr.close()
    ctx.close()
