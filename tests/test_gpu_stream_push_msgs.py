"""LaserScan messages from the push (rpl_capsule_stream_push_laserscan_msgs[_dev]).  Every case pairs two sessions fed the
same pieces: A pushes with the entry point of the push's kind and then takes rpl_capsule_stream_laserscan_msgs, B takes
both from the one call.  Message sizes and bytes, scans_per_stream, the offsets (against the bound rule with B's node
counts), the guard bytes behind min(total, capacity), and every later call on the two sessions must agree."""
import ctypes

import numpy as np
import pytest

from test_gpu_capsule_stream import _pieces_from_cuts, _random_cuts
from test_gpu_stream_stamps import _capsule_rx, _normal_rx, _rx_times, _streams
from test_normal_stream_pieces import normal_stream
from test_stream_push_msgs_abi import packing
from test_timestamps_vs_ref import TIMINGS

pytestmark = pytest.mark.gpu

FRAMES = ["", "a", "abc", "abcd", "x" * 255, "laser_frame"]  # 0, 1, 3, 4, 255 characters: every header padding
GUARD = 0xA5
CHUNK = 64  # bytes per receive time of a stamped byte push


@pytest.fixture(scope="module")
def R():
    import rplidar_ros2_driver_b200 as R

    return R


def make_session(R, ctx, kind, ans, n, stride, max_nodes, ms, types=None):
    if types is not None:
        return R.MixedByteStreamSession(ctx, types, stride, max_nodes, ms)
    if kind == "framed":
        return R.CapsuleStreamSession(ctx, ans, n, stride, max_nodes, ms)
    return R.CapsuleByteStreamSession(ctx, ans, n, stride, max_nodes, ms)


class Pair:
    """A: push + laserscan_msgs; B: push_laserscan_msgs.  Fed identical pieces."""

    def __init__(self, R, ctx, kind, ans, n, stride, max_nodes, ms, frames=None, settings=None, types=None):
        self.R, self.kind, self.n, self.stride, self.ms, self.max_nodes = R, kind, n, stride, ms, max_nodes
        self.A = make_session(R, ctx, kind, ans, n, stride, max_nodes, ms, types)
        self.B = make_session(R, ctx, kind, ans, n, stride, max_nodes, ms, types)
        self.frames = frames or [FRAMES[s % len(FRAMES)] for s in range(n)]
        rmax = np.linspace(0.5, 40.0, n).astype(np.float32)
        for x in (self.A, self.B):
            x.set_frames(self.frames, rmax)
            if settings:
                x.set_lidars(settings)
        self.timing = R.Timing(*TIMINGS[0])
        self.n_msgs = 0

    def buffers(self, push):
        n = self.n
        if self.kind == "framed":
            buf = np.zeros((n, self.stride, self.A.capsule_bytes), np.uint8)
        else:
            buf = np.full((n, self.stride), 0xEE, np.uint8)
        cnt = np.zeros(n, np.uint32)
        for s, p in enumerate(push):
            buf[s, : len(p)] = p
            cnt[s] = len(p)
        return buf, cnt

    def push(self, push, prm, off, rx=None, dev=False, capacity=None, timing=True):
        """one push on both; checks the messages; returns B's packed result"""
        buf, cnt = self.buffers(push)
        tm = (self.timing if timing else None) if rx is not None else None
        cb = CHUNK if (rx is not None and self.kind != "framed") else None
        if rx is None:
            out = self.A.push(buf, cnt, prm)
        elif self.kind == "framed":
            out = self.A.push(buf, cnt, prm, rx_us=rx, timing=tm)
        else:
            out = self.A.push(buf, cnt, prm, chunk_bytes=CHUNK, chunk_rx_us=rx, timing=tm)
        exp = self.A.laserscan_msgs(prm, off)
        got = self.push_b(buf, cnt, prm, off, rx, tm, cb, dev, capacity)
        assert got["sps"].tolist() == out["scans_per_stream"].tolist()
        self.check(got, exp, capacity)
        return got

    def push_b(self, buf, cnt, prm, off, rx, tm, cb, dev, capacity):
        ns = self.n * self.ms
        big = ns * ((288 + 32 + 8 * self.max_nodes + 4 + 15) // 16 * 16)
        cap = big if capacity is None else capacity
        if not dev:
            store = np.full(cap + 256, GUARD, np.uint8)
            res, sps = self.B.push_laserscan_msgs(buf, cnt, prm, off, rx_us=rx, timing=tm, chunk_bytes=cb,
                                                  msgs=store[:cap], packed=True)
            res["msgs"], res["sps"], res["capacity"] = store, sps, cap
            return res
        import torch

        d = torch.device("cuda", 0)
        tb = torch.from_numpy(buf).to(d)
        tc = torch.from_numpy(cnt.view(np.int32)).to(d)
        trx = None if rx is None else torch.from_numpy(np.ascontiguousarray(rx).view(np.int64)).to(d)
        store = torch.full((cap + 256,), GUARD, dtype=torch.uint8, device=d)
        offs = torch.full((ns,), -1, dtype=torch.int64, device=d)
        sizes = torch.full((ns,), -1, dtype=torch.int32, device=d)
        total = torch.full((1,), -1, dtype=torch.int64, device=d)
        sps = torch.full((self.n,), -1, dtype=torch.int32, device=d)
        self.B.push_laserscan_msgs_dev(tb.data_ptr(), tc.data_ptr(), prm, off, store.data_ptr(), cap, offs.data_ptr(),
                                       sizes.data_ptr(), total.data_ptr(), sps.data_ptr(),
                                       rx_us=None if trx is None else trx.data_ptr(), timing=tm, chunk_bytes=cb)
        torch.cuda.synchronize()
        return dict(msgs=store.cpu().numpy(), msg_offsets=offs.cpu().numpy().view(np.uint64),
                    msg_sizes=sizes.cpu().numpy().view(np.uint32), total_bytes=int(total.cpu().numpy()[0]),
                    sps=sps.cpu().numpy().view(np.uint32), result=None, capacity=cap)

    def check(self, got, exp, capacity):
        R, ms = self.R, self.ms
        cap = got["capacity"]
        nodes = self.B.nodes(packed=True)
        counts = nodes["node_counts"]
        a_nodes = self.A.nodes(packed=True)["node_counts"]
        assert counts.tolist() == a_nodes.tolist()
        sps = got["sps"]
        bounds, offs, total, written = packing([len(f) for f in self.frames], counts, sps, ms, cap)
        assert got["msg_offsets"].tolist() == offs.tolist()
        assert got["total_bytes"] == total
        if got["result"] is not None:  # the host form's code; the device form reports through total_bytes only
            assert got["result"] == (R.RESULT_OK if total <= cap else R.capi.RESULT_INSUFFICIENT_MEMORY)
        buf = got["msgs"]
        for i, m in enumerate(exp):
            size = int(got["msg_sizes"][i])
            if not written[i] or m is None:
                assert size == 0, i
                continue
            assert size == len(m), i
            o = int(offs[i])
            assert bytes(buf[o:o + size]) == m, i
            self.n_msgs += 1
        assert (buf[min(total, cap):] == GUARD).all()
        if capacity is None:
            assert all((m is None) == (int(got["msg_sizes"][i]) == 0) for i, m in enumerate(exp))

    def compare_after(self, prm, cprm, off):
        """every later read of the last push agrees"""
        A, B = self.A, self.B
        assert [a.tolist() for a in A.state()] == [b.tolist() for b in B.state()]
        assert A.counters().tobytes() == B.counters().tobytes()
        na, sa = A.nodes()
        nb, sb = B.nodes()
        assert [x.tobytes() for x in na] == [x.tobytes() for x in nb] and list(sa) == list(sb)
        assert A.cloud_msgs(cprm, off) == B.cloud_msgs(cprm, off)
        assert A.laserscan_msgs(prm, off) == B.laserscan_msgs(prm, off)

    def close(self):
        self.A.close()
        self.B.close()


def lidar_settings(R, n):
    """streams mixing Mode A / Mode B, inversion and both intensity protocols"""
    return [R.lidar_settings(s % 2, (s // 2) % 2, (s // 4) % 2, R.Timing(*TIMINGS[s % len(TIMINGS)])) for s in range(n)]


def pieces_for(O, kind, ans, n, seed, rng):
    if kind == "framed":
        streams = _streams(O, ans, n, seed)
        cuts = [sorted(set(int(x) for x in rng.integers(1, len(c), 3)) | {len(c)}) for c in streams]
    else:
        streams = [c.reshape(-1) for c in _streams(O, ans, n, seed)]
        cuts = [_random_cuts(rng, len(b), [1, 83, 85, 4000, 20000]) for b in streams]
    cuts[1] = [0] + cuts[1]  # stream 1 pushes nothing the first time
    pieces, _ = _pieces_from_cuts(streams, cuts)
    stride = max(1, max(len(p) for push in pieces for p in push))
    return streams, pieces, stride


def receive_times(kind, rng, streams, pieces, stride):
    if kind == "framed":
        return _capsule_rx(pieces, [_rx_times(rng, len(c)) for c in streams], stride)
    return _normal_rx(rng, pieces, stride, CHUNK)[0]


CASES = [("framed", a) for a in (0x82, 0x83, 0x84, 0x85, 0x86)] + \
        [("bytes", a) for a in (0x81, 0x82, 0x83, 0x84, 0x85, 0x86)]


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
@pytest.mark.parametrize("kind,ans", CASES)
def test_every_answer_type(R, oracle, kind, ans, dev):
    """stamped and unstamped pushes on one session, a reset between pushes, scans dropped past max_scans; the device
    cases with per-stream settings mixing the modes, inversion and protocols"""
    O = oracle
    n, ms = 6, 3
    rng = np.random.default_rng(ans * 4 + dev + (kind == "bytes") * 2)
    streams, pieces, stride = pieces_for(O, kind, ans, n, 7000 + ans, rng)
    rx = receive_times(kind, rng, streams, pieces, stride)
    ctx = R.Context(0, 4096, n * ms)
    p = Pair(R, ctx, kind, ans, n, stride, 4096, ms, settings=lidar_settings(R, n) if dev else None)
    if dev:
        prm = R.scan_params(0, 1, 0, 1, R.FLAG_PER_STREAM)
        cprm = R.cloud_params(flags=R.CLOUD_PER_STREAM)
    else:
        prm = R.scan_params(int(ans % 2), int(ans > 0x83), int(ans % 3 == 0), 1)
        cprm = R.cloud_params(is_new_protocol=int(ans % 2))
    off = -1_234_567_891 if dev else 987_654_321
    for t, push in enumerate(pieces):
        stamped = t % 2 == 0
        p.push(push, prm, off, rx=rx[t] if stamped else None, dev=dev, timing=not dev)
        p.compare_after(prm, cprm, off)
        if t == 1:
            mask = np.zeros(n, np.uint8)
            mask[::2] = 1
            p.A.reset(mask)
            p.B.reset(mask)
    assert p.n_msgs > n
    p.close()
    ctx.close()


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
def test_mixed_byte_session_with_a_switch(R, oracle, dev):
    O = oracle
    types = [0x81, 0x82, 0x83, 0x84, 0x85, 0x86]
    after = [0x85, 0x86, 0x81, 0x82, 0x83, 0x84]
    n, ms = len(types), 3
    rng = np.random.default_rng(11 + dev)
    before_s = [_streams(O, t, 1, 300 + s)[0].reshape(-1) for s, t in enumerate(types)]
    after_s = [_streams(O, t, 1, 400 + s)[0].reshape(-1) for s, t in enumerate(after)]
    cut = lambda b: _random_cuts(rng, len(b), [1, 83, 85, 4000, 20000])  # noqa: E731
    p1, _ = _pieces_from_cuts(before_s, [cut(b) for b in before_s])
    p2, _ = _pieces_from_cuts(after_s, [cut(b) for b in after_s])
    stride = max(len(x) for push in p1 + p2 for x in push)
    rx1 = _normal_rx(rng, p1, stride, CHUNK)[0]
    ctx = R.Context(0, 4096, n * ms)
    p = Pair(R, ctx, "bytes", 0, n, stride, 4096, ms, types=types)
    prm = R.scan_params(1, 0, 1, 1)
    cprm = R.cloud_params(is_new_protocol=1)
    for t, push in enumerate(p1):
        p.push(push, prm, 5, rx=rx1[t] if t % 2 else None, dev=dev)
        p.compare_after(prm, cprm, 5)
    for x in (p.A, p.B):
        x.set_answer_types(after)
    for push in p2:
        p.push(push, prm, 5, dev=dev)
        p.compare_after(prm, cprm, 5)
    assert p.n_msgs > n
    p.close()
    ctx.close()


@pytest.mark.parametrize("flags", [0, "FLAG_FORCE_GENERAL"])
@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
def test_general_kernel_and_large_revolutions(R, oracle, dev, flags):
    """max_nodes 8192 with revolutions above 4096 nodes (0x81), the ultra feed's duplicate measured keys, and every scan
    through the general kernel; one stream's revolution without a measured node (size 0, extent reserved)"""
    O = oracle
    n, ms = 4, 3
    streams = [normal_stream(30000, 77 + s, nodes_per_rev=4100 + 1000 * s, noise=50) for s in range(n)]
    # stream 0: no measured node in its second revolution
    b0 = normal_stream(30000, 77, nodes_per_rev=4100, bad=False).reshape(-1, 5).copy()
    first = int(np.flatnonzero(b0[:, 0] & 1)[1])
    b0[first: first + 4100, 3:5] = 0
    streams[0] = b0.reshape(-1)
    rng = np.random.default_rng(5 + dev)
    cuts = [_random_cuts(rng, len(b), [1, 4, 5000, 40000]) for b in streams]
    pieces, _ = _pieces_from_cuts(streams, cuts)
    stride = max(len(x) for push in pieces for x in push)
    ctx = R.Context(0, 8192, n * ms)
    p = Pair(R, ctx, "bytes", 0x81, n, stride, 8192, ms)
    f = getattr(R, flags) if flags else 0
    prm = R.scan_params(0, 0, 1, 1, f)
    cprm = R.cloud_params()
    empty = 0
    for push in pieces:
        got = p.push(push, prm, 0, dev=dev)
        p.compare_after(prm, cprm, 0)
        empty += int(((got["msg_sizes"] == 0) & (got["msg_offsets"] < np.append(got["msg_offsets"][1:],
                                                                                  got["total_bytes"]))).sum())
    assert empty > 0
    p.close()
    ctx.close()
    # the ultra feed: duplicate measured keys send revolutions to the general kernel from the shared-memory kernel
    streams, pieces, stride = pieces_for(O, "framed", 0x84, 6, 8100, np.random.default_rng(3))
    ctx = R.Context(0, 4096, 18)
    p = Pair(R, ctx, "framed", 0x84, 6, stride, 4096, 3)
    prm = R.scan_params(1, 0, 0, 1)
    for push in pieces:
        p.push(push, prm, 0, dev=dev)
        p.compare_after(prm, R.cloud_params(), 0)
    p.close()
    ctx.close()


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
def test_carry_across_chunks_and_lanes(R, oracle, dev):
    """23 streams: device chunks of 7 (the context's max_scans) and host chunks of 4 (the 16 MiB input rule), so that
    the directory's carry crosses chunk and lane boundaries"""
    O = oracle
    n, ms = 23, 3
    streams = [c.reshape(-1) for c in _streams(O, 0x82, n, 1200)]
    rng = np.random.default_rng(9 + dev)
    cuts = [_random_cuts(rng, len(b), [1, 83, 85, 4000, 20000]) for b in streams]
    pieces, _ = _pieces_from_cuts(streams, cuts)
    stride = (16 << 20) // 5 + 1  # 16 MiB // stride = 4 streams per host chunk
    ctx = R.Context(0, 4096, 7 * ms)
    p = Pair(R, ctx, "bytes", 0x82, n, stride, 4096, ms)
    prm = R.scan_params(0, 1, 0, 1)
    for push in pieces:
        p.push(push, prm, 42, dev=dev)
        p.compare_after(prm, R.cloud_params(), 42)
    assert p.n_msgs > n
    p.close()
    ctx.close()


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
def test_capacity(R, oracle, dev):
    """capacity 0, inside the first message, inside a middle message, exactly the total; then every message again from
    laserscan_msgs on the same push"""
    O = oracle
    n, ms = 6, 3
    rng = np.random.default_rng(21 + dev)
    streams, pieces, stride = pieces_for(O, "framed", 0x85, n, 5100, rng)
    ctx = R.Context(0, 4096, n * ms)
    p = Pair(R, ctx, "framed", 0x85, n, stride, 4096, ms)
    prm = R.scan_params(1, 0, 0, 1)
    probe = Pair(R, ctx, "framed", 0x85, n, stride, 4096, ms)
    for t, push in enumerate(pieces):
        full = probe.push(push, prm, 0)  # the totals and offsets of this push
        offs, total = full["msg_offsets"], full["total_bytes"]
        used = np.flatnonzero(full["msg_sizes"])
        if len(used) < 3:
            caps = [0, total]
        else:
            mid = int(used[len(used) // 2])
            caps = [0, int(offs[used[0]]) + 8, int(offs[mid]) + 8, total]
        cap = caps[t % len(caps)]
        got = p.push(push, prm, 0, dev=dev, capacity=cap)
        assert got["total_bytes"] == total
        assert p.B.laserscan_msgs(prm, 0) == p.A.laserscan_msgs(prm, 0)  # recovery
        p.compare_after(prm, R.cloud_params(), 0)
    probe.close()
    p.close()
    ctx.close()


def test_argument_checks(R, oracle):
    import torch

    O = oracle
    n, ms = 3, 2
    ctx = R.Context(0, 4096, n * ms)
    fr = R.CapsuleStreamSession(ctx, 0x85, n, 8, 4096, ms)
    by = R.CapsuleByteStreamSession(ctx, 0x82, n, 256, 4096, ms)
    L = R.lib()
    prm = R.scan_params(1, 0, 0, 1)
    caps = np.zeros((n, 8, 84), np.uint8)
    cnt = np.zeros(n, np.uint32)
    msgs = np.zeros(1 << 16, np.uint8)
    offs, sizes, total, sps = np.zeros(n * ms, np.uint64), np.zeros(n * ms, np.uint32), np.zeros(1, np.uint64), \
        np.zeros(n, np.uint32)
    P = lambda a: ctypes.c_void_p(a.ctypes.data)  # noqa: E731
    pi = R.PushInput(caps.ctypes.data, cnt.ctypes.data, None, None, 31, 0)
    fn = L.rpl_capsule_stream_push_laserscan_msgs
    ok = fn(fr._h, ctypes.byref(pi), ctypes.byref(prm), 0, P(msgs), msgs.size, P(offs), P(sizes), P(total), P(sps))
    assert ok == R.RESULT_OK
    bad = R.RESULT_INVALID_DATA
    assert fn(fr._h, None, ctypes.byref(prm), 0, P(msgs), msgs.size, P(offs), P(sizes), P(total), P(sps)) == bad
    assert fn(fr._h, ctypes.byref(pi), None, 0, P(msgs), msgs.size, P(offs), P(sizes), P(total), P(sps)) == bad
    for k in range(4):
        a = [P(msgs), P(offs), P(sizes), P(total), P(sps)]
        a[k] = None
        assert fn(fr._h, ctypes.byref(pi), ctypes.byref(prm), 0, a[0], msgs.size, a[1], a[2], a[3], a[4]) == bad
    assert fn(fr._h, ctypes.byref(pi), ctypes.byref(prm), 0, P(msgs), msgs.size, P(offs), P(sizes), P(total), None) == bad
    for field in ("data", "counts"):
        q = R.PushInput(caps.ctypes.data, cnt.ctypes.data, None, None, 31, 0)
        setattr(q, field, None)
        assert fn(fr._h, ctypes.byref(q), ctypes.byref(prm), 0, P(msgs), msgs.size, P(offs), P(sizes), P(total),
                  P(sps)) == bad
    # chunk_bytes on a framed session (a byte input) and on an unstamped byte push
    q = R.PushInput(caps.ctypes.data, cnt.ctypes.data, None, None, 31, 64)
    assert fn(fr._h, ctypes.byref(q), ctypes.byref(prm), 0, P(msgs), msgs.size, P(offs), P(sizes), P(total), P(sps)) == bad
    bb = np.zeros((n, 256), np.uint8)
    q = R.PushInput(bb.ctypes.data, cnt.ctypes.data, None, None, 31, 64)
    assert fn(by._h, ctypes.byref(q), ctypes.byref(prm), 0, P(msgs), msgs.size, P(offs), P(sizes), P(total), P(sps)) == bad
    # a stamped push without timing (and without RPL_FLAG_PER_STREAM), or with chunk_bytes 0 on a byte session
    rx = np.zeros((n, 8), np.uint64)
    q = R.PushInput(caps.ctypes.data, cnt.ctypes.data, rx.ctypes.data, None, 0, 0)
    assert fn(fr._h, ctypes.byref(q), ctypes.byref(prm), 0, P(msgs), msgs.size, P(offs), P(sizes), P(total), P(sps)) == bad
    rxb = np.zeros((n, 4), np.uint64)
    tm = R.Timing(*TIMINGS[0])
    q = R.PushInput(bb.ctypes.data, cnt.ctypes.data, rxb.ctypes.data, ctypes.pointer(tm), 0, 0)
    assert fn(by._h, ctypes.byref(q), ctypes.byref(prm), 0, P(msgs), msgs.size, P(offs), P(sizes), P(total), P(sps)) == bad
    # the unstamped push's sample duration rule; per-stream settings before set_lidars
    q = R.PushInput(caps.ctypes.data, cnt.ctypes.data, None, None, 0, 0)
    assert fn(fr._h, ctypes.byref(q), ctypes.byref(prm), 0, P(msgs), msgs.size, P(offs), P(sizes), P(total), P(sps)) == bad
    pp = R.scan_params(1, 0, 0, 1, R.FLAG_PER_STREAM)
    assert fn(fr._h, ctypes.byref(pi), ctypes.byref(pp), 0, P(msgs), msgs.size, P(offs), P(sizes), P(total), P(sps)) == bad
    # a failed call leaves no last push, as a failed push does
    with pytest.raises(R.RplError):
        fr.laserscan_msgs(prm)
    # misaligned device outputs
    d = torch.device("cuda", 0)
    tcap = torch.zeros((n, 8, 84), dtype=torch.uint8, device=d)
    tcnt = torch.zeros(n, dtype=torch.int32, device=d)
    buf = torch.zeros(1 << 16, dtype=torch.uint8, device=d)
    t64 = torch.zeros(n * ms + 2, dtype=torch.int64, device=d)
    t32 = torch.zeros(n * ms + 2, dtype=torch.int32, device=d)
    one = torch.zeros(2, dtype=torch.int64, device=d)
    s32 = torch.zeros(n + 1, dtype=torch.int32, device=d)
    fd = L.rpl_capsule_stream_push_laserscan_msgs_dev
    q = R.PushInput(tcap.data_ptr(), tcnt.data_ptr(), None, None, 31, 0)
    good = [buf.data_ptr(), t64.data_ptr(), t32.data_ptr(), one.data_ptr(), s32.data_ptr()]
    assert fd(fr._h, ctypes.byref(q), ctypes.byref(prm), 0, *[ctypes.c_void_p(x) for x in good[:1]], 1 << 15,
              *[ctypes.c_void_p(x) for x in good[1:]], None) == R.RESULT_OK
    torch.cuda.synchronize()
    for k, shift in ((0, 4), (1, 4), (2, 2), (3, 4), (4, 2)):
        a = list(good)
        a[k] += shift
        v = [ctypes.c_void_p(x) for x in a]
        assert fd(fr._h, ctypes.byref(q), ctypes.byref(prm), 0, v[0], 1 << 15, v[1], v[2], v[3], v[4], None) == bad, k
    fr.close()
    by.close()
    ctx.close()
