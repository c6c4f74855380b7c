"""LaserScans and their projected clouds from the push (rpl_capsule_stream_push_scan_cloud_msgs[_dev]).  Every case pairs
two sessions fed the same pieces, with the same lidar, filter and footprint tables: A pushes with
rpl_capsule_stream_push_laserscan_msgs (the same scan capacity) and then takes rpl_capsule_stream_scan_cloud_msgs, B
takes both from the one call.  B's LaserScan side must be A's push output in every case; its cloud side must be A's
projection of each LaserScan message B wrote, packed exactly (the clouds of unwritten scans have size 0 and no room),
written iff it fits, with nothing at or past min(total, capacity) touched in either buffer.  Every later call on the
two sessions must agree."""
import ctypes
import math

import numpy as np
import pytest

from oracle import cdr_oracle as CDR
from test_gpu_capsule_stream import _pieces_from_cuts, _random_cuts
from test_gpu_scan_cloud import CUTOFFS
from test_gpu_scan_filters import fleet_filters, flagged
from test_gpu_scan_footprints import fleet_footprints
from test_gpu_stream_push_msgs import CASES, CHUNK, GUARD, Pair, lidar_settings, pieces_for, receive_times
from test_gpu_stream_stamps import _normal_rx, _streams
from test_normal_stream_pieces import normal_stream
from test_timestamps_vs_ref import TIMINGS

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def R():
    import rplidar_ros2_driver_b200 as R

    return R


def channel_sets(R):
    """laser_geometry's default, every channel, none, distances and stamps"""
    return [R.scan_cloud_params(), R.scan_cloud_params(0x0F, 6.0), R.scan_cloud_params(0),
            R.scan_cloud_params(R.SCAN_CLOUD_TIMESTAMP | R.SCAN_CLOUD_DISTANCE, 0.0)]


def exclusive(sizes):
    return np.concatenate([[0], np.cumsum([(int(s) + 15) // 16 * 16 for s in sizes])[:-1]]).astype(np.uint64)


class ScanCloudPair(Pair):
    """A: push_laserscan_msgs + scan_cloud_msgs; B: push_scan_cloud_msgs.  Fed identical pieces."""

    def __init__(self, R, ctx, kind, ans, n, stride, max_nodes, ms, table=None, fps=None, settings=None, types=None):
        super().__init__(R, ctx, kind, ans, n, stride, max_nodes, ms, settings=settings, types=types)
        for x in (self.A, self.B):
            if table is not None:
                x.set_scan_filters(table)
            if fps is not None:
                x.set_scan_footprints(fps)
        self.points = self.empty = self.cut_scans = self.cut_clouds = 0

    def scan_big(self):
        return self.n * self.ms * ((288 + 32 + 8 * self.max_nodes + 4 + 15) // 16 * 16)

    def cloud_big(self, cp):
        per = 288 + 192 + self.R.capi.scan_cloud_point_step(cp.channels) * self.max_nodes + 1
        return self.n * self.ms * ((per + 15) // 16 * 16)

    def push(self, push, prm, cp, off, rx=None, dev=False, scap=None, ccap=None, timing=True):
        """one push on both; checks both sets; returns B's (scans, clouds)"""
        buf, cnt = self.buffers(push)
        tm = (self.timing if timing else None) if rx is not None else None
        cb = CHUNK if (rx is not None and self.kind != "framed") else None
        scap = self.scan_big() if scap is None else scap
        ccap = self.cloud_big(cp) if ccap is None else ccap
        exp, a_sps = self.A.push_laserscan_msgs(buf, cnt, prm, off, rx_us=rx, timing=tm, chunk_bytes=cb,
                                                msgs=np.zeros(scap, np.uint8), packed=True)
        a_clouds = self.A.scan_cloud_msgs(prm, cp, off)  # every slot's, from the replay
        scans, clouds = self.push_b(buf, cnt, prm, cp, off, rx, tm, cb, dev, scap, ccap)
        assert scans["sps"].tolist() == a_sps.tolist()
        self.check_scans(scans, exp, scap)
        self.check_clouds(clouds, scans, a_clouds, ccap)
        if scans["result"] is not None:
            over = scans["total_bytes"] > scap or clouds["total_bytes"] > ccap
            assert scans["result"] == (self.R.capi.RESULT_INSUFFICIENT_MEMORY if over else self.R.RESULT_OK)
        return scans, clouds

    def push_b(self, buf, cnt, prm, cp, off, rx, tm, cb, dev, scap, ccap):
        ns = self.n * self.ms
        if not dev:
            ss, cs = np.full(scap + 256, GUARD, np.uint8), np.full(ccap + 256, GUARD, np.uint8)
            scans, clouds, sps = self.B.push_scan_cloud_msgs(buf, cnt, prm, cp, off, rx_us=rx, timing=tm,
                                                             chunk_bytes=cb, msgs=ss[:scap], cloud_msgs=cs[:ccap])
            scans["msgs"], clouds["msgs"], scans["sps"] = ss, cs, sps
            return scans, clouds
        import torch

        R = self.R
        d = torch.device("cuda", 0)
        tb = torch.from_numpy(buf).to(d)
        tc = torch.from_numpy(cnt.view(np.int32)).to(d)
        trx = None if rx is None else torch.from_numpy(np.ascontiguousarray(rx).view(np.int64)).to(d)
        sets = []
        for cap in (scap, ccap):
            t = dict(store=torch.full((cap + 256,), GUARD, dtype=torch.uint8, device=d),
                     offs=torch.full((ns,), -1, dtype=torch.int64, device=d),
                     sizes=torch.full((ns,), -1, dtype=torch.int32, device=d),
                     total=torch.full((1,), -1, dtype=torch.int64, device=d))
            t["out"] = R.MsgsOut(t["store"].data_ptr(), cap, t["offs"].data_ptr(), t["sizes"].data_ptr(),
                                 t["total"].data_ptr())
            sets.append(t)
        sps = torch.full((self.n,), -1, dtype=torch.int32, device=d)
        torch.cuda.synchronize()  # the context's stream does not wait for torch's
        self.B.push_scan_cloud_msgs_dev(tb.data_ptr(), tc.data_ptr(), prm, cp, off, sets[0]["out"], sets[1]["out"],
                                        sps.data_ptr(), rx_us=None if trx is None else trx.data_ptr(), timing=tm,
                                        chunk_bytes=cb)
        torch.cuda.synchronize()
        res = [dict(msgs=t["store"].cpu().numpy(), msg_offsets=t["offs"].cpu().numpy().view(np.uint64),
                    msg_sizes=t["sizes"].cpu().numpy().view(np.uint32), total_bytes=int(t["total"].cpu().numpy()[0]),
                    result=None) for t in sets]
        res[0]["sps"] = sps.cpu().numpy().view(np.uint32)
        return res[0], res[1]

    def check_scans(self, got, exp, cap):
        """A's push_laserscan_msgs output: offsets, sizes, total, every written message's bytes; B's guard bytes"""
        assert got["msg_offsets"].tolist() == exp["msg_offsets"].tolist()
        assert got["msg_sizes"].tolist() == exp["msg_sizes"].tolist()
        assert got["total_bytes"] == exp["total_bytes"]
        buf, ref = got["msgs"], exp["msgs"]
        for i in np.flatnonzero(exp["msg_sizes"]):
            o, n = int(exp["msg_offsets"][i]), int(exp["msg_sizes"][i])
            assert bytes(buf[o:o + n]) == bytes(ref[o:o + n]), i
        assert (buf[min(got["total_bytes"], cap):] == GUARD).all()
        self.cut_scans += int(got["total_bytes"] > cap)

    def check_clouds(self, got, scans, a_clouds, cap):
        """the projection of every LaserScan message B wrote, packed exactly, written iff it fits"""
        want = [m if m is not None and scans["msg_sizes"][i] > 0 else None for i, m in enumerate(a_clouds)]
        assert all((m is None) == (s == 0) for m, s in zip(want, scans["msg_sizes"]))  # a cloud iff a scan message
        sizes = np.array([0 if m is None else len(m) for m in want], np.uint64)
        offs = exclusive(sizes)
        total = max([int(o) + int(s) for o, s in zip(offs, sizes) if s] or [0])
        assert got["msg_offsets"].tolist() == offs.tolist()
        assert got["total_bytes"] == total
        fits = (sizes > 0) & (offs + sizes <= cap)
        assert got["msg_sizes"].tolist() == np.where(fits, sizes, 0).tolist()
        buf = got["msgs"]
        for i in np.flatnonzero(fits):
            o = int(offs[i])
            assert bytes(buf[o:o + int(sizes[i])]) == want[i], i
            w = CDR.parse_pointcloud2(want[i])["width"]
            self.points += w
            self.empty += int(w == 0)
            self.n_msgs += 1
        assert (buf[min(total, cap):] == GUARD).all()
        self.cut_clouds += int(total > cap)

    def compare_after(self, prm, cp, off):
        """every later read of the last push agrees"""
        super().compare_after(prm, self.R.cloud_params(), off)
        assert self.A.scan_cloud_msgs(prm, cp, off) == self.B.scan_cloud_msgs(prm, cp, off)


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
@pytest.mark.parametrize("kind,ans", CASES)
def test_every_answer_type(R, oracle, kind, ans, dev):
    """stamped and unstamped pushes with a nonzero clock offset, a reset between pushes, scans dropped past max_scans,
    the filters and footprints on every other push; the device cases with per-stream lidars mixing Mode A / B and
    inversion"""
    n, ms = 7, 3
    rng = np.random.default_rng(ans * 4 + dev + (kind == "bytes") * 2 + 5000)
    streams, pieces, stride = pieces_for(oracle, kind, ans, n, 9900 + ans, rng)
    rx = receive_times(kind, rng, streams, pieces, stride)
    ctx = R.Context(0, 4096, n * ms)
    p = ScanCloudPair(R, ctx, kind, ans, n, stride, 4096, ms, fleet_filters(R, n), fleet_footprints(R, n),
                      settings=lidar_settings(R, n) if dev else None)
    base = R.scan_params(0, 1, 0, 1, R.FLAG_PER_STREAM) if dev else R.scan_params(int(ans % 2), int(ans > 0x83),
                                                                                 int(ans % 3 == 0), 1)
    cps = channel_sets(R)
    off = -1_234_567_891 if dev else 987_654_321
    for t, push in enumerate(pieces):
        prm = flagged(R, base) if t % 2 == 0 else base
        p.push(push, prm, cps[t % len(cps)], off, rx=rx[t] if t % 2 == 0 else None, dev=dev, timing=not dev)
        p.compare_after(prm, cps[(t + 1) % len(cps)], off)
        if t == 1:
            mask = np.zeros(n, np.uint8)
            mask[::2] = 1
            p.A.reset(mask)
            p.B.reset(mask)
    assert p.n_msgs > n and p.points > 0
    p.close()
    ctx.close()


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
def test_mixed_byte_session_with_a_switch(R, oracle, dev):
    types = [0x81, 0x82, 0x83, 0x84, 0x85, 0x86]
    after = [0x85, 0x86, 0x81, 0x82, 0x83, 0x84]
    n, ms = len(types), 3
    rng = np.random.default_rng(71 + dev)
    before_s = [_streams(oracle, t, 1, 910 + s)[0].reshape(-1) for s, t in enumerate(types)]
    after_s = [_streams(oracle, t, 1, 920 + s)[0].reshape(-1) for s, t in enumerate(after)]
    cut = lambda b: _random_cuts(rng, len(b), [1, 83, 85, 4000, 20000])  # noqa: E731
    p1, _ = _pieces_from_cuts(before_s, [cut(b) for b in before_s])
    p2, _ = _pieces_from_cuts(after_s, [cut(b) for b in after_s])
    stride = max(len(x) for push in p1 + p2 for x in push)
    rx1 = _normal_rx(rng, p1, stride, CHUNK)[0]
    ctx = R.Context(0, 4096, n * ms)
    p = ScanCloudPair(R, ctx, "bytes", 0, n, stride, 4096, ms, fleet_filters(R, n), fleet_footprints(R, n),
                      types=types)
    prm = flagged(R, R.scan_params(1, 0, 1, 1))
    cps = channel_sets(R)
    for t, push in enumerate(p1):
        p.push(push, prm, cps[t % 4], 5, rx=rx1[t] if t % 2 else None, dev=dev)
        p.compare_after(prm, cps[t % 4], 5)
    for x in (p.A, p.B):
        x.set_answer_types(after)
    for t, push in enumerate(p2):
        p.push(push, prm, cps[(t + 2) % 4], 5, dev=dev)
        p.compare_after(prm, cps[t % 4], 5)
    assert p.n_msgs > n
    p.close()
    ctx.close()


def test_every_channel_set_and_cutoff(R, oracle):
    """all 16 channel sets, each with one of the cutoffs of the projection's tests, host and device pushes"""
    n, ms = 5, 3
    rng = np.random.default_rng(88)
    streams, pieces, stride = pieces_for(oracle, "framed", 0x85, n, 9800, rng)
    rx = receive_times("framed", rng, streams, pieces, stride)
    ctx = R.Context(0, 4096, n * ms)
    p = ScanCloudPair(R, ctx, "framed", 0x85, n, stride, 4096, ms, fleet_filters(R, n), fleet_footprints(R, n),
                      settings=lidar_settings(R, n))
    prm = flagged(R, R.scan_params(0, 1, 0, 1, R.FLAG_PER_STREAM))
    for ch in range(16):
        t = ch % len(pieces)
        cp = R.scan_cloud_params(ch, CUTOFFS[ch % len(CUTOFFS)])
        p.push(pieces[t], prm, cp, 77 * ch, rx=rx[t] if ch % 2 else None, dev=ch % 3 == 0)
        p.compare_after(prm, cp, 77 * ch)
    assert p.n_msgs > n
    p.close()
    ctx.close()


@pytest.mark.parametrize("flags", [0, "FLAG_FORCE_GENERAL"])
@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
def test_large_revolutions_and_the_general_kernel(R, oracle, dev, flags):
    """8192-node holders with revolutions above 4096 nodes, every scan through the general kernel, and the ultra feed's
    duplicate measured keys (the shared-memory kernel's hand-off to the general kernel)"""
    n, ms = 4, 3
    streams = [normal_stream(30000, 377 + s, nodes_per_rev=4100 + 1000 * s, noise=50) for s in range(n)]
    rng = np.random.default_rng(25 + dev)
    cuts = [_random_cuts(rng, len(b), [1, 4, 5000, 40000]) for b in streams]
    pieces, _ = _pieces_from_cuts(streams, cuts)
    stride = max(len(x) for push in pieces for x in push)
    ctx = R.Context(0, 8192, n * ms)
    p = ScanCloudPair(R, ctx, "bytes", 0x81, n, stride, 8192, ms, fleet_filters(R, n), fleet_footprints(R, n))
    f = getattr(R, flags) if flags else 0
    cps = channel_sets(R)
    for t, push in enumerate(pieces):
        prm = R.scan_params(0, t % 2, 1, 1, f | (R.FLAG_PER_STREAM_FILTERS if t % 2 else 0))
        p.push(push, prm, cps[t % 4], 0, dev=dev)
        p.compare_after(prm, cps[t % 4], 0)
    assert p.n_msgs > 0
    p.close()
    ctx.close()
    streams, pieces, stride = pieces_for(oracle, "framed", 0x84, 6, 8300, np.random.default_rng(13))
    ctx = R.Context(0, 4096, 18)
    p = ScanCloudPair(R, ctx, "framed", 0x84, 6, stride, 4096, 3)
    prm = R.scan_params(1, 0, 0, 1, f)
    for push in pieces:
        p.push(push, prm, cps[1], 0, dev=dev)
        p.compare_after(prm, cps[1], 0)
    p.close()
    ctx.close()


def fleet(R, oracle, seed):
    """23 streams whose last 7 are idle on every other push, a filter table with disabled entries and a stream whose
    filters remove every beam, and footprints"""
    n, ms = 23, 3
    streams = [c.reshape(-1) for c in _streams(oracle, 0x82, n, seed)]
    rng = np.random.default_rng(seed)
    cuts = [_random_cuts(rng, len(b), [1, 83, 85, 4000, 20000]) for b in streams]
    pieces, _ = _pieces_from_cuts(streams, cuts)
    for push in pieces[::2]:  # the last device chunk and most of the last two host chunks idle
        for s in range(16, n):
            push[s] = push[s][:0]
    stride = (16 << 20) // 5 + 1  # 16 MiB // stride = 4 streams per host chunk
    rx = _normal_rx(rng, pieces, stride, CHUNK)[0]
    table = fleet_filters(R, n)
    table[3] = R.scan_filter_settings(range_lo=1e6, range_hi=1e7)  # every beam removed: width-0 clouds
    table[4] = R.scan_filter_settings(enabled=False)
    return n, ms, pieces, stride, rx, table


def test_fleet_carries_across_chunks_lanes_and_forms(R, oracle):
    """device chunks of 3 streams and host chunks of 4, host and device calls alternating on one session: both
    directories' carries cross chunk and lane boundaries"""
    n, ms, pieces, stride, rx, table = fleet(R, oracle, 1400)
    ctx = R.Context(0, 4096, 3 * ms)
    p = ScanCloudPair(R, ctx, "bytes", 0x82, n, stride, 4096, ms, table, fleet_footprints(R, n))
    prm = flagged(R, R.scan_params(0, 1, 0, 1))
    cps = channel_sets(R)
    for t, push in enumerate(pieces):
        p.push(push, prm, cps[t % 4], 42, rx=rx[t] if t % 2 == 0 else None, dev=(t // 2) % 2 == 1)
        p.compare_after(prm, cps[t % 4], 42)
    assert p.n_msgs > n and p.empty > 0
    p.close()
    ctx.close()


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
def test_capacity(R, oracle, dev):
    """the scan capacity exactly met and one byte short in a middle chunk (the clouds of unwritten scans have size 0
    and take no room); the cloud capacity exactly met and one byte short (the written clouds are a prefix); then every
    message again from laserscan_msgs and scan_cloud_msgs on the same push"""
    n, ms, pieces, stride, rx, table = fleet(R, oracle, 1500)
    ctx = R.Context(0, 4096, 3 * ms)
    p = ScanCloudPair(R, ctx, "bytes", 0x82, n, stride, 4096, ms, table, fleet_footprints(R, n))
    probe = ScanCloudPair(R, ctx, "bytes", 0x82, n, stride, 4096, ms, table, fleet_footprints(R, n))
    prm = flagged(R, R.scan_params(0, 1, 0, 1))
    cp = R.scan_cloud_params(0x0B)
    for t, push in enumerate(pieces):
        scans, clouds = probe.push(push, prm, cp, 7)  # the totals and offsets of this push
        s_used, c_used = np.flatnonzero(scans["msg_sizes"]), np.flatnonzero(clouds["msg_sizes"])
        s_tot, c_tot = scans["total_bytes"], clouds["total_bytes"]
        # both exactly met; a middle scan message (of a middle chunk) one byte short; a middle cloud one byte short; the
        # last cloud one byte short (without three messages: the last one)
        cases = [(s_tot, c_tot), (max(s_tot - 1, 1), None), (None, max(c_tot - 1, 1)), (None, max(c_tot - 1, 1))]
        if len(s_used) >= 3:
            mid = int(s_used[len(s_used) // 2])
            cases[1] = (int(scans["msg_offsets"][mid]) + int(scans["msg_sizes"][mid]) - 1, None)
        if len(c_used) >= 3:
            mid = int(c_used[len(c_used) // 2])
            cases[2] = (None, int(clouds["msg_offsets"][mid]) + int(clouds["msg_sizes"][mid]) - 1)
        scap, ccap = cases[t % len(cases)]
        got_s, got_c = p.push(push, prm, cp, 7, dev=dev, scap=scap, ccap=ccap)
        assert got_s["total_bytes"] == s_tot
        if scap is not None and scap < s_tot:  # the clouds of the unwritten scans take no room
            assert got_c["total_bytes"] <= c_tot
        assert p.B.laserscan_msgs(prm, 7) == p.A.laserscan_msgs(prm, 7)  # recovery
        p.compare_after(prm, cp, 7)
    assert p.cut_scans > 0 and p.cut_clouds > 0
    probe.close()
    p.close()
    ctx.close()


def test_argument_checks(R, oracle):
    import torch

    n, ms = 3, 2
    ctx = R.Context(0, 4096, n * ms)
    fr = R.CapsuleStreamSession(ctx, 0x85, n, 8, 4096, ms)
    by = R.CapsuleByteStreamSession(ctx, 0x82, n, 256, 4096, ms)
    L = R.lib()
    prm = R.scan_params(1, 0, 0, 1)
    cp = R.scan_cloud_params()
    caps = np.zeros((n, 8, 84), np.uint8)
    cnt = np.zeros(n, np.uint32)
    host = [dict(msgs=np.zeros(1 << 16, np.uint8), offs=np.zeros(n * ms, np.uint64), sizes=np.zeros(n * ms, np.uint32),
                 total=np.zeros(1, np.uint64)) for _ in range(2)]
    outs = [R.MsgsOut(h["msgs"].ctypes.data, h["msgs"].size, h["offs"].ctypes.data, h["sizes"].ctypes.data,
                      h["total"].ctypes.data) for h in host]
    sps = np.zeros(n, np.uint32)
    P = lambda a: ctypes.c_void_p(a.ctypes.data)  # noqa: E731
    pi = R.PushInput(caps.ctypes.data, cnt.ctypes.data, None, None, 31, 0)
    fn = L.rpl_capsule_stream_push_scan_cloud_msgs
    bad = R.RESULT_INVALID_DATA
    ref = lambda x: None if x is None else ctypes.byref(x)  # noqa: E731

    def call(sess, q, p, c, s, cl, spsp):
        return fn(sess._h, ref(q), ref(p), ref(c), 0, ref(s), ref(cl), spsp)

    def ok(sess, q=pi):
        assert call(sess, q, prm, cp, outs[0], outs[1], P(sps)) == R.RESULT_OK
        assert sess.scan_cloud_msgs(prm, cp) is not None

    def fails(sess, q, p, c, s, cl, spsp=None):
        """refused, and the session left as the refused push would: no last push"""
        assert call(sess, q, p, c, s, cl, P(sps) if spsp is None else spsp) == bad
        with pytest.raises(R.RplError):
            sess.laserscan_msgs(prm)

    for args in ((None, prm, cp, outs[0], outs[1]), (pi, None, cp, outs[0], outs[1]), (pi, prm, None, outs[0], outs[1]),
                 (pi, prm, cp, None, outs[1]), (pi, prm, cp, outs[0], None)):
        ok(fr)
        fails(fr, *args)
    ok(fr)
    assert call(fr, pi, prm, cp, outs[0], outs[1], None) == bad
    for k, field in enumerate(("msgs", "msg_offsets", "msg_sizes", "total_bytes") * 2):
        ok(fr)
        o = [R.MsgsOut.from_buffer_copy(x) for x in outs]
        setattr(o[k // 4], field, None)
        fails(fr, pi, prm, cp, o[0], o[1])
    for field in ("data", "counts"):
        ok(fr)
        q = R.PushInput(caps.ctypes.data, cnt.ctypes.data, None, None, 31, 0)
        setattr(q, field, None)
        fails(fr, q, prm, cp, outs[0], outs[1])
    # the projection's rules: an unknown channel bit (the viewpoint), a NaN cutoff
    for c in (R.scan_cloud_params(0x10), R.scan_cloud_params(0x03, math.nan)):
        ok(fr)
        fails(fr, pi, prm, c, outs[0], outs[1])
    # chunk_bytes on a framed session and on an unstamped byte push; the unstamped sample duration rule
    ok(fr)
    fails(fr, R.PushInput(caps.ctypes.data, cnt.ctypes.data, None, None, 31, 64), prm, cp, outs[0], outs[1])
    bb = np.zeros((n, 256), np.uint8)
    ok(by, R.PushInput(bb.ctypes.data, cnt.ctypes.data, None, None, 31, 0))
    fails(by, R.PushInput(bb.ctypes.data, cnt.ctypes.data, None, None, 31, 64), prm, cp, outs[0], outs[1])
    ok(fr)
    fails(fr, R.PushInput(caps.ctypes.data, cnt.ctypes.data, None, None, 0, 0), prm, cp, outs[0], outs[1])
    # a stamped push without timing
    rx = np.zeros((n, 8), np.uint64)
    ok(fr)
    fails(fr, R.PushInput(caps.ctypes.data, cnt.ctypes.data, rx.ctypes.data, None, 0, 0), prm, cp, outs[0], outs[1])
    # flags before set_lidars / set_scan_filters
    for f in (R.FLAG_PER_STREAM, R.FLAG_PER_STREAM_FILTERS):
        ok(fr)
        fails(fr, pi, R.scan_params(1, 0, 0, 1, f), cp, outs[0], outs[1])
    # misaligned device outputs, in either set
    d = torch.device("cuda", 0)
    tcap = torch.zeros((n, 8, 84), dtype=torch.uint8, device=d)
    tcnt = torch.zeros(n, dtype=torch.int32, device=d)
    bufs = [torch.zeros(1 << 16, dtype=torch.uint8, device=d) for _ in range(2)]
    t64 = [torch.zeros(n * ms + 2, dtype=torch.int64, device=d) for _ in range(2)]
    t32 = [torch.zeros(n * ms + 2, dtype=torch.int32, device=d) for _ in range(2)]
    one = [torch.zeros(2, dtype=torch.int64, device=d) for _ in range(2)]
    s32 = torch.zeros(n + 1, dtype=torch.int32, device=d)
    fd = L.rpl_capsule_stream_push_scan_cloud_msgs_dev
    q = R.PushInput(tcap.data_ptr(), tcnt.data_ptr(), None, None, 31, 0)
    good = [[bufs[k].data_ptr(), t64[k].data_ptr(), t32[k].data_ptr(), one[k].data_ptr()] for k in range(2)]

    def dev_call(g, spsp):
        o = [R.MsgsOut(x[0], 1 << 15, x[1], x[2], x[3]) for x in g]
        r = fd(fr._h, ctypes.byref(q), ctypes.byref(prm), ctypes.byref(cp), 0, ctypes.byref(o[0]), ctypes.byref(o[1]),
               ctypes.c_void_p(spsp), None)
        torch.cuda.synchronize()
        return r

    for k in range(2):
        for j, shift in ((0, 4), (1, 4), (2, 2), (3, 4)):
            assert dev_call(good, s32.data_ptr()) == R.RESULT_OK
            assert fr.scan_cloud_msgs(prm, cp) is not None
            g = [list(x) for x in good]
            g[k][j] += shift
            assert dev_call(g, s32.data_ptr()) == bad, (k, j)
            with pytest.raises(R.RplError):
                fr.scan_cloud_msgs(prm, cp)
    assert dev_call(good, s32.data_ptr() + 2) == bad  # scans_per_stream
    fr.close()
    by.close()
    ctx.close()


def test_per_stream_lidars_on_the_host(R, oracle):
    """RPL_FLAG_PER_STREAM in the host form, a stamped push taking every stream's own timing (timing NULL), with the
    filters"""
    n, ms = 6, 3
    rng = np.random.default_rng(97)
    streams, pieces, stride = pieces_for(oracle, "bytes", 0x84, n, 7400, rng)
    rx = receive_times("bytes", rng, streams, pieces, stride)
    ctx = R.Context(0, 4096, n * ms)
    p = ScanCloudPair(R, ctx, "bytes", 0x84, n, stride, 4096, ms, fleet_filters(R, n), fleet_footprints(R, n),
                      settings=[R.lidar_settings(s % 2, (s // 2) % 2, 1 - s % 2, R.Timing(*TIMINGS[s % len(TIMINGS)]))
                                for s in range(n)])
    prm = flagged(R, R.scan_params(0, 1, 0, 1, R.FLAG_PER_STREAM))
    cps = channel_sets(R)
    for t, push in enumerate(pieces):
        p.push(push, prm, cps[t % 4], 11, rx=rx[t] if t % 2 == 0 else None, timing=False)
        p.compare_after(prm, cps[t % 4], 11)
    assert p.n_msgs > n
    p.close()
    ctx.close()
