"""PointCloud2 messages from the push (rpl_capsule_stream_push_cloud_msgs[_dev]).  Every case pairs two sessions fed the
same pieces: A pushes with the entry point of the push's kind (RPL_FLAG_PER_STREAM iff the cloud takes
RPL_CLOUD_PER_STREAM) and then takes rpl_capsule_stream_cloud_msgs, B takes both from the one call.  The packing is
exact, so offsets, sizes, the total, every written message's bytes and scans_per_stream must equal A's; with a capacity
below the total B writes the prefix of messages that fit and nothing at or past it.  Every later call on the two
sessions must agree."""
import ctypes

import numpy as np
import pytest

from test_gpu_capsule_stream import _pieces_from_cuts, _random_cuts
from test_gpu_stream_push_msgs import CHUNK, GUARD, Pair, lidar_settings, pieces_for, receive_times
from test_gpu_stream_stamps import _normal_rx, _streams
from test_normal_stream_pieces import normal_stream
from test_timestamps_vs_ref import TIMINGS

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def R():
    import rplidar_ros2_driver_b200 as R

    return R


def chains(R, per_stream=False):
    """window only, 5 cm voxels, SOR 8 + 5 cm voxels; each fused and with RPL_CLOUD_NO_FUSED"""
    f = R.CLOUD_PER_STREAM if per_stream else 0
    out = []
    for nf in (0, R.CLOUD_NO_FUSED):
        out += [R.cloud_params(0.2, 30.0, 2.0, flags=f | nf),
                R.cloud_params(0.15, 40.0, 0.0, voxel_size=0.05, is_new_protocol=1, flags=f | nf),
                R.cloud_params(0.15, 40.0, 0.0, voxel_size=0.05, sor_k=8, sor_alpha=1.0, flags=f | nf)]
    return out


def data_offset(frame):
    """where a PointCloud2 message's data starts: the header, then the 116-byte tail"""
    return 4 + ((12 + len(frame) + 1 + 3) & ~3) + 116


class CloudPair(Pair):
    """A: push + cloud_msgs; B: push_cloud_msgs.  Fed identical pieces."""

    def push(self, push, cprm, off, rx=None, dev=False, capacity=None, timing=True):
        R = self.R
        buf, cnt = self.buffers(push)
        prm = R.scan_params(0, 1, 0, 1, R.FLAG_PER_STREAM if cprm.flags & R.CLOUD_PER_STREAM else 0)
        tm = (self.timing if timing else None) if rx is not None else None
        cb = CHUNK if (rx is not None and self.kind != "framed") else None
        if rx is None:
            out = self.A.push(buf, cnt, prm)
        elif self.kind == "framed":
            out = self.A.push(buf, cnt, prm, rx_us=rx, timing=tm)
        else:
            out = self.A.push(buf, cnt, prm, chunk_bytes=CHUNK, chunk_rx_us=rx, timing=tm)
        exp = self.A.cloud_msgs(cprm, off, packed=True)
        got = self.push_b(buf, cnt, cprm, off, rx, tm, cb, dev, capacity)
        assert got["sps"].tolist() == out["scans_per_stream"].tolist()
        self.check(got, exp)
        return got

    def big(self):
        return self.n * self.ms * ((288 + 116 + 16 * self.max_nodes + 1 + 15) // 16 * 16)

    def push_b(self, buf, cnt, cprm, off, rx, tm, cb, dev, capacity):
        ns = self.n * self.ms
        cap = self.big() if capacity is None else capacity
        if not dev:
            store = np.full(cap + 256, GUARD, np.uint8)
            res, sps = self.B.push_cloud_msgs(buf, cnt, cprm, off, rx_us=rx, timing=tm, chunk_bytes=cb,
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
        self.B.push_cloud_msgs_dev(tb.data_ptr(), tc.data_ptr(), cprm, off, store.data_ptr(), cap, offs.data_ptr(),
                                   sizes.data_ptr(), total.data_ptr(), sps.data_ptr(),
                                   rx_us=None if trx is None else trx.data_ptr(), timing=tm, chunk_bytes=cb)
        torch.cuda.synchronize()
        return dict(msgs=store.cpu().numpy(), msg_offsets=offs.cpu().numpy().view(np.uint64),
                    msg_sizes=sizes.cpu().numpy().view(np.uint32), total_bytes=int(total.cpu().numpy()[0]),
                    sps=sps.cpu().numpy().view(np.uint32), result=None, capacity=cap)

    def check(self, got, exp):
        R = self.R
        cap, total = got["capacity"], exp["total_bytes"]
        offs, sizes = exp["msg_offsets"], exp["msg_sizes"]
        assert got["total_bytes"] == total
        assert got["msg_offsets"].tolist() == offs.tolist()
        if got["result"] is not None:  # the host form's code; the device form reports through total_bytes only
            assert got["result"] == (R.RESULT_OK if total <= cap else R.capi.RESULT_INSUFFICIENT_MEMORY)
        fits = (sizes > 0) & (offs + sizes.astype(np.uint64) <= cap)
        assert got["msg_sizes"].tolist() == np.where(fits, sizes, 0).tolist()
        buf, ref = got["msgs"], exp["msgs"]
        for i in np.flatnonzero(fits):
            o, n = int(offs[i]), int(sizes[i])
            assert bytes(buf[o:o + n]) == bytes(ref[o:o + n]), i
            self.n_msgs += 1
        assert (buf[min(total, cap):] == GUARD).all()


def run_pieces(p, pieces, cps, off, dev, rx=None, check_after=True):
    prm = p.R.scan_params(1, 0, 1, 1)
    for t, push in enumerate(pieces):
        d = dev(t) if callable(dev) else dev
        p.push(push, cps[t % len(cps)], off, rx=rx[t] if rx is not None and t % 2 == 0 else None, dev=d)
        if check_after:
            p.compare_after(prm, cps[t % len(cps)], off)


CASES = [("framed", a) for a in (0x82, 0x83, 0x84, 0x85, 0x86)] + \
        [("bytes", a) for a in (0x81, 0x82, 0x83, 0x84, 0x85, 0x86)]


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
@pytest.mark.parametrize("kind,ans", CASES)
def test_every_answer_type(R, oracle, kind, ans, dev):
    """stamped and unstamped pushes on one session with a nonzero clock offset, a reset between pushes, scans dropped
    past max_scans, every chain fused and not; the device cases with RPL_CLOUD_PER_STREAM over mixed lidar settings"""
    O = oracle
    n, ms = 6, 3
    rng = np.random.default_rng(ans * 4 + dev + (kind == "bytes") * 2 + 100)
    streams, pieces, stride = pieces_for(O, kind, ans, n, 7100 + ans, rng)
    rx = receive_times(kind, rng, streams, pieces, stride)
    ctx = R.Context(0, 4096, n * ms)
    p = CloudPair(R, ctx, kind, ans, n, stride, 4096, ms, settings=lidar_settings(R, n) if dev else None)
    assert {data_offset(f) % 16 == 0 for f in p.frames} == {True, False}  # both data paths of the writer
    cps = chains(R, per_stream=dev)
    off = -1_234_567_891 if dev else 987_654_321
    prm = R.scan_params(1, 0, 1, 1)
    for t, push in enumerate(pieces):
        p.push(push, cps[t % len(cps)], off, rx=rx[t] if t % 2 == 0 else None, dev=dev, timing=not dev)
        p.compare_after(prm, cps[(t + 1) % len(cps)], off)
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
    rng = np.random.default_rng(31 + dev)
    before_s = [_streams(O, t, 1, 310 + s)[0].reshape(-1) for s, t in enumerate(types)]
    after_s = [_streams(O, t, 1, 410 + s)[0].reshape(-1) for s, t in enumerate(after)]
    cut = lambda b: _random_cuts(rng, len(b), [1, 83, 85, 4000, 20000])  # noqa: E731
    p1, _ = _pieces_from_cuts(before_s, [cut(b) for b in before_s])
    p2, _ = _pieces_from_cuts(after_s, [cut(b) for b in after_s])
    stride = max(len(x) for push in p1 + p2 for x in push)
    rx1 = _normal_rx(rng, p1, stride, CHUNK)[0]
    ctx = R.Context(0, 4096, n * ms)
    p = CloudPair(R, ctx, "bytes", 0, n, stride, 4096, ms, types=types)
    cps = chains(R)
    prm = R.scan_params(1, 0, 1, 1)
    for t, push in enumerate(p1):
        p.push(push, cps[t % 6], 5, rx=rx1[t] if t % 2 else None, dev=dev)
        p.compare_after(prm, cps[t % 6], 5)
    for x in (p.A, p.B):
        x.set_answer_types(after)
    for t, push in enumerate(p2):
        p.push(push, cps[(t + 3) % 6], 5, dev=dev)
        p.compare_after(prm, cps[t % 6], 5)
    assert p.n_msgs > n
    p.close()
    ctx.close()


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
def test_large_revolutions_and_duplicate_keys(R, oracle, dev):
    """max_nodes 8192 with revolutions above 4096 nodes (0x81: the fused kernel hands them to the general kernel and
    the post passes restricted to the hand-off list), and the ultra feed's duplicate measured keys"""
    O = oracle
    n, ms = 4, 3
    streams = [normal_stream(30000, 177 + s, nodes_per_rev=3900 + 700 * s, noise=50) for s in range(n)]
    rng = np.random.default_rng(15 + dev)
    cuts = [_random_cuts(rng, len(b), [1, 4, 5000, 40000]) for b in streams]
    pieces, _ = _pieces_from_cuts(streams, cuts)
    stride = max(len(x) for push in pieces for x in push)
    ctx = R.Context(0, 8192, n * ms)
    p = CloudPair(R, ctx, "bytes", 0x81, n, stride, 8192, ms)
    run_pieces(p, pieces, chains(R), 0, dev)
    assert p.n_msgs > n
    p.close()
    ctx.close()
    streams, pieces, stride = pieces_for(O, "framed", 0x84, 6, 8200, np.random.default_rng(4))
    ctx = R.Context(0, 4096, 18)
    p = CloudPair(R, ctx, "framed", 0x84, 6, stride, 4096, 3)
    run_pieces(p, pieces, chains(R)[::-1], 0, dev)
    p.close()
    ctx.close()


def test_carry_across_chunks_lanes_and_forms(R, oracle):
    """23 streams: device chunks of 7 (the context's max_scans) and host chunks of 4 (the 16 MiB input rule), so that
    the directory's carry crosses chunk and lane boundaries; host and device calls alternate on one session, and the
    last chunks publish nothing"""
    O = oracle
    n, ms = 23, 3
    streams = [c.reshape(-1) for c in _streams(O, 0x82, n, 1300)]
    rng = np.random.default_rng(19)
    cuts = [_random_cuts(rng, len(b), [1, 83, 85, 4000, 20000]) for b in streams]
    pieces, _ = _pieces_from_cuts(streams, cuts)
    for push in pieces[::2]:  # streams 16..22 (the last device chunk, and most of the last two host chunks) idle
        for s in range(16, n):
            push[s] = push[s][:0]
    stride = (16 << 20) // 5 + 1  # 16 MiB // stride = 4 streams per host chunk
    rx = _normal_rx(rng, pieces, stride, CHUNK)[0]
    ctx = R.Context(0, 4096, 7 * ms)
    p = CloudPair(R, ctx, "bytes", 0x82, n, stride, 4096, ms)
    run_pieces(p, pieces, chains(R), 42, lambda t: (t // 2) % 2 == 1, rx=rx)
    assert p.n_msgs > n
    p.close()
    ctx.close()


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
def test_capacity(R, oracle, dev):
    """capacity 0, total - 1, exactly the total, and cuts inside a middle message and at a message's end (across the
    chunks of a several-chunk push): only the fitting prefix is written, the guard bytes behind it stay; then every
    message again from cloud_msgs on the same push"""
    O = oracle
    n, ms = 9, 3
    rng = np.random.default_rng(41 + dev)
    streams, pieces, stride = pieces_for(O, "framed", 0x85, n, 5200, rng)
    ctx = R.Context(0, 4096, 3 * ms)  # device chunks of 3 streams
    p = CloudPair(R, ctx, "framed", 0x85, n, stride, 4096, ms)
    probe = CloudPair(R, ctx, "framed", 0x85, n, stride, 4096, ms)
    cps = chains(R)
    prm = R.scan_params(1, 0, 0, 1)
    n_cut = 0
    for t, push in enumerate(pieces):
        cp = cps[t % len(cps)]
        full = probe.push(push, cp, 7)  # the totals and offsets of this push
        offs, sizes, total = full["msg_offsets"], full["msg_sizes"], full["total_bytes"]
        used = np.flatnonzero(sizes)
        caps = [0, max(total - 1, 0), total]
        if len(used) >= 3:
            mid = int(used[len(used) // 2])
            caps += [int(offs[mid]) + 8, int(offs[mid]) + int(sizes[mid])]
        cap = caps[t % len(caps)]
        got = p.push(push, cp, 7, dev=dev, capacity=cap)
        assert got["total_bytes"] == total
        n_cut += int(0 < (got["msg_sizes"] > 0).sum() < len(used))
        assert p.B.cloud_msgs(cp, 7) == p.A.cloud_msgs(cp, 7)  # recovery
        p.compare_after(prm, cp, 7)
    assert n_cut > 0
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
    cp = R.cloud_params(voxel_size=0.05)
    caps = np.zeros((n, 8, 84), np.uint8)
    cnt = np.zeros(n, np.uint32)
    msgs = np.zeros(1 << 16, np.uint8)
    offs, sizes, total, sps = np.zeros(n * ms, np.uint64), np.zeros(n * ms, np.uint32), np.zeros(1, np.uint64), \
        np.zeros(n, np.uint32)
    P = lambda a: ctypes.c_void_p(a.ctypes.data)  # noqa: E731
    pi = R.PushInput(caps.ctypes.data, cnt.ctypes.data, None, None, 31, 0)
    fn = L.rpl_capsule_stream_push_cloud_msgs
    bad = R.RESULT_INVALID_DATA

    def fails(sess, q, c):
        """the call fails its checks and leaves no last push, as a failed push does"""
        r = fn(sess._h, None if q is None else ctypes.byref(q), None if c is None else ctypes.byref(c), 0, P(msgs),
               msgs.size, P(offs), P(sizes), P(total), P(sps))
        with pytest.raises(R.RplError):
            sess.cloud_msgs(cp)
        return r == bad

    def ok(sess, q):
        assert fn(sess._h, ctypes.byref(q), ctypes.byref(cp), 0, P(msgs), msgs.size, P(offs), P(sizes), P(total),
                  P(sps)) == R.RESULT_OK
        assert sess.cloud_msgs(cp) is not None

    ok(fr, pi)
    assert fails(fr, None, cp)
    ok(fr, pi)
    assert fails(fr, pi, None)
    for k in range(5):
        ok(fr, pi)
        a = [P(msgs), P(offs), P(sizes), P(total), P(sps)]
        a[k] = None
        assert fn(fr._h, ctypes.byref(pi), ctypes.byref(cp), 0, a[0], msgs.size, a[1], a[2], a[3], a[4]) == bad
        with pytest.raises(R.RplError):
            fr.cloud_msgs(cp)
    for field in ("data", "counts"):
        ok(fr, pi)
        q = R.PushInput(caps.ctypes.data, cnt.ctypes.data, None, None, 31, 0)
        setattr(q, field, None)
        assert fails(fr, q, cp)
    # chunk_bytes on a framed session and on an unstamped byte push
    ok(fr, pi)
    assert fails(fr, R.PushInput(caps.ctypes.data, cnt.ctypes.data, None, None, 31, 64), cp)
    bb = np.zeros((n, 256), np.uint8)
    ok(by, R.PushInput(bb.ctypes.data, cnt.ctypes.data, None, None, 31, 0))
    assert fails(by, R.PushInput(bb.ctypes.data, cnt.ctypes.data, None, None, 31, 64), cp)
    # a stamped push without timing, or with chunk_bytes 0 on a byte session; the unstamped sample duration rule
    rx = np.zeros((n, 8), np.uint64)
    ok(fr, pi)
    assert fails(fr, R.PushInput(caps.ctypes.data, cnt.ctypes.data, rx.ctypes.data, None, 0, 0), cp)
    rxb = np.zeros((n, 4), np.uint64)
    tm = R.Timing(*TIMINGS[0])
    ok(by, R.PushInput(bb.ctypes.data, cnt.ctypes.data, None, None, 31, 0))
    assert fails(by, R.PushInput(bb.ctypes.data, cnt.ctypes.data, rxb.ctypes.data, ctypes.pointer(tm), 0, 0), cp)
    ok(fr, pi)
    assert fails(fr, R.PushInput(caps.ctypes.data, cnt.ctypes.data, None, None, 0, 0), cp)
    # the cloud chain's rules, and RPL_CLOUD_PER_STREAM before set_lidars
    for c in (R.cloud_params(sor_k=33), R.cloud_params(voxel_size=1e-7), R.cloud_params(voxel_size=0.05,
                                                                                         range_max=1000.0),
              R.cloud_params(flags=R.CLOUD_PER_STREAM)):
        ok(fr, pi)
        assert fails(fr, pi, c)
    # misaligned device outputs
    d = torch.device("cuda", 0)
    tcap = torch.zeros((n, 8, 84), dtype=torch.uint8, device=d)
    tcnt = torch.zeros(n, dtype=torch.int32, device=d)
    buf = torch.zeros(1 << 16, dtype=torch.uint8, device=d)
    t64 = torch.zeros(n * ms + 2, dtype=torch.int64, device=d)
    t32 = torch.zeros(n * ms + 2, dtype=torch.int32, device=d)
    one = torch.zeros(2, dtype=torch.int64, device=d)
    s32 = torch.zeros(n + 1, dtype=torch.int32, device=d)
    fd = L.rpl_capsule_stream_push_cloud_msgs_dev
    q = R.PushInput(tcap.data_ptr(), tcnt.data_ptr(), None, None, 31, 0)
    good = [buf.data_ptr(), t64.data_ptr(), t32.data_ptr(), one.data_ptr(), s32.data_ptr()]
    for k, shift in ((0, 4), (1, 4), (2, 2), (3, 4), (4, 2)):
        v = [ctypes.c_void_p(x) for x in good]
        assert fd(fr._h, ctypes.byref(q), ctypes.byref(cp), 0, v[0], 1 << 15, v[1], v[2], v[3], v[4], None) == \
            R.RESULT_OK
        torch.cuda.synchronize()
        assert fr.cloud_msgs(cp) is not None
        a = list(good)
        a[k] += shift
        v = [ctypes.c_void_p(x) for x in a]
        assert fd(fr._h, ctypes.byref(q), ctypes.byref(cp), 0, v[0], 1 << 15, v[1], v[2], v[3], v[4], None) == bad, k
        with pytest.raises(R.RplError):
            fr.cloud_msgs(cp)
    fr.close()
    by.close()
    ctx.close()


def test_per_stream_settings_on_the_host(R, oracle):
    """RPL_CLOUD_PER_STREAM in the host form, a stamped push taking every stream's own timing (timing NULL)"""
    O = oracle
    n, ms = 6, 3
    rng = np.random.default_rng(77)
    streams, pieces, stride = pieces_for(O, "bytes", 0x84, n, 7300, rng)
    rx = receive_times("bytes", rng, streams, pieces, stride)
    ctx = R.Context(0, 4096, n * ms)
    p = CloudPair(R, ctx, "bytes", 0x84, n, stride, 4096, ms, settings=lidar_settings(R, n))
    cps = chains(R, per_stream=True)
    prm = R.scan_params(0, 1, 0, 1, R.FLAG_PER_STREAM)
    for t, push in enumerate(pieces):
        p.push(push, cps[t % 6], 11, rx=rx[t] if t % 2 == 0 else None, timing=False)
        p.compare_after(prm, cps[t % 6], 11)
    assert p.n_msgs > n
    p.close()
    ctx.close()
