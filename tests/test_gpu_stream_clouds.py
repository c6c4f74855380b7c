"""Per-stream clouds (rpl_capsule_stream_set_clouds, RPL_CLOUD_PER_STREAM_CHAIN).  Every case feeds a fleet session and,
for each of its streams, a session of that stream alone the same pieces.  With the flag, every output of an enabled
stream -- point counts, xyzi rows, message sizes and bytes -- must be what its lone session gives with uniform
rpl_cloud_params equal to the stream's resolved entry; a disabled stream has point count 0, untouched rows and no
message.  The fleets mix every route: window only, a voxel grid or SOR the fused kernel takes, a voxel grid too fine for
its 16-bit cell keys (the separate passes), and no cloud."""
import ctypes

import numpy as np
import pytest

from test_gpu_capsule_stream import _pieces_from_cuts, _random_cuts
from test_gpu_stream_push_msgs import CHUNK, FRAMES, make_session, pieces_for, receive_times
from test_gpu_stream_stamps import _normal_rx, _streams
from test_normal_stream_pieces import normal_stream
from test_timestamps_vs_ref import TIMINGS

pytestmark = pytest.mark.gpu
FILL = np.float32(-7.25)  # rows a call must not write


@pytest.fixture(scope="module")
def R():
    import rplidar_ros2_driver_b200 as R

    return R


def fleet_settings(R, n):
    """every route: window only (range_max 0: the frame's), 5 cm voxels, SOR 8 + voxels, no cloud, 1 mm voxels at 40 m
    (past the fused kernel's cell keys) with SOR 4, SOR 12 with an intensity floor, SOR 32 + 4 m voxels"""
    table = [
        R.cloud_settings(0.2, 0.0, 0.0),
        R.cloud_settings(0.15, 0.0, 0.0, voxel_size=0.05),
        R.cloud_settings(0.15, 30.0, 0.0, voxel_size=0.05, sor_k=8, sor_alpha=1.0),
        R.cloud_settings(0.15, 40.0, 0.0, voxel_size=0.05, enabled=False),
        R.cloud_settings(0.1, 40.0, 0.0, voxel_size=0.001, sor_k=4, sor_alpha=0.5),
        R.cloud_settings(0.3, 25.0, 2.0, sor_k=12, sor_alpha=2.0),
        R.cloud_settings(0.15, 0.0, 1.0, voxel_size=4.0, sor_k=32, sor_alpha=1.0),
    ]
    return [table[s % len(table)] for s in range(n)]


def lidar_settings(R, n):
    return [R.lidar_settings(s % 2, (s // 2) % 2, (s // 4) % 2, R.Timing(*TIMINGS[s % len(TIMINGS)])) for s in range(n)]


def uniform(R, e, rmax, flags, newp=0):
    """the rpl_cloud_params of a lone session for table entry e (range_max resolved)"""
    return R.cloud_params(e.range_min, e.range_max or rmax, e.intensity_min, e.voxel_size, e.sor_k, e.sor_alpha, newp,
                          flags & ~R.CLOUD_PER_STREAM_CHAIN)


class Fleet:
    """F: the fleet session with the table; S[s]: stream s alone.  Fed identical pieces."""

    def __init__(self, R, ctx, kind, ans, n, stride, max_nodes, ms, table, lidars=None, types=None):
        self.R, self.kind, self.n, self.stride, self.ms, self.max_nodes = R, kind, n, stride, ms, max_nodes
        self.F = make_session(R, ctx, kind, ans, n, stride, max_nodes, ms, types)
        self.S = [make_session(R, ctx, kind, ans, 1, stride, max_nodes, ms, None if types is None else [types[s]])
                  for s in range(n)]
        self.frames = [FRAMES[s % len(FRAMES)] for s in range(n)]
        self.rmax = np.linspace(0.5, 40.0, n).astype(np.float32)
        self.F.set_frames(self.frames, self.rmax)
        for s, x in enumerate(self.S):
            x.set_frames([self.frames[s]], self.rmax[s:s + 1])
        self.lidars = lidars
        if lidars:
            self.F.set_lidars(lidars)
            for s, x in enumerate(self.S):
                x.set_lidars([lidars[s]])
        self.table = list(table)
        self.F.set_clouds(self.table)
        self.timing = R.Timing(*TIMINGS[0])
        self.n_clouds = 0

    def set_frames_range(self, rmax):
        self.rmax = np.asarray(rmax, np.float32)
        self.F.set_frames(self.frames, self.rmax)
        for s, x in enumerate(self.S):
            x.set_frames([self.frames[s]], self.rmax[s:s + 1])

    def set_clouds(self, table, mask=None):
        self.F.set_clouds(table, mask)
        self.table = [table[s] if mask is None or mask[s] else self.table[s] for s in range(self.n)]

    def buffers(self, push, streams):
        if self.kind == "framed":
            buf = np.zeros((len(streams), self.stride, self.F.capsule_bytes), np.uint8)
        else:
            buf = np.full((len(streams), self.stride), 0xEE, np.uint8)
        cnt = np.zeros(len(streams), np.uint32)
        for j, s in enumerate(streams):
            buf[j, : len(push[s])] = push[s]
            cnt[j] = len(push[s])
        return buf, cnt

    def _push(self, x, buf, cnt, prm, rx):
        if rx is None:
            return x.push(buf, cnt, prm)
        tm = None if prm.flags & self.R.FLAG_PER_STREAM else self.timing
        if self.kind == "framed":
            return x.push(buf, cnt, prm, rx_us=rx, timing=tm)
        return x.push(buf, cnt, prm, chunk_bytes=CHUNK, chunk_rx_us=rx, timing=tm)

    def scan_params(self):
        R = self.R
        return R.scan_params(1, 0, 1, 1, R.FLAG_PER_STREAM if self.lidars else 0)

    def push(self, push, rx=None):
        """a LaserScan push on every session"""
        prm = self.scan_params()
        sps = self._push(self.F, *self.buffers(push, range(self.n)), prm, rx)["scans_per_stream"]
        for s, x in enumerate(self.S):
            o = self._push(x, *self.buffers(push, [s]), prm, None if rx is None else rx[s:s + 1])
            assert o["scans_per_stream"][0] == sps[s]

    def params(self, flags):
        R = self.R
        f = flags | R.CLOUD_PER_STREAM_CHAIN | (R.CLOUD_PER_STREAM if self.lidars else 0)
        return R.cloud_params(0.5, 1.0, 9.0, 0.0, 0, 1.0, 1, f)  # the six chain fields are the table's

    def lone(self, s, flags):
        R = self.R
        return uniform(R, self.table[s], self.rmax[s], flags | (R.CLOUD_PER_STREAM if self.lidars else 0), 1)

    # ---- checks of the calls on the last push ----
    def check_cloud(self, flags, dev=False):
        ms = self.ms
        got = self._cloud(self.F, self.params(flags), dev)
        for s, x in enumerate(self.S):
            c, xyz = got["point_counts"][s * ms:(s + 1) * ms], got["xyzi"][s * ms:(s + 1) * ms]
            if not self.table[s].enabled:  # its rows untouched (the host form copies whole rows back)
                assert (c == 0).all() and (not dev or (xyz == FILL).all()), s
                continue
            exp = x.cloud(self.lone(s, flags))
            assert c.tolist() == exp["point_counts"].tolist(), s
            for k in range(ms):
                assert xyz[k, : c[k]].tobytes() == exp["xyzi"][k, : c[k]].tobytes(), (s, k)
                self.n_clouds += int(c[k] > 0)

    def _cloud(self, x, prm, dev):
        ns = self.n * self.ms
        if not dev:
            return x.cloud(prm, out=dict(xyzi=np.full((ns, self.max_nodes, 4), FILL, np.float32),
                                         point_counts=np.full(ns, 0xFFFF, np.uint32)))
        import torch

        d = torch.device("cuda", 0)
        xyzi = torch.full((ns, self.max_nodes, 4), float(FILL), dtype=torch.float32, device=d)
        cnt = torch.full((ns,), 0xFFFF, dtype=torch.int32, device=d)
        x.cloud_dev(prm, xyzi.data_ptr(), cnt.data_ptr())
        torch.cuda.synchronize()
        return dict(xyzi=xyzi.cpu().numpy(), point_counts=cnt.cpu().numpy().view(np.uint32))

    def check_msgs(self, flags, off, dev=False):
        ms = self.ms
        got = self._msgs(self.F, self.params(flags), off, dev)
        for s, x in enumerate(self.S):
            exp = [None] * ms if not self.table[s].enabled else x.cloud_msgs(self.lone(s, flags), off)
            assert got[s * ms:(s + 1) * ms] == exp, s

    def _msgs(self, x, prm, off, dev):
        if not dev:
            res = x.cloud_msgs(prm, off, packed=True)
            check_packing(res["msgs"], res["msg_offsets"], res["msg_sizes"], res["total_bytes"])
            return [bytes(res["msgs"][o: o + n]) if n else None
                    for o, n in zip(res["msg_offsets"].tolist(), res["msg_sizes"].tolist())]
        import torch

        d = torch.device("cuda", 0)
        ns = self.n * self.ms
        cap = ns * ((288 + 116 + 16 * self.max_nodes + 1 + 15) // 16 * 16)
        store = torch.zeros(cap, dtype=torch.uint8, device=d)
        offs = torch.zeros(ns, dtype=torch.int64, device=d)
        sizes = torch.zeros(ns, dtype=torch.int32, device=d)
        total = torch.zeros(1, dtype=torch.int64, device=d)
        x.cloud_msgs_dev(prm, off, store.data_ptr(), cap, offs.data_ptr(), sizes.data_ptr(), total.data_ptr())
        torch.cuda.synchronize()
        m, o, z = store.cpu().numpy(), offs.cpu().numpy().view(np.uint64), sizes.cpu().numpy().view(np.uint32)
        check_packing(m, o, z, int(total.cpu().numpy()[0]))
        return [bytes(m[a: a + b]) if b else None for a, b in zip(o.tolist(), z.tolist())]

    def push_cloud_msgs(self, push, flags, off, rx=None, dev=False):
        """push_cloud_msgs on the fleet against each lone session's with uniform params"""
        ms = self.ms
        got, sps = self._push_cloud(self.F, self.buffers(push, range(self.n)), self.params(flags), off, rx, dev)
        for s, x in enumerate(self.S):
            exp, esps = self._push_cloud(x, self.buffers(push, [s]), self.lone(s, flags), off,
                                         None if rx is None else rx[s:s + 1], dev)
            assert sps[s] == esps[0], s
            assert got[s * ms:(s + 1) * ms] == (exp if self.table[s].enabled else [None] * ms), s
            self.n_clouds += sum(m is not None for m in exp)

    def _push_cloud(self, x, bufcnt, prm, off, rx, dev):
        R = self.R
        buf, cnt = bufcnt
        tm = (None if prm.flags & R.CLOUD_PER_STREAM else self.timing) if rx is not None else None
        cb = CHUNK if (rx is not None and self.kind != "framed") else None
        nsl = len(cnt) * self.ms
        cap = nsl * ((288 + 116 + 16 * self.max_nodes + 1 + 15) // 16 * 16)
        if not dev:
            res, sps = x.push_cloud_msgs(buf, cnt, prm, off, rx_us=rx, timing=tm, chunk_bytes=cb,
                                         msgs=np.zeros(cap, np.uint8), packed=True)
            m, o, z, t = res["msgs"], res["msg_offsets"], res["msg_sizes"], res["total_bytes"]
        else:
            import torch

            d = torch.device("cuda", 0)
            tb, tc = torch.from_numpy(buf).to(d), torch.from_numpy(cnt.view(np.int32)).to(d)
            trx = None if rx is None else torch.from_numpy(np.ascontiguousarray(rx).view(np.int64)).to(d)
            store = torch.zeros(cap, dtype=torch.uint8, device=d)
            offs = torch.zeros(nsl, dtype=torch.int64, device=d)
            sizes = torch.zeros(nsl, dtype=torch.int32, device=d)
            total = torch.zeros(1, dtype=torch.int64, device=d)
            tsps = torch.zeros(len(cnt), dtype=torch.int32, device=d)
            x.push_cloud_msgs_dev(tb.data_ptr(), tc.data_ptr(), prm, off, store.data_ptr(), cap, offs.data_ptr(),
                                  sizes.data_ptr(), total.data_ptr(), tsps.data_ptr(),
                                  rx_us=None if trx is None else trx.data_ptr(), timing=tm, chunk_bytes=cb)
            torch.cuda.synchronize()
            m, o, z = store.cpu().numpy(), offs.cpu().numpy().view(np.uint64), sizes.cpu().numpy().view(np.uint32)
            t, sps = int(total.cpu().numpy()[0]), tsps.cpu().numpy().view(np.uint32)
        check_packing(m, o, z, t)
        return [bytes(m[a: a + b]) if b else None for a, b in zip(o.tolist(), z.tolist())], sps

    def check_all(self, off, dev):
        """every call on the last push, fused and not"""
        R = self.R
        for flags in (0, R.CLOUD_NO_FUSED):
            self.check_cloud(flags, dev)
            self.check_msgs(flags, off, dev)

    def close(self):
        self.F.close()
        for x in self.S:
            x.close()


def check_packing(msgs, offs, sizes, total):
    """the exclusive scan of the sizes rounded up to 16; a slot without a message takes no room"""
    rounded = (sizes.astype(np.int64) + 15) // 16 * 16
    assert offs.astype(np.int64).tolist() == np.concatenate([[0], np.cumsum(rounded)[:-1]]).tolist()
    used = sizes > 0
    assert total == (int((offs.astype(np.int64) + sizes)[used].max()) if used.any() else 0)


CASES = [("framed", a) for a in (0x82, 0x83, 0x84, 0x85, 0x86)] + \
        [("bytes", a) for a in (0x81, 0x82, 0x83, 0x84, 0x85, 0x86)]


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
@pytest.mark.parametrize("kind,ans", CASES)
def test_every_answer_type(R, oracle, kind, ans, dev):
    """stamped and unstamped pushes; cloud, cloud_msgs and push_cloud_msgs in the call's form, fused and not; the
    device cases with RPL_CLOUD_PER_STREAM over mixed lidar settings"""
    O = oracle
    n, ms = 7, 3
    rng = np.random.default_rng(ans * 4 + dev + (kind == "bytes") * 2 + 900)
    streams, pieces, stride = pieces_for(O, kind, ans, n, 9100 + ans, rng)
    rx = receive_times(kind, rng, streams, pieces, stride)
    ctx = R.Context(0, 4096, n * ms)
    f = Fleet(R, ctx, kind, ans, n, stride, 4096, ms, fleet_settings(R, n), lidars=lidar_settings(R, n) if dev else None)
    for t, push in enumerate(pieces):
        r = rx[t] if t % 2 == 0 else None
        if t % 2 == 0:
            f.push(push, rx=r)
            f.check_all(11, dev)
        else:
            f.push_cloud_msgs(push, R.CLOUD_NO_FUSED if t % 4 == 3 else 0, -5, rx=r, dev=dev)
            f.check_cloud(0, not dev)
    assert f.n_clouds > n
    f.close()
    ctx.close()


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
def test_mixed_byte_session_with_a_switch(R, oracle, dev):
    O = oracle
    types = [0x81, 0x82, 0x83, 0x84, 0x85, 0x86, 0x82]
    after = [0x85, 0x86, 0x81, 0x82, 0x83, 0x84, 0x81]
    n, ms = len(types), 3
    rng = np.random.default_rng(51 + dev)
    before_s = [_streams(O, t, 1, 510 + s)[0].reshape(-1) for s, t in enumerate(types)]
    after_s = [_streams(O, t, 1, 610 + s)[0].reshape(-1) for s, t in enumerate(after)]
    cut = lambda b: _random_cuts(rng, len(b), [1, 83, 85, 4000, 20000])  # noqa: E731
    p1, _ = _pieces_from_cuts(before_s, [cut(b) for b in before_s])
    p2, _ = _pieces_from_cuts(after_s, [cut(b) for b in after_s])
    stride = max(len(x) for push in p1 + p2 for x in push)
    rx1 = _normal_rx(rng, p1, stride, CHUNK)[0]
    ctx = R.Context(0, 4096, n * ms)
    f = Fleet(R, ctx, "bytes", 0, n, stride, 4096, ms, fleet_settings(R, n)[::-1], types=types)
    for t, push in enumerate(p1):
        f.push_cloud_msgs(push, 0, 5, rx=rx1[t] if t % 2 else None, dev=dev)
        f.check_all(5, dev)
    f.F.set_answer_types(after)
    for s, x in enumerate(f.S):
        x.set_answer_types([after[s]])
    for t, push in enumerate(p2):
        f.push(push)
        f.check_all(5, dev)
    assert f.n_clouds > n
    f.close()
    ctx.close()


@pytest.mark.parametrize("dev", [False, True], ids=["host", "dev"])
def test_large_revolutions_and_duplicate_keys(R, oracle, dev):
    """max_nodes 8192 with revolutions above 4096 nodes (the fused kernel hands them to the general kernel and the post
    passes restricted to the hand-off list), and the ultra feed's duplicate measured keys"""
    O = oracle
    n, ms = 7, 3
    streams = [normal_stream(30000, 277 + s, nodes_per_rev=3500 + 600 * s, noise=50) for s in range(n)]
    rng = np.random.default_rng(25 + dev)
    cuts = [_random_cuts(rng, len(b), [1, 4, 5000, 40000]) for b in streams]
    pieces, _ = _pieces_from_cuts(streams, cuts)
    stride = max(len(x) for push in pieces for x in push)
    ctx = R.Context(0, 8192, n * ms)
    f = Fleet(R, ctx, "bytes", 0x81, n, stride, 8192, ms, fleet_settings(R, n))
    for t, push in enumerate(pieces):
        if t % 2:
            f.push_cloud_msgs(push, 0, 0, dev=dev)
        else:
            f.push(push)
        f.check_all(0, dev)
    f.close()
    streams, pieces, stride = pieces_for(O, "framed", 0x84, n, 8300, np.random.default_rng(5))
    f = Fleet(R, ctx, "framed", 0x84, n, stride, 4096, ms, fleet_settings(R, n)[3:] + fleet_settings(R, n)[:3])
    for t, push in enumerate(pieces):
        f.push(push)
        f.check_all(0, dev)
    assert f.n_clouds > n
    f.close()
    ctx.close()


def test_several_chunks_per_push(R, oracle):
    """23 streams in device chunks of 3 and host chunks of 4, host and device calls alternating on one session"""
    O = oracle
    n, ms = 23, 3
    streams = [c.reshape(-1) for c in _streams(O, 0x82, n, 1700)]
    rng = np.random.default_rng(29)
    cuts = [_random_cuts(rng, len(b), [1, 83, 85, 4000, 20000]) for b in streams]
    pieces, _ = _pieces_from_cuts(streams, cuts)
    stride = (16 << 20) // 5 + 1  # 16 MiB // stride = 4 streams per host chunk
    rx = _normal_rx(rng, pieces, stride, CHUNK)[0]
    ctx = R.Context(0, 4096, 3 * ms)
    f = Fleet(R, ctx, "bytes", 0x82, n, stride, 4096, ms, fleet_settings(R, n))
    for t, push in enumerate(pieces):
        dev = (t // 2) % 2 == 1
        f.push_cloud_msgs(push, R.CLOUD_NO_FUSED if t % 3 == 2 else 0, 42, rx=rx[t] if t % 2 == 0 else None, dev=dev)
        f.check_all(42, not dev)
    assert f.n_clouds > n
    f.close()
    ctx.close()


def test_range_max_follows_frames_and_masked_reconfiguration(R, oracle):
    """range_max 0 takes set_frames' range_max when the call is made (a set_frames between two calls on one push moves
    the window); masked set_clouds between pushes; a set_frames that moves a 0 entry with a voxel grid past 1000 m
    fails the next flagged call, and a later set_frames mends it"""
    O = oracle
    n, ms = 7, 3
    rng = np.random.default_rng(77)
    streams, pieces, stride = pieces_for(O, "framed", 0x85, n, 7700, rng)
    ctx = R.Context(0, 4096, n * ms)
    f = Fleet(R, ctx, "framed", 0x85, n, stride, 4096, ms, fleet_settings(R, n))
    new = [R.cloud_settings(0.15, 0.0, 0.0, voxel_size=0.02, sor_k=6) if s % 2 else
           R.cloud_settings(0.5, 0.0, 3.0, enabled=s != 4) for s in range(n)]
    mask = np.array([s % 3 != 0 for s in range(n)], np.uint8)
    for t, push in enumerate(pieces):
        f.push(push)
        f.check_all(3, False)
        f.set_frames_range(f.rmax[::-1].copy())
        f.check_all(3, t % 2 == 1)
        if t == 1:
            f.set_clouds(new, mask)
    before = f.rmax.copy()
    f.set_frames_range(np.full(n, 1500.0, np.float32))  # stream 1: 5 cm voxels at range_max 0
    with pytest.raises(R.RplError):
        f.F.cloud(f.params(0))
    with pytest.raises(R.RplError):
        f.F.cloud_msgs(f.params(0))
    f.set_frames_range(before)
    f.check_all(3, False)
    assert f.n_clouds > n
    f.close()
    ctx.close()


def test_uniform_table_is_the_flagless_call(R, oracle):
    """a table with every stream's entry equal to the call's params gives exactly the flagless call's outputs, and the
    flag after push_laserscan_msgs takes that push's scans"""
    O = oracle
    n, ms = 6, 3
    rng = np.random.default_rng(3)
    streams, pieces, stride = pieces_for(O, "bytes", 0x84, n, 3300, rng)
    ctx = R.Context(0, 4096, n * ms)
    s = make_session(R, ctx, "bytes", 0x84, n, stride, 4096, ms)
    fleet = Fleet(R, ctx, "bytes", 0x84, n, stride, 4096, ms, fleet_settings(R, n))
    for e in (R.cloud_params(0.2, 30.0, 2.0), R.cloud_params(0.15, 40.0, 0.0, voxel_size=0.05),
              R.cloud_params(0.15, 40.0, 0.0, voxel_size=0.05, sor_k=8, sor_alpha=1.0),
              R.cloud_params(0.15, 40.0, 0.0, voxel_size=0.001, sor_k=3)):
        s.set_clouds([R.cloud_settings(e.range_min, e.range_max, e.intensity_min, e.voxel_size, e.sor_k, e.sor_alpha)]
                     * n)
        for t, push in enumerate(pieces):
            buf, cnt = fleet.buffers(push, range(n))
            s.push(buf, cnt, R.scan_params(1, 0, 1, 1))
            for nf in (0, R.CLOUD_NO_FUSED):
                flagged = R.cloud_params(9.0, 1.0, 99.0, 0.0, 0, 1.0, 0, nf | R.CLOUD_PER_STREAM_CHAIN)
                plain = R.cloud_params(e.range_min, e.range_max, e.intensity_min, e.voxel_size, e.sor_k, e.sor_alpha,
                                       0, nf)
                a, b = s.cloud(flagged), s.cloud(plain)
                assert a["point_counts"].tolist() == b["point_counts"].tolist()
                assert a["xyzi"].tobytes() == b["xyzi"].tobytes()
                assert s.cloud_msgs(flagged, 9) == s.cloud_msgs(plain, 9)
    # push_laserscan_msgs, then a flagged cloud_msgs on the fleet: the lone sessions' after their pushes
    for push in pieces[:3]:
        res, sps = fleet.F.push_laserscan_msgs(*fleet.buffers(push, range(n)), R.scan_params(1, 0, 1, 1))
        for j, x in enumerate(fleet.S):
            x.push_laserscan_msgs(*fleet.buffers(push, [j]), R.scan_params(1, 0, 1, 1))
        fleet.check_all(1, False)
    s.close()
    fleet.close()
    ctx.close()


def test_argument_checks(R, oracle):
    n, ms = 3, 2
    ctx = R.Context(0, 4096, n * ms)
    s = R.CapsuleStreamSession(ctx, 0x85, n, 8, 4096, ms)
    L = R.lib()
    bad = R.RESULT_INVALID_DATA
    flagged = R.cloud_params(flags=R.CLOUD_PER_STREAM_CHAIN)
    ok = [R.cloud_settings(voxel_size=0.05)] * n
    arr = lambda t: ctypes.cast((R.CloudSettings * n)(*t), ctypes.c_void_p)  # noqa: E731
    mask = lambda m: np.ascontiguousarray(m, np.uint8).ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    caps, cnt = np.zeros((n, 8, 84), np.uint8), np.zeros(n, np.uint32)
    s.push(caps, cnt, R.scan_params(1, 0, 0, 1))
    # the flag before the first set_clouds
    for call in (lambda: s.cloud(flagged), lambda: s.cloud_msgs(flagged),
                 lambda: s.push_cloud_msgs(caps, cnt, flagged)):
        with pytest.raises(R.RplError):
            call()
    s.push(caps, cnt, R.scan_params(1, 0, 0, 1))
    # null table, a first call that leaves a stream out
    assert L.rpl_capsule_stream_set_clouds(s._h, None, None) == bad
    assert L.rpl_capsule_stream_set_clouds(s._h, arr(ok), mask([1, 0, 1])) == bad
    assert L.rpl_capsule_stream_set_clouds(None, arr(ok), None) == bad
    # entries that break the chain's rules, also among otherwise good ones; the table stays as it was (unset)
    for e in (R.cloud_settings(sor_k=33), R.cloud_settings(voxel_size=1e-7), R.cloud_settings(voxel_size=-1.0),
              R.cloud_settings(range_max=1000.0, voxel_size=0.05), R.cloud_settings(voxel_size=float("nan"))):
        assert L.rpl_capsule_stream_set_clouds(s._h, arr([ok[0], e, ok[0]]), None) == bad
    with pytest.raises(R.RplError):
        s.cloud(flagged)
    # a bad entry outside the mask is not read; disabled entries are checked all the same
    s.set_clouds(ok)
    assert L.rpl_capsule_stream_set_clouds(s._h, arr([ok[0], R.cloud_settings(sor_k=99), ok[0]]), mask([1, 0, 1])) == 0
    assert L.rpl_capsule_stream_set_clouds(s._h, arr([R.cloud_settings(sor_k=33, enabled=False)] * n), None) == bad
    s.cloud(flagged)
    # with the flag the call's own chain fields are ignored, even where they break the rules
    s.cloud(R.cloud_params(sor_k=99, voxel_size=-3.0, range_max=5000.0, flags=R.CLOUD_PER_STREAM_CHAIN))
    s.cloud_msgs(R.cloud_params(sor_k=99, flags=R.CLOUD_PER_STREAM_CHAIN))
    # RPL_CLOUD_PER_STREAM still needs set_lidars
    with pytest.raises(R.RplError):
        s.cloud(R.cloud_params(flags=R.CLOUD_PER_STREAM_CHAIN | R.CLOUD_PER_STREAM))
    # a 0 range_max entry with a voxel grid resolved past 1000 m
    s.set_frames(["a"] * n, np.array([12.0, 1000.0, 12.0], np.float32))
    with pytest.raises(R.RplError):
        s.cloud(flagged)
    with pytest.raises(R.RplError):
        s.push_cloud_msgs(caps, cnt, flagged)
    s.set_frames(["a"] * n, np.array([12.0, 999.0, 12.0], np.float32))
    s.push(caps, cnt, R.scan_params(1, 0, 0, 1))
    s.cloud(flagged)
    # calls without the flag ignore the table
    s.cloud(R.cloud_params())
    s.close()
    ctx.close()
